// nidx_b200 — NidxSearcher.Suggest's paragraph pass on the device (sm_90a): the fuzzy fallback and the suggest mask
// (reference: nidx_paragraph/src/reader.rs:58-90 suggest, search_query.rs:87-183 suggest_query, query_parser/fuzzy_parser.rs,
//  fuzzy_query.rs:88-116).
//
// The keyword pass is bm25_kernel (phrases included) on nidx_txt_views under the suggest mask.  When it finds nothing, the fuzzy
// pass runs one clause per query token over the same mask:
//   graph_dict_match_kernel  (nidx_suggest_expand) one pass over the paragraph vocabulary as code points: a bitset over the
//                            dictionary's term ids for every fuzzy / fuzzy-prefix literal (distance 1, transpositions cost one);
//   suggest_chunk_count_kernel + cub::DeviceScan  per (fuzzy clause, 64-term word of its expansion) the number of SG_CHUNK-posting
//                            chunks of the word's expanded terms, and their exclusive prefix sum: every chunk of every expanded term
//                            becomes one warp task, so a frequent expanded term is spread over many warps instead of one;
//   suggest_scatter_kernel   a warp per task scatters one chunk of postings into its clause's document bitset: the chunks of the
//                            expanded terms (found by binary search in the prefix sum, then a walk over the word's bits), then the
//                            chunks of each exact term and of each phrase's virtual list (phrase.cuh); posting reads are 8-byte and
//                            coalesced;
//   suggest_score_kernel     the twin of graph_eval_kernel: per document under the mask, matched = OR of the clause bits and
//                            score = 0.5 * (sum in clause order of 1.0 per matched fuzzy clause, BM25 at tf = 1 per exact term, BM25 at
//                            the phrase frequency per phrase), each in f32 with explicit roundings: a document's score depends only
//                            on its postings, never on launch or atomics order;
//   graph_topk_kernel +      the best k of (score bits << 32 | ~doc): ties go to the lower document;
//   graph_topk_merge_kernel
//   suggest_matches_kernel   for the first hits (at most SG_MAX_HITS), which expanded terms of which fuzzy clause occur in them: a
//                            binary search of each expanded term's postings per hit, appended as (hit, clause, term) to a list whose
//                            order the caller fixes by sorting.
// suggest_mask_kernel builds the suggest mask in one pass over the words: NOT repeated AND security AND op(paragraph_filter, prefilter),
// an absent operand dropped.
// HBM traffic of the fuzzy pass = 8 B per posting of every expanded and exact term and phrase (scatter), per document 1/8 B of alive
// and 1/8 B per clause bitset, 4 B of score and 1/8 B of bits (scored pass), and a binary search per (hit, expanded term).
#pragma once
#include <cstdint>

#include "graph.cuh"
#include "phrase.cuh"

namespace nidx {

constexpr int SG_MAX_CLAUSES = 64;      // clauses of one fuzzy pass (a literal, quoted group or excluded word each)
constexpr int SG_MAX_HITS = 16;         // hits whose matched terms are listed
constexpr int SG_THREADS = 256;
constexpr uint32_t SG_CHUNK = 1024;     // postings per warp task of the scatter

enum SgKind : uint32_t { SG_FUZZY = 0, SG_TERM = 1, SG_PHRASE = 2 };

struct SgClause {      // resolved on the host
    uint32_t kind;     // SgKind
    uint32_t arg;      // FUZZY: row of the expansion bitsets; TERM: term id (NIL: none in the segment); PHRASE: index of its virtual list
    float w;           // TERM: the term's weight, PHRASE: the phrase's (idf sum * (1 + k1)); FUZZY: unused
    uint32_t task0;    // TERM / PHRASE: first of the clause's tasks after the fuzzy chunks (task0 of clause n_clauses = their count);
                       // FUZZY clauses take no task here (their chunks come from fz_off)
};

struct SgArgs {
    const uint64_t* term_off;   // [n_terms + 1]
    const uint2* post;          // (doc, tf << 8 | fieldnorm id)
    const uint64_t* ph_range;   // [2 phrases] (first, end) of every phrase's compacted list in ph_post
    const uint2* ph_post;       // (doc, freq << 8 | fieldnorm id)
    const float* norm_cache;    // [256] k1 * (1 - b + b * fieldnorm / avg)
    const uint64_t* exp_bits;   // [fuzzy rows][exp_words] expanded terms over the dictionary
    size_t exp_words;
    uint32_t n_dict;            // dictionary terms (<= the segment's terms)
    const SgClause* clauses;    // [n_clauses + 1]: the last entry holds only task0
    uint32_t n_clauses;
    const uint32_t* fz_clause;  // [n_fuzzy] the clause index of each fuzzy clause, in order
    uint32_t n_fuzzy;
    const uint64_t* fz_off;     // [n_fuzzy * exp_words + 1] exclusive prefix of the chunks per (fuzzy clause, word)
    uint32_t n_docs;
    size_t words;               // (n_docs + 63) / 64
    uint64_t* bits;             // [n_clauses][words] clause bitsets (zeroed by the caller)
    const uint64_t* alive;      // the segment's (or view's) alive bits; NULL = all
    float* score;               // [n_docs]
    uint32_t* hit_bits;         // [2 words] matched documents
};

__device__ __forceinline__ uint32_t sg_clause_of(const SgClause* c, uint32_t n, uint64_t task) {
    uint32_t i = 0;
    while (i + 1 < n && c[i + 1].task0 <= task) ++i;
    return i;
}

// one clause's postings [b, e) into its bitset, a lane per posting
__device__ __forceinline__ void sg_scatter(const uint2* post, uint64_t b, uint64_t e, uint64_t* out, uint32_t lane) {
    for (uint64_t p = b + lane; p < e; p += 32) {
        const uint32_t d = __ldg(&post[p].x);
        atomicOr(reinterpret_cast<unsigned long long*>(out) + (d >> 6), 1ull << (d & 63));
    }
}

__device__ __forceinline__ uint64_t sg_chunks(const uint64_t* term_off, uint32_t t) {
    return (__ldg(term_off + t + 1) - __ldg(term_off + t) + SG_CHUNK - 1) / SG_CHUNK;
}

// cnt[i] = the chunks of the expanded terms of word i % exp_words of fuzzy clause i / exp_words (cnt[n] is left to the caller)
__global__ void suggest_chunk_count_kernel(SgArgs A, uint64_t* __restrict__ cnt) {
    const uint64_t n = (uint64_t)A.n_fuzzy * A.exp_words;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t j = i % A.exp_words;
        uint64_t word = __ldg(A.exp_bits + (size_t)A.clauses[A.fz_clause[i / A.exp_words]].arg * A.exp_words + j), c = 0;
        while (word) {
            c += sg_chunks(A.term_off, (uint32_t)(j * 64 + (__ffsll((long long)word) - 1)));
            word &= word - 1;
        }
        cnt[i] = c;
    }
}

__global__ void __launch_bounds__(SG_THREADS) suggest_scatter_kernel(SgArgs A) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_fw = (uint64_t)A.n_fuzzy * A.exp_words;
    const uint64_t n_fz = n_fw ? __ldg(A.fz_off + n_fw) : 0;
    const uint64_t n_tasks = n_fz + A.clauses[A.n_clauses].task0;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t task = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; task < n_tasks; task += n_warps) {
        if (task < n_fz) {   // a chunk of an expanded term: the word whose chunks hold it, then the term inside the word
            uint64_t lo = 0, hi = n_fw;   // the last word i with fz_off[i] <= task (it has chunks: fz_off[i + 1] > task)
            while (hi - lo > 1) {
                const uint64_t mid = (lo + hi) >> 1;
                if (__ldg(A.fz_off + mid) <= task) lo = mid; else hi = mid;
            }
            const uint64_t j = lo % A.exp_words;
            const uint32_t c = A.fz_clause[lo / A.exp_words];
            uint64_t rem = task - __ldg(A.fz_off + lo);
            uint64_t word = __ldg(A.exp_bits + (size_t)A.clauses[c].arg * A.exp_words + j);
            while (word) {
                const uint32_t t = (uint32_t)(j * 64 + (__ffsll((long long)word) - 1));
                word &= word - 1;
                const uint64_t ch = sg_chunks(A.term_off, t);
                if (rem >= ch) { rem -= ch; continue; }
                const uint64_t b = __ldg(A.term_off + t) + rem * SG_CHUNK, e = __ldg(A.term_off + t + 1);
                sg_scatter(A.post, b, b + SG_CHUNK < e ? b + SG_CHUNK : e, A.bits + (size_t)c * A.words, lane);
                break;
            }
            continue;
        }
        const uint64_t task2 = task - n_fz;   // chunk j of an exact term's or a phrase's list
        const uint32_t c = sg_clause_of(A.clauses, A.n_clauses, task2);
        const SgClause C = A.clauses[c];
        if (C.kind == SG_FUZZY) continue;   // (a fuzzy clause owns no task here)
        const uint64_t j = task2 - C.task0;
        uint64_t b, e;
        if (C.kind == SG_TERM) { b = __ldg(A.term_off + C.arg); e = __ldg(A.term_off + C.arg + 1); }
        else { b = __ldg(A.ph_range + 2 * C.arg); e = __ldg(A.ph_range + 2 * C.arg + 1); }
        b += j * SG_CHUNK;
        sg_scatter(C.kind == SG_TERM ? A.post : A.ph_post, b, b + SG_CHUNK < e ? b + SG_CHUNK : e, A.bits + (size_t)c * A.words, lane);
    }
}

__global__ void __launch_bounds__(SG_THREADS) suggest_score_kernel(SgArgs A) {
    __shared__ SgClause cl[SG_MAX_CLAUSES];
    for (uint32_t i = threadIdx.x; i < A.n_clauses; i += blockDim.x) cl[i] = A.clauses[i];
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n32 = 2 * A.words;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n32; w += n_warps) {
        const uint32_t d = (uint32_t)(w * 32 + lane);
        const uint32_t live = A.alive ? (uint32_t)(__ldg(A.alive + (w >> 1)) >> (32 * (w & 1))) : 0xFFFFFFFFu;
        uint32_t bit = 0;
        float s = 0.f;
        if (d < A.n_docs && ((live >> lane) & 1u)) {
            for (uint32_t c = 0; c < A.n_clauses; ++c) {
                const uint32_t cw = (uint32_t)(__ldg(A.bits + (size_t)c * A.words + (w >> 1)) >> (32 * (w & 1)));   // one word per warp
                if (!((cw >> lane) & 1u)) continue;
                bit = 1;
                const SgClause& C = cl[c];
                float v = 1.0f;
                if (C.kind != SG_FUZZY) {
                    uint64_t b, e;
                    const uint2* post = C.kind == SG_TERM ? A.post : A.ph_post;
                    if (C.kind == SG_TERM) { b = __ldg(A.term_off + C.arg); e = __ldg(A.term_off + C.arg + 1); }
                    else { b = __ldg(A.ph_range + 2 * C.arg); e = __ldg(A.ph_range + 2 * C.arg + 1); }
                    const uint2 p = __ldg(post + post_lower_bound(post, b, e, d));   // the bit says the posting is there
                    const float nc = __ldg(A.norm_cache + (p.y & 0xFFu));
                    if (C.kind == SG_TERM) {
                        v = __fmul_rn(C.w, __fdiv_rn(1.0f, __fadd_rn(1.0f, nc)));           // Basic: tf = 1
                    } else {
                        const float f = (float)(p.y >> 8);
                        v = __fmul_rn(C.w, __fdiv_rn(f, __fadd_rn(f, nc)));
                    }
                }
                s = __fadd_rn(s, v);
            }
            s = __fmul_rn(0.5f, s);   // BoostQuery(.., 0.5)
        }
        const uint32_t word = __ballot_sync(0xFFFFFFFFu, bit);
        if (d < A.n_docs) A.score[d] = bit ? s : 0.f;
        if (lane == 0) A.hit_bits[w] = word;
    }
}

// Per (fuzzy clause, dictionary word) warp task: for every expanded term of the word, lane h < n_hits looks hit h's document up in the
// term's postings; a find appends (h << 40 | clause << 32 | term) to out (the first cap entries are kept, *n_out counts them all).
__global__ void __launch_bounds__(SG_THREADS) suggest_matches_kernel(SgArgs A, const uint32_t* __restrict__ ids, const int* __restrict__ count,
                                                                     int max_hits, uint64_t* __restrict__ out, uint32_t cap, uint32_t* __restrict__ n_out) {
    const uint32_t lane = threadIdx.x & 31;
    const int nh = min(*count, max_hits);
    const uint32_t doc = lane < (uint32_t)nh ? ids[lane] : 0u;
    uint64_t n_tasks = 0;
    for (uint32_t c = 0; c < A.n_clauses; ++c)
        if (A.clauses[c].kind == SG_FUZZY) n_tasks += A.exp_words;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t task = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; task < n_tasks; task += n_warps) {
        uint32_t c = 0;
        uint64_t j = task;
        for (;; ++c) {   // the (j / exp_words)-th fuzzy clause
            if (A.clauses[c].kind != SG_FUZZY) continue;
            if (j < A.exp_words) break;
            j -= A.exp_words;
        }
        uint64_t word = __ldg(A.exp_bits + (size_t)A.clauses[c].arg * A.exp_words + j);
        while (word) {
            const uint32_t t = (uint32_t)(j * 64 + (__ffsll((long long)word) - 1));
            word &= word - 1;
            if (lane >= (uint32_t)nh) continue;
            const uint64_t b = __ldg(A.term_off + t), e = __ldg(A.term_off + t + 1);
            const uint64_t p = post_lower_bound(A.post, b, e, doc);
            if (p < e && __ldg(&A.post[p].x) == doc) {
                const uint32_t at = atomicAdd(n_out, 1u);
                if (at < cap) out[at] = ((uint64_t)lane << 40) | ((uint64_t)c << 32) | t;
            }
        }
    }
}

// The expanded terms of every automaton term: counts[row] = set bits of its bitset.
__global__ void suggest_popc_kernel(const uint64_t* __restrict__ bits, size_t words, uint32_t rows, unsigned long long* __restrict__ counts) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < (uint64_t)rows * words; i += (uint64_t)gridDim.x * blockDim.x) {
        const int n = __popcll(__ldg(bits + i));
        if (n) atomicAdd(counts + i / words, (unsigned long long)n);
    }
}

// mask = NOT repeated AND sec AND op(pf, joined); a NULL operand is dropped (repeated NULL: none is repeated), padding bits zero.
__global__ void suggest_mask_kernel(uint32_t n_docs, const uint64_t* __restrict__ repeated, const uint64_t* __restrict__ sec, const uint64_t* __restrict__ pf,
                                    const uint64_t* __restrict__ joined, int op_or, uint64_t* __restrict__ out, unsigned long long* count) {
    const size_t words = ((size_t)n_docs + 63) / 64;
    unsigned long long local = 0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < words; i += (size_t)gridDim.x * blockDim.x) {
        uint64_t m = repeated ? ~__ldg(repeated + i) : ~0ull;
        if (sec) m &= __ldg(sec + i);
        if (pf && joined) m &= op_or ? (__ldg(pf + i) | __ldg(joined + i)) : (__ldg(pf + i) & __ldg(joined + i));
        else if (pf) m &= __ldg(pf + i);
        else if (joined) m &= __ldg(joined + i);
        if (i == words - 1 && (n_docs & 63)) m &= (1ull << (n_docs & 63)) - 1;
        out[i] = m;
        local += __popcll(m);
    }
    if (count && local) atomicAdd(count, local);
}

}  // namespace nidx
