// nidx_b200 — boolean filters on the device (sm_90a): one evaluator, two front ends.
//
// A filter is a program: its leaves and binary AND / OR in post-order, NOT flipping the top of the bit stack (PfOp).  Two front ends
// compile into it (api.cu):
//   the prefilter      nidx_txt_prefilter, an expression over a text segment's documents (nidx_text/src/reader.rs:147-180:
//                      filter_to_query over every document, the FieldUuidCollector); its leaves read the document columns or, for
//                      keywords, a bitset slot;
//   paragraph formulas nidx_vec_filter / nidx_vec_search_formula / nidx_vec_prefilter_bits, a formula over a vector segment's
//                      paragraphs (inverted_index/paragraph.rs:124-186); its leaves are bitset slots set from the label and field
//                      postings, looked up on the host.
// One run: the slots are zeroed, set by the scatter kernels, and the program is evaluated over the documents, ANDed with the alive
// set and counted.
//   prefilter_scatter_kernel  before the pass: one CTA per posting range (a term's list, a phrase's virtual list from phrase.cuh,
//                             or a paragraph leaf's range) sets its documents in the range's slot;
//   prefilter_eval_kernel     one pass over the documents: a warp covers 32 consecutive documents, every lane runs the program (in
//                             shared memory) for its own document on a bit stack held in a register; the warp's ballot is one 32-bit
//                             word of the result, ANDed with the alive bits, and counted;
//   prefilter_join_kernel     text documents -> paragraphs of one vector segment: every matched document with a join entry sets the
//                             paragraphs of that field key (the NIDX_INV_FIELDS postings).
// HBM traffic of the pass = per document the columns the program reads (4 B per ord column, 8 B per date column, the facet or
// access group CSR entry and ords) + 1/8 B of alive bits + 1/8 B per bitset leaf + 1/8 B of output.
#pragma once
#include <cstdint>

#include "bm25.cuh"

namespace nidx {

constexpr int PF_MAX_DEPTH = 64;        // the bit stack is one 64-bit register: NIDX_PREFILTER_MAX_DEPTH
constexpr int PF_MAX_PROGRAM = 4096;    // instructions (32 B each) in shared memory
constexpr int PF_THREADS = 256;

enum PfOpcode : uint32_t { PF_FACET, PF_FIELD, PF_RESOURCE, PF_DATE, PF_BITS, PF_CONST, PF_AND, PF_OR, PF_NOT, PF_PUBLIC };

struct PfOp {          // one instruction: leaves push a bit, AND / OR pop two and push one, NOT flips the top
    int64_t lo, hi;    // FACET / FIELD / RESOURCE: ord range [lo, hi); DATE: since, until (inclusive)
    uint32_t op;       // PfOpcode
    uint32_t arg;      // FACET / PUBLIC: the CSR column (0 facets, 1 access groups); DATE: the seconds column (0 created, 1 modified);
                       // BITS: the keyword leaf's slot; CONST: the bit
    float w;           // graph.cuh's scored leaves and CONST_SCORE: the score (unread here)
    uint32_t pad;
};

struct PrefilterArgs {
    uint32_t n_docs;
    const uint32_t* res_ord;     // [n_docs] (nidx_txt_set_doc_columns)
    const uint32_t* field_ord;   // [n_docs]
    const uint32_t* fdoc_off;    // [n_docs + 1] facet CSR (nidx_txt_set_facets)
    const uint32_t* ford;
    const uint32_t* gdoc_off;    // [n_docs + 1] access group CSR (nidx_txt_set_doc_groups)
    const uint32_t* gord;
    const int64_t* secs0;        // [n_docs] created, modified seconds (nidx_txt_set_dates); INT64_MIN = no date
    const int64_t* secs1;
    const uint64_t* kw_bits;     // [slots][words] keyword leaves
    size_t words;                // (n_docs + 63) / 64
    const uint64_t* alive;       // NULL = all alive
    const PfOp* prog;
    uint32_t n_prog;
    uint32_t* out;               // [2 * words]: the result as 32-bit words, padding bits zero
    unsigned long long* count;   // += set bits of out
};

__global__ void __launch_bounds__(PF_THREADS) prefilter_eval_kernel(PrefilterArgs A) {
    extern __shared__ PfOp prog[];
    for (uint32_t i = threadIdx.x; i < A.n_prog; i += blockDim.x) prog[i] = A.prog[i];
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n32 = 2 * (uint64_t)A.words;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    unsigned long long local = 0;
    // w is the same for the 32 lanes of a warp: the ballot always has the full warp
    for (uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n32; w += n_warps) {
        const uint64_t d = w * 32 + lane;
        uint32_t bit = 0;
        if (d < A.n_docs) {
            uint64_t st = 0;
            for (uint32_t i = 0; i < A.n_prog; ++i) {
                const PfOp& o = prog[i];
                uint64_t b;
                switch (o.op) {
                    case PF_FACET: {   // ords ascend: the first one >= lo decides
                        const uint32_t* off = o.arg ? A.gdoc_off : A.fdoc_off;
                        const uint32_t* ords = o.arg ? A.gord : A.ford;
                        b = 0;
                        for (uint32_t j = __ldg(off + d), e = __ldg(off + d + 1); j < e; ++j) {
                            const int64_t u = __ldg(ords + j);
                            if (u >= o.lo) { b = u < o.hi; break; }
                        }
                        break;
                    }
                    case PF_PUBLIC: { const uint32_t* off = o.arg ? A.gdoc_off : A.fdoc_off; b = __ldg(off + d) == __ldg(off + d + 1); break; }
                    case PF_FIELD: { const int64_t u = __ldg(A.field_ord + d); b = u >= o.lo && u < o.hi; break; }
                    case PF_RESOURCE: { const int64_t u = __ldg(A.res_ord + d); b = u >= o.lo && u < o.hi; break; }
                    case PF_DATE: {
                        const int64_t s = __ldg((o.arg ? A.secs1 : A.secs0) + d);
                        b = s != INT64_MIN && s >= o.lo && s <= o.hi;
                        break;
                    }
                    case PF_BITS: b = (__ldg(A.kw_bits + (size_t)o.arg * A.words + (d >> 6)) >> (d & 63)) & 1ull; break;
                    case PF_CONST: b = o.arg; break;
                    case PF_AND: b = st & (st >> 1) & 1ull; st >>= 2; break;
                    case PF_OR: b = (st | (st >> 1)) & 1ull; st >>= 2; break;
                    default: st ^= 1ull; continue;   // PF_NOT
                }
                st = (st << 1) | b;
            }
            bit = (uint32_t)(st & 1ull);
        }
        uint32_t word = __ballot_sync(0xFFFFFFFFu, bit);
        if (A.alive) word &= __ldg(reinterpret_cast<const uint32_t*>(A.alive) + w);
        if (lane == 0) { A.out[w] = word; local += __popc(word); }
    }
    if (lane == 0 && local) atomicAdd(A.count, local);
}

__device__ __forceinline__ uint32_t pf_doc(const uint2* p) { return __ldg(&p->x); }   // a text posting: (doc, tf)
__device__ __forceinline__ uint32_t pf_doc(const uint32_t* p) { return __ldg(p); }   // a paragraph posting

// One CTA per posting range, which sets slot (slot ? slot[blockIdx.x] : slot0 + blockIdx.x): terms != NULL -> the posting list of
// terms[blockIdx.x] in `post` (none when the id is not a term of the segment), else the range ranges[2 blockIdx.x .. +1] of `post`
// for the first n_post ranges and of `post1` for the rest.
template <typename Post>
__global__ void prefilter_scatter_kernel(const Post* __restrict__ post, const Post* __restrict__ post1, uint32_t n_post,
                                         const uint64_t* __restrict__ term_off, uint32_t n_terms, const uint32_t* __restrict__ terms,
                                         const uint64_t* __restrict__ ranges, const uint32_t* __restrict__ slot, uint32_t slot0,
                                         uint64_t* __restrict__ bits, size_t words) {
    uint64_t b, e;
    if (terms) {
        const uint32_t t = terms[blockIdx.x];
        if (t >= n_terms) return;
        b = term_off[t]; e = term_off[t + 1];
    } else {
        b = ranges[2 * blockIdx.x]; e = ranges[2 * blockIdx.x + 1];
    }
    if (blockIdx.x >= n_post) post = post1;
    const uint32_t sl = slot ? slot[blockIdx.x] : slot0 + blockIdx.x;
    unsigned long long* out = reinterpret_cast<unsigned long long*>(bits + (size_t)sl * words);
    for (uint64_t i = b + threadIdx.x; i < e; i += blockDim.x) {
        const uint32_t doc = pf_doc(post + i);
        atomicOr(out + (doc >> 6), 1ull << (doc & 63));
    }
}

// doc_bits [n_docs] -> out (paragraph bits, zeroed by the caller): join[d] = the document's key in the field index (NIL or >= n_keys:
// none), whose paragraphs are post[post_off[key] .. post_off[key + 1]).
__global__ void prefilter_join_kernel(const uint64_t* __restrict__ doc_bits, const uint32_t* __restrict__ join, uint64_t n_docs, uint32_t n_keys,
                                      const uint64_t* __restrict__ post_off, const uint32_t* __restrict__ post, uint64_t* __restrict__ out) {
    for (uint64_t d = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; d < n_docs; d += (uint64_t)gridDim.x * blockDim.x) {
        if (!((__ldg(doc_bits + (d >> 6)) >> (d & 63)) & 1ull)) continue;
        const uint32_t j = __ldg(join + d);
        if (j >= n_keys) continue;
        for (uint64_t i = __ldg(post_off + j), e = __ldg(post_off + j + 1); i < e; ++i) {
            const uint32_t p = __ldg(post + i);
            atomicOr(reinterpret_cast<unsigned long long*>(out) + (p >> 6), 1ull << (p & 63));
        }
    }
}

// JSON filters (nidx_txt_resource_bits, nidx_vec_prefilter_bits' resource part, nidx_txt_join_mask): a JSON document's result is a resource.
// doc_bits [n_docs] -> out (resource bits, zeroed by the caller): res_ord[d] = the document's resource ord (>= n_res: none).
__global__ void prefilter_resource_kernel(const uint64_t* __restrict__ doc_bits, const uint32_t* __restrict__ res_ord, uint64_t n_docs, uint64_t n_res,
                                          uint64_t* __restrict__ out) {
    for (uint64_t d = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; d < n_docs; d += (uint64_t)gridDim.x * blockDim.x) {
        if (!((__ldg(doc_bits + (d >> 6)) >> (d & 63)) & 1ull)) continue;
        const uint64_t r = __ldg(res_ord + d);
        if (r < n_res) atomicOr(reinterpret_cast<unsigned long long*>(out) + (r >> 6), 1ull << (r & 63));
    }
}

// res_bits [n_res] -> out (paragraph bits, zeroed by the caller): resource r's paragraphs are post[ranges[2 r] .. ranges[2 r + 1]) (the
// postings of the field index keys that start with its 16 uuid bytes: one contiguous run of keys).
__global__ void prefilter_res_join_kernel(const uint64_t* __restrict__ res_bits, uint64_t n_res, const uint64_t* __restrict__ ranges,
                                          const uint32_t* __restrict__ post, uint64_t* __restrict__ out) {
    for (uint64_t r = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; r < n_res; r += (uint64_t)gridDim.x * blockDim.x) {
        if (!((__ldg(res_bits + (r >> 6)) >> (r & 63)) & 1ull)) continue;
        for (uint64_t i = __ldg(ranges + 2 * r), e = __ldg(ranges + 2 * r + 1); i < e; ++i) {
            const uint32_t p = __ldg(post + i);
            atomicOr(reinterpret_cast<unsigned long long*>(out) + (p >> 6), 1ull << (p & 63));
        }
    }
}

// One mask over n documents: bit d = and_bits[d] (NULL: 1) AND op(doc_bits[doc_join[d]] (doc_bits NULL: 1), res_bits[res_join[d]]),
// a join entry of NIDX_NIL (or >= the bitset's length) reading 0; op: 0 AND, 1 OR.  out: [2 * words] 32-bit words, padding bits zero;
// *count += set bits.  A warp writes one 32-bit word by ballot, as prefilter_eval_kernel does.
__global__ void __launch_bounds__(PF_THREADS) join_mask_kernel(uint64_t n, const uint64_t* __restrict__ and_bits, const uint64_t* __restrict__ doc_bits,
                                                               uint64_t n_doc_bits, const uint32_t* __restrict__ doc_join,
                                                               const uint64_t* __restrict__ res_bits, uint64_t n_res, const uint32_t* __restrict__ res_join,
                                                               int op, uint32_t* __restrict__ out, uint64_t n32, unsigned long long* count) {
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    unsigned long long local = 0;
    for (uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n32; w += n_warps) {
        const uint64_t d = w * 32 + lane;
        uint32_t bit = 0;
        if (d < n) {
            uint32_t t = 1;
            if (doc_bits) {
                const uint64_t j = __ldg(doc_join + d);
                t = j < n_doc_bits ? (uint32_t)((__ldg(doc_bits + (j >> 6)) >> (j & 63)) & 1ull) : 0u;
            }
            const uint64_t r = __ldg(res_join + d);
            const uint32_t j = r < n_res ? (uint32_t)((__ldg(res_bits + (r >> 6)) >> (r & 63)) & 1ull) : 0u;
            bit = op ? (t | j) : (t & j);
            if (and_bits) bit &= (uint32_t)((__ldg(and_bits + (d >> 6)) >> (d & 63)) & 1ull);
        }
        const uint32_t word = __ballot_sync(0xFFFFFFFFu, bit);
        if (lane == 0) { out[w] = word; local += __popc(word); }
    }
    if (lane == 0 && local) atomicAdd(count, local);
}

}  // namespace nidx
