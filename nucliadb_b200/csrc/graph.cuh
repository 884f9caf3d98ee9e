// nidx_b200 — graph search on the device (sm_90a): NidxSearcher.GraphSearch over the relation index (reference: nidx_relation).
//
// The relation documents are a text segment without terms (facets, resource / field ords, alive bits); the graph columns live
// beside it (nidx_graph_set_columns).  One search is:
//   graph_dict_match_kernel  one pass over a dictionary in HBM (normalised values or default tokens, as code points): for every
//                            automaton term of the query (fuzzy and / or prefix, distance <= 2) a bitset over the dictionary's ords,
//                            by a banded restricted Damerau-Levenshtein DP per entry;
//   graph_eval_kernel        the scored twin of prefilter_eval_kernel: the same PfOp post-order program and limits, a bit stack in a
//                            register and an f32 score per level in shared memory -> per document its score and its matched bit;
//   graph_unique_kernel      NODES / RELATIONS: the max score of every key ord (atomicMax on the score's bits, scores are >= 0);
//   graph_topk_kernel +      the best k keys (score << 32 | ~id): documents for PATH (ties: lower document first), key ords for
//   graph_topk_merge_kernel  NODES / RELATIONS (ties: lower key ord first), as topk.cuh's per-CTA top-k and one merge.
// The score of every node keeps the invariant "0 when the bit is 0", so OR adds both operands, AND adds both when both match and
// NOT drops the operand's score.
// HBM traffic of the scored pass = per document 4 B per ord column the program reads, the token CSR entry and its ords per token
// leaf, the facet CSR entry and ords per facet leaf, 1/8 B per automaton bitset read, 1/8 B of alive, 4 B of score and 1/8 B of bits.
#pragma once
#include <cstdint>

#include "prefilter.cuh"
#include "topk.cuh"

namespace nidx {

constexpr int GF_MAX_DIST = 2;         // d <= 2 (FuzzyTermQuery's limit)
constexpr int GF_MAX_TERMS = 64;       // automaton terms of one search
constexpr int GF_MAX_TERM_CPS = 4096;  // code points of all automaton terms together (shared memory)
constexpr int GF_COLS = 11;            // per-document ord columns (NIDX_G_* of the header, same order)
constexpr int GF_THREADS = 256;

// Graph leaves share PfOp's layout: lo / hi as below, arg the column, w the leaf's score.
enum GfOpcode : uint32_t {
    GF_EQ = 100,    // column arg == lo
    GF_COLBITS,     // column arg's ord is set in automaton bitset lo (over the values dictionary)
    GF_TOKBITS,     // some token of side arg (0 source, 1 target) is set in automaton bitset lo (over the token dictionary)
    GF_TOKSET,      // some token of side arg is one of ords[lo .. hi) (ascending)
    GF_FACET,       // a facet ord in [lo, hi)
    GF_CONST,       // bit arg
    GF_AND, GF_OR, GF_NOT,
    GF_CONST_SCORE  // the top's score becomes w where its bit is set
};

struct RelGraphDev {   // the relation index (not an HNSW graph: common.cuh's GraphDev)
    uint32_t n_docs;
    const uint32_t* col[GF_COLS];    // [n_docs] each
    const uint32_t* tok_off[2];      // [n_docs + 1] source / target token CSR
    const uint32_t* tok[2];
    const uint32_t* fdoc_off;        // facet CSR of the segment
    const uint32_t* ford;
};

struct GraphEvalArgs {
    RelGraphDev G;
    const uint64_t* alive;           // NULL = all
    const uint64_t* mask;            // NULL = all
    const uint64_t* val_bits;        // [terms][val_words] automaton bitsets over the values dictionary
    const uint64_t* tok_bits;        // [terms][tok_words] over the token dictionary
    size_t val_words, tok_words;
    const uint32_t* ords;            // TOKSET lists
    const PfOp* prog;
    uint32_t n_prog, depth;          // depth: the most levels the program's stack holds
    float* score;                    // [n_docs]
    uint32_t* bits;                  // [2 * words]
};

__device__ __forceinline__ uint32_t gf_bit(const uint64_t* b, uint64_t i) { return (uint32_t)((__ldg(b + (i >> 6)) >> (i & 63)) & 1ull); }

__global__ void __launch_bounds__(GF_THREADS) graph_eval_kernel(GraphEvalArgs A) {
    extern __shared__ __align__(16) unsigned char gf_smem[];
    PfOp* prog = reinterpret_cast<PfOp*>(gf_smem);
    float* sc = reinterpret_cast<float*>(gf_smem + (size_t)A.n_prog * sizeof(PfOp));   // [depth][blockDim.x]
    for (uint32_t i = threadIdx.x; i < A.n_prog; i += blockDim.x) prog[i] = A.prog[i];
    __syncthreads();
    const uint32_t lane = threadIdx.x & 31;
    const uint64_t words = ((uint64_t)A.G.n_docs + 63) / 64, n32 = 2 * words;
    const uint64_t n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t w = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n32; w += n_warps) {
        const uint64_t d = w * 32 + lane;
        uint32_t bit = 0;
        float s = 0.f;
        if (d < A.G.n_docs && (!A.alive || gf_bit(A.alive, d)) && (!A.mask || gf_bit(A.mask, d))) {
            uint64_t st = 0;
            uint32_t top = 0;   // levels in use
            for (uint32_t i = 0; i < A.n_prog; ++i) {
                const PfOp& o = prog[i];
                uint64_t b;
                switch (o.op) {
                    case GF_EQ: b = __ldg(A.G.col[o.arg] + d) == (uint64_t)o.lo; break;
                    case GF_COLBITS: b = gf_bit(A.val_bits + (size_t)o.lo * A.val_words, __ldg(A.G.col[o.arg] + d)); break;
                    case GF_TOKBITS: case GF_TOKSET: {
                        b = 0;
                        for (uint32_t j = __ldg(A.G.tok_off[o.arg] + d), e = __ldg(A.G.tok_off[o.arg] + d + 1); j < e && !b; ++j) {
                            const uint32_t t = __ldg(A.G.tok[o.arg] + j);
                            if (o.op == GF_TOKBITS) {
                                b = gf_bit(A.tok_bits + (size_t)o.lo * A.tok_words, t);
                            } else {
                                for (int64_t k = o.lo; k < o.hi; ++k)
                                    if (__ldg(A.ords + k) == t) { b = 1; break; }
                            }
                        }
                        break;
                    }
                    case GF_FACET: {   // ords ascend: the first one >= lo decides
                        b = 0;
                        for (uint32_t j = __ldg(A.G.fdoc_off + d), e = __ldg(A.G.fdoc_off + d + 1); j < e; ++j) {
                            const int64_t u = __ldg(A.G.ford + j);
                            if (u >= o.lo) { b = u < o.hi; break; }
                        }
                        break;
                    }
                    case GF_CONST: b = o.arg; break;
                    case GF_AND: {
                        const float a = sc[(top - 2) * blockDim.x + threadIdx.x], c = sc[(top - 1) * blockDim.x + threadIdx.x];
                        b = st & (st >> 1) & 1ull;
                        st >>= 2; top -= 2;
                        sc[top * blockDim.x + threadIdx.x] = b ? a + c : 0.f;
                        st = (st << 1) | b; ++top;
                        continue;
                    }
                    case GF_OR: {
                        const float a = sc[(top - 2) * blockDim.x + threadIdx.x], c = sc[(top - 1) * blockDim.x + threadIdx.x];
                        b = (st | (st >> 1)) & 1ull;
                        st >>= 2; top -= 2;
                        sc[top * blockDim.x + threadIdx.x] = a + c;   // an unmatched operand's score is 0
                        st = (st << 1) | b; ++top;
                        continue;
                    }
                    case GF_NOT: st ^= 1ull; sc[(top - 1) * blockDim.x + threadIdx.x] = 0.f; continue;
                    default:   // GF_CONST_SCORE
                        sc[(top - 1) * blockDim.x + threadIdx.x] = (st & 1ull) ? o.w : 0.f;
                        continue;
                }
                st = (st << 1) | b;
                sc[top * blockDim.x + threadIdx.x] = b ? o.w : 0.f;
                ++top;
            }
            bit = (uint32_t)(st & 1ull);
            s = sc[threadIdx.x];
        }
        const uint32_t word = __ballot_sync(0xFFFFFFFFu, bit);
        if (d < A.G.n_docs) A.score[d] = bit ? s : 0.f;
        if (lane == 0) A.bits[w] = word;
    }
}

// Restricted Damerau-Levenshtein (optimal string alignment) between the query q [m] and a dictionary entry s [n], in a band of
// |i - j| <= GF_MAX_DIST cells, values capped at GF_MAX_DIST + 1.  Returns whether dist(q, s) <= d (prefix: dist(q, s[0..j]) <= d for
// some j).  Row j (entry position) cell k stands for query position i = j - GF_MAX_DIST + k.
__device__ bool gf_within(const uint32_t* q, int m, const uint32_t* s, int n, int d, bool prefix) {
    constexpr int W = 2 * GF_MAX_DIST + 1, INF = GF_MAX_DIST + 1;
    int p2[W], p1[W], cur[W];
#pragma unroll
    for (int k = 0; k < W; ++k) {
        const int i = k - GF_MAX_DIST;
        p2[k] = INF;
        p1[k] = (i >= 0 && i <= m) ? min(i, INF) : INF;
    }
    if (prefix && m <= d) return true;   // j = 0: the empty prefix
    uint32_t sj1 = 0;              // s[j - 2]
    const int last = prefix ? min(n, m + d) : n;
    for (int j = 1; j <= last; ++j) {
        const uint32_t sj = __ldg(s + j - 1);
        int row_min = INF;
#pragma unroll
        for (int k = 0; k < W; ++k) {
            const int i = j - GF_MAX_DIST + k;
            int v = INF;
            if (i == 0) {
                v = min(j, INF);
            } else if (i > 0 && i <= m) {
                const uint32_t qi = q[i - 1];
                v = p1[k] + (qi != sj);                       // D[i-1][j-1]
                if (k + 1 < W) v = min(v, p1[k + 1] + 1);      // D[i][j-1]
                if (k > 0) v = min(v, cur[k - 1] + 1);         // D[i-1][j]
                if (i > 1 && j > 1 && qi == sj1 && q[i - 2] == sj) v = min(v, p2[k] + 1);   // a transposition
                v = min(v, INF);
            }
            cur[k] = v;
            row_min = min(row_min, v);
        }
        const int km = m - j + GF_MAX_DIST;   // the cell of i = m
        if (prefix && km >= 0 && km < W && cur[km] <= d) return true;
        if (!prefix && j == n) return km >= 0 && km < W && cur[km] <= d;
        if (row_min > d) {
            // every later cell grows from this row or the previous one: once both exceed d nothing can match
            int prev_min = INF;
#pragma unroll
            for (int k = 0; k < W; ++k) prev_min = min(prev_min, p1[k]);
            if (prev_min > d) return false;
        }
#pragma unroll
        for (int k = 0; k < W; ++k) { p2[k] = p1[k]; p1[k] = cur[k]; }
        sj1 = sj;
    }
    return !prefix && n == 0 && m <= d;
}

struct GraphTerm {     // one automaton term in shared memory
    uint32_t off, len; // code points q[off .. off + len) of the term array
    uint32_t dist, prefix;
};

// One pass over a dictionary of n entries (code points cp[off[e] .. off[e + 1])): for every term t, bit e of out[t] (words per
// term, zeroed by the caller) when the entry matches.  A thread takes one entry and every term; entries longer than the term plus
// d (not prefix) or shorter than the term less d are skipped without DP.
__global__ void __launch_bounds__(GF_THREADS) graph_dict_match_kernel(const uint32_t* __restrict__ cp, const uint64_t* __restrict__ off, uint32_t n,
                                                                      const GraphTerm* __restrict__ terms, uint32_t n_terms, const uint32_t* __restrict__ term_cp,
                                                                      uint32_t n_term_cp, uint64_t* __restrict__ out, size_t words) {
    __shared__ GraphTerm t_sh[GF_MAX_TERMS];
    extern __shared__ uint32_t q_sh[];
    for (uint32_t i = threadIdx.x; i < n_terms; i += blockDim.x) t_sh[i] = terms[i];
    for (uint32_t i = threadIdx.x; i < n_term_cp; i += blockDim.x) q_sh[i] = term_cp[i];
    __syncthreads();
    for (uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; e < n; e += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t b = __ldg(off + e);
        const int len = (int)(__ldg(off + e + 1) - b);
        for (uint32_t t = 0; t < n_terms; ++t) {
            const GraphTerm T = t_sh[t];
            const int m = (int)T.len, d = (int)T.dist;
            if (len + d < m || (!T.prefix && len > m + d)) continue;
            if (gf_within(q_sh + T.off, m, cp + b, len, d, T.prefix != 0))
                atomicOr(reinterpret_cast<unsigned long long*>(out + t * words) + (e >> 6), 1ull << (e & 63));
        }
    }
}

// NODES / RELATIONS: kmax[key[d]] = max(kmax, score bits + 1) over the matched documents (0 = the key was not matched).
__global__ void graph_unique_kernel(uint32_t n_docs, const uint32_t* __restrict__ bits, const float* __restrict__ score,
                                    const uint32_t* __restrict__ key, uint32_t* __restrict__ kmax) {
    for (uint64_t d = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; d < n_docs; d += (uint64_t)gridDim.x * blockDim.x) {
        if (!((__ldg(bits + (d >> 5)) >> (d & 31)) & 1u)) continue;
        atomicMax(kmax + __ldg(key + d), __float_as_uint(__ldg(score + d)) + 1u);
    }
}

// Per CTA the best k of its grid-stride slice of n items, as keys (score bits << 32 | ~id) into partial[blockIdx.x][k] (0 padded).
// PATH (kmax NULL): item = document, present when its bit is set; else item = key ord, present when kmax != 0.
__global__ void __launch_bounds__(GF_THREADS) graph_topk_kernel(uint32_t n, const uint32_t* __restrict__ bits, const float* __restrict__ score,
                                                                const uint32_t* __restrict__ kmax, int k, int cap, uint64_t* __restrict__ partial) {
    extern __shared__ __align__(16) uint64_t gk_buf[];
    __shared__ int gk_count;
    __shared__ uint64_t gk_thr;
    BlockTopK tk;
    tk.init(gk_buf, &gk_count, &gk_thr, k, cap);
    const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
    const uint64_t rounds = (n + stride - 1) / stride;
    for (uint64_t r = 0; r < rounds; ++r) {
        const uint64_t i = r * stride + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
        uint64_t key = 0;
        if (i < n) {
            if (kmax) {
                const uint32_t v = __ldg(kmax + i);
                if (v) key = ((uint64_t)(v - 1u) << 32) | (uint32_t)~(uint32_t)i;
            } else if ((__ldg(bits + (i >> 5)) >> (i & 31)) & 1u) {
                key = ((uint64_t)__float_as_uint(__ldg(score + i)) << 32) | (uint32_t)~(uint32_t)i;
            }
        }
        tk.offer(key);
    }
    const int c = tk.finish();
    for (int j = threadIdx.x; j < k; j += blockDim.x) partial[(size_t)blockIdx.x * k + j] = j < c ? gk_buf[j] : 0;
}

__global__ void __launch_bounds__(GF_THREADS) graph_topk_merge_kernel(const uint64_t* __restrict__ keys_in, int n_in, int k, int cap,
                                                                      uint32_t* __restrict__ out_ids, float* __restrict__ out_scores, int* __restrict__ out_count) {
    extern __shared__ __align__(16) uint64_t gk_buf[];
    __shared__ int gk_count;
    __shared__ uint64_t gk_thr;
    BlockTopK tk;
    tk.init(gk_buf, &gk_count, &gk_thr, k, cap);
    for (int base = 0; base < n_in; base += blockDim.x) {
        const int i = base + threadIdx.x;
        tk.offer(i < n_in ? keys_in[i] : 0);
    }
    const int c = tk.finish();
    for (int j = threadIdx.x; j < k; j += blockDim.x) {
        const uint64_t key = j < c ? gk_buf[j] : 0;
        out_ids[j] = key ? ~(uint32_t)key : 0xFFFFFFFFu;
        out_scores[j] = key ? __uint_as_float((uint32_t)(key >> 32)) : 0.f;
    }
    if (threadIdx.x == 0) *out_count = c;
}

}  // namespace nidx
