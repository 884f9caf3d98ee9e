// nidx_b200 — exact phrases of the keyword search as virtual posting lists (sm_90a).
//
// Replaces tantivy's PhraseQuery scorer (slop 0) in the keyword query of nidx_paragraph (keyword_parser.rs:27-91) [recalled]:
//   freq(doc) = | intersection over i of { p - i : p in pos(t_i, doc) } |,   a match when freq >= 1,
// scored by bm25_body with freq in the place of tf and the phrase's weight (idf summed over its terms, times 1 + k1).
//
// Positions (nidx_txt_set_positions): for every posting, in posting order, its tf ascending token positions; pos_off[i] = the first
// of posting i's, the exclusive prefix sum of the exact tf (posting n_post holds the total).
// A query's phrases become virtual posting lists in the `post` record format, (doc, freq << 8 | fieldnorm id) ascending by doc:
//   phrase_match_kernel    one thread per posting of the phrase's rarest term (the driver): every other term's posting of the
//                          same document is found through its skip row (else a binary search of its whole list), then the
//                          driver's start positions (32 at a time, a bit each) are merged with each term's positions; the result
//                          lands in the slot of the driver posting, freq 0 where nothing matched;
//   phrase_compact_kernel  one CTA per phrase drops the freq-0 slots in place, keeping doc order, and writes the list's range;
//   bm25_build_skip_kernel a skip row for every phrase whose driver has at least BM_SKIP_DF postings.
// HBM traffic = the driver's postings and positions once + per (driver posting, other term) the probe's postings and positions.
#pragma once
#include <cub/block/block_scan.cuh>

#include "bm25.cuh"

namespace nidx {

constexpr int PHRASE_MAX_TERMS = 64;

struct PhraseArgs {
    const uint64_t* pos_off;   // [n_post + 1]
    const uint32_t* pos;       // [pos_off[n_post]]
    const uint32_t* terms;     // the phrases' term ids, concatenated (every id < n_terms)
    const uint32_t* off;       // [nv + 1]
    const uint32_t* driver;    // [nv] index in the phrase of its rarest term
    const uint64_t* cap_off;   // [nv + 1] first slot of every phrase's list in out: exclusive prefix of the drivers' df
    uint32_t nv;
    uint2* out;                // [cap_off[nv]]
    uint64_t* range;           // [2 nv] (first, end) slot of every compacted list
};

// index-time: tf of every posting (the exact one: a clamped tf is flagged) -> pos_off before its exclusive scan
__global__ void pos_tf_kernel(const uint2* __restrict__ post, uint64_t n_post, uint64_t* __restrict__ tf, unsigned int* __restrict__ clamped) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= n_post; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t t = i < n_post ? post[i].y >> 8 : 0u;
        if (t >= 0xFFFFFFu) atomicOr(clamped, 1u);
        tf[i] = t;
    }
}

// index-time: every posting's positions strictly ascending
__global__ void pos_check_kernel(const uint64_t* __restrict__ pos_off, const uint32_t* __restrict__ pos, uint64_t n_post, unsigned int* __restrict__ bad) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_post; i += (uint64_t)gridDim.x * blockDim.x)
        for (uint64_t j = pos_off[i] + 1; j < pos_off[i + 1]; ++j)
            if (pos[j] <= pos[j - 1]) { atomicOr(bad, 1u); break; }
}

// first posting of [b, e) with doc >= d (e if none)
__device__ __forceinline__ uint64_t post_lower_bound(const uint2* post, uint64_t b, uint64_t e, uint32_t d) {
    while (b < e) {
        const uint64_t m = (b + e) >> 1;
        if (__ldg(&post[m].x) < d) b = m + 1; else e = m;
    }
    return b;
}

__global__ void __launch_bounds__(256) phrase_match_kernel(TxtDev T, PhraseArgs A) {
    const uint64_t total = A.cap_off[A.nv];
    for (uint64_t g = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; g < total; g += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t lo = 0, hi = A.nv;   // the phrase of slot g: the last v with cap_off[v] <= g (empty phrases are skipped over)
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (__ldg(A.cap_off + mid) <= g) lo = mid; else hi = mid;
        }
        const uint32_t v = lo;
        const uint32_t* pt = A.terms + A.off[v];
        const uint32_t m = A.off[v + 1] - A.off[v], dv = A.driver[v];
        const uint64_t P = T.term_off[pt[dv]] + (g - A.cap_off[v]);
        const uint2 dp = T.post[P];
        const uint32_t doc = dp.x, f = doc / BM_FINE;
        const uint64_t p0 = A.pos_off[P], tf = A.pos_off[P + 1] - p0;
        uint32_t freq = 0;
        for (uint64_t c0 = 0; c0 < tf; c0 += 32) {   // 32 start positions at a time, one bit each
            const uint32_t n = tf - c0 < 32 ? (uint32_t)(tf - c0) : 32u;
            uint32_t mask = 0;
            for (uint32_t c = 0; c < n; ++c) mask |= (uint32_t)(__ldg(A.pos + p0 + c0 + c) >= dv) << c;   // a start below 0 cannot match
            for (uint32_t j = 0; j < m && mask; ++j) {
                if (j == dv) continue;
                const uint32_t t = pt[j];
                uint64_t b = T.term_off[t], e = T.term_off[t + 1];
                const uint32_t row = T.skip_row[t];
                if (row != NIL) {
                    const uint32_t* sk = T.skip + (uint64_t)row * (T.n_fine + 1) + f;
                    e = b + __ldg(sk + 1);
                    b += __ldg(sk);
                }
                const uint64_t Q = post_lower_bound(T.post, b, e, doc);
                if (Q == e || __ldg(&T.post[Q].x) != doc) { mask = 0; break; }
                uint64_t q = A.pos_off[Q];
                const uint64_t qe = A.pos_off[Q + 1];
                for (uint32_t bits = mask; bits; bits &= bits - 1) {   // starts ascend: one merge pass over the term's positions
                    const uint32_t c = __ffs(bits) - 1;
                    const uint32_t want = __ldg(A.pos + p0 + c0 + c) - dv + j;
                    while (q < qe && __ldg(A.pos + q) < want) ++q;
                    if (q == qe || __ldg(A.pos + q) != want) mask &= ~(1u << c);
                }
            }
            freq += __popc(mask);
        }
        A.out[g] = make_uint2(doc, (freq << 8) | (dp.y & 0xFFu));
    }
}

// one CTA per phrase: drop the slots that did not match, in place and in doc order; range = the list that is left
constexpr int PHRASE_COMPACT_THREADS = 1024;
__global__ void __launch_bounds__(PHRASE_COMPACT_THREADS) phrase_compact_kernel(PhraseArgs A) {
    using Scan = cub::BlockScan<uint32_t, PHRASE_COMPACT_THREADS>;
    __shared__ typename Scan::TempStorage tmp;
    const uint32_t v = blockIdx.x;
    const uint64_t b = A.cap_off[v], e = A.cap_off[v + 1];
    uint64_t kept = 0;
    for (uint64_t c = b; c < e; c += PHRASE_COMPACT_THREADS) {   // (uniform) a chunk is read before any of its slots is written
        const uint64_t i = c + threadIdx.x;
        const uint2 r = i < e ? A.out[i] : make_uint2(0, 0);
        const uint32_t keep = (r.y >> 8) != 0;
        uint32_t at, n;
        Scan(tmp).ExclusiveSum(keep, at, n);
        if (keep) A.out[b + kept + at] = r;
        kept += n;
        __syncthreads();
    }
    if (threadIdx.x == 0) { A.range[2 * v] = b; A.range[2 * v + 1] = b + kept; }
}

}  // namespace nidx
