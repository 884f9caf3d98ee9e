// nidx_b200 — K9: rank fusion on the device (sm_90a).  SURVEY 8f rank 4: the step that follows a shard search in the reference
// runs in Python on the host:
//   nucliadb/src/nucliadb/search/search/rank_fusion.py:78-96    RankFusionAlgorithm.fuse (one non-empty source: no fusion)
//   nucliadb/src/nucliadb/search/search/rank_fusion.py:143-186  ReciprocalRankFusion._fuse
//       score(d) = sum over the sources r, in the order given, of 1 / (k + rank_r(d)) * w(r)       (Python floats: IEEE doubles)
// One CTA per query.  The items of all sources are laid out in shared memory in insertion order (source by source, best first:
// every source arrives sorted by score descending, which is what the reference's stable re-sort would produce).  A thread per
// item finds the item's first occurrence (the reference keeps that object), the first occurrence adds the terms of all its later
// occurrences IN ORDER -- the f64 sum then has the reference's association -- and a rank by counting (score desc, insertion order
// for ties = Python's stable sort) places it.  Work is O(items^2 / threads) per query: a few hundred items at most.
// Scores are bit-identical to the reference's (tests/golden/rank_fusion.json comes from the reference's own class).
#pragma once
#include "common.cuh"

namespace nidx {

constexpr int RF_THREADS = 128;
constexpr int RF_MAX_SOURCES = 4;

struct RrfSourceDev {
    const uint64_t* keys;     // [nq][k] item keys (a paragraph id), best first
    const float* scores;      // [nq][k] the source's own scores (only reported when fusion is skipped)
    const int32_t* counts;    // [nq] valid entries per query (nullptr: k, minus trailing key == ~0)
    int k;
    double weight;
};

struct RrfArgs {
    RrfSourceDev src[RF_MAX_SOURCES];
    int n_sources, nq, cap;   // cap = sum of the sources' k = row length of the outputs
    double k;
    uint64_t* out_keys;       // [nq][cap]
    double* out_scores;       // [nq][cap]
    uint32_t* out_refs;       // [nq][cap] first occurrence: source << 28 | source mask << 24 | position in that source
    int32_t* out_counts;      // [nq]
};

__host__ __device__ __forceinline__ size_t rf_smem_bytes(int cap) { return (size_t)cap * (8 + 8 + 4 + 4) + 64; }

__global__ void __launch_bounds__(RF_THREADS) rrf_fuse_kernel(RrfArgs a) {
    extern __shared__ __align__(16) unsigned char rf_smem[];
    __shared__ int s_off[RF_MAX_SOURCES + 1], s_nonempty, s_nout;
    uint64_t* key = reinterpret_cast<uint64_t*>(rf_smem);
    double* val = reinterpret_cast<double*>(key + a.cap);
    uint32_t* ref = reinterpret_cast<uint32_t*>(val + a.cap);   // source << 28 | mask << 24 | position
    int* slot = reinterpret_cast<int*>(ref + a.cap);            // output position of a first occurrence, -1 for the others
    const int q = blockIdx.x;
    if (threadIdx.x == 0) {
        int off = 0, ne = 0;
        for (int s = 0; s < a.n_sources; ++s) {
            s_off[s] = off;
            int c = a.src[s].counts ? a.src[s].counts[q] : a.src[s].k;
            c = max(0, min(c, a.src[s].k));
            if (!a.src[s].counts) while (c > 0 && a.src[s].keys[(size_t)q * a.src[s].k + c - 1] == ~0ull) --c;
            off += c;
            ne += c > 0;
        }
        s_off[a.n_sources] = off;
        s_nonempty = ne;
        s_nout = 0;
    }
    __syncthreads();
    const int total = s_off[a.n_sources];
    const bool fuse = s_nonempty != 1;                     // rank_fusion.py:86-89
    for (int t = threadIdx.x; t < total; t += RF_THREADS) {
        int s = 0;
        while (t >= s_off[s + 1]) ++s;
        int r = t - s_off[s];
        key[t] = a.src[s].keys[(size_t)q * a.src[s].k + r];
        val[t] = fuse ? __dmul_rn(__ddiv_rn(1.0, __dadd_rn(a.k, (double)r)), a.src[s].weight)     // 1 / (k + rank) * weight
                      : (double)a.src[s].scores[(size_t)q * a.src[s].k + r];
        ref[t] = ((uint32_t)s << 28) | (1u << (24 + s)) | (uint32_t)r;
    }
    __syncthreads();
    // First occurrences accumulate their later occurrences, in insertion order (the reference's `rrf_score.score += ...`).  In place:
    // a first occurrence writes only its own val / ref, and reads val / ref of LATER occurrences, which nobody writes.
    for (int t = threadIdx.x; t < total; t += RF_THREADS) {
        bool f = true;
        if (fuse) {
            uint64_t kt = key[t];
            for (int u = 0; u < t && f; ++u) f = key[u] != kt;
            if (f) {
                double acc = val[t];
                uint32_t rf = ref[t];
                for (int u = t + 1; u < total; ++u)
                    if (key[u] == kt) { acc = __dadd_rn(acc, val[u]); rf |= ref[u] & 0x0F000000u; }
                val[t] = acc;
                ref[t] = rf;
            }
        }
        slot[t] = f ? 0 : -1;          // -1 = a later occurrence (dropped); ranks written below are >= 0
    }
    __syncthreads();
    // stable rank: score descending, insertion order among equals (list.sort(key=score, reverse=True) is stable)
    for (int t = threadIdx.x; t < total; t += RF_THREADS) {
        if (slot[t] < 0) continue;
        double v = val[t];
        int r = 0;
        for (int u = 0; u < total; ++u)
            if (slot[u] >= 0) r += (val[u] > v) || (val[u] == v && u < t);
        slot[t] = r;
        atomicAdd(&s_nout, 1);
    }
    __syncthreads();
    const int nout = s_nout;
    uint64_t* ok = a.out_keys + (size_t)q * a.cap;
    double* os = a.out_scores + (size_t)q * a.cap;
    uint32_t* orf = a.out_refs + (size_t)q * a.cap;
    for (int t = threadIdx.x; t < total; t += RF_THREADS)
        if (slot[t] >= 0) { int r = slot[t]; ok[r] = key[t]; os[r] = val[t]; orf[r] = ref[t]; }
    for (int i = nout + threadIdx.x; i < a.cap; i += RF_THREADS) { ok[i] = ~0ull; os[i] = 0.0; orf[i] = NIL; }
    if (threadIdx.x == 0) a.out_counts[q] = nout;
}

// ids -> caller keys: vector results (vector address -> paragraph -> key) and BM25 results (document -> key); NIL -> ~0
__global__ void ids_to_keys_kernel(const uint32_t* __restrict__ ids, size_t n, const uint32_t* __restrict__ paragraph_of, const uint64_t* __restrict__ keys,
                                   uint64_t* __restrict__ out) {
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
        uint32_t id = ids[i];
        if (id == NIL) { out[i] = ~0ull; continue; }
        uint32_t p = paragraph_of ? paragraph_of[id] : id;
        out[i] = keys ? keys[p] : (uint64_t)p;
    }
}

}  // namespace nidx
