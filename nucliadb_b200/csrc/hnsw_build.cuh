// nidx_b200 — K4: HNSW construction for nidx_vector (sm_90a).
//
// Reference: HnswBuilder (nidx/nidx_vector/src/hnsw/build.rs:36-166), driven by
// create_indexes / merge_indexes (segment.rs:241-286, 137-197) with rayon + per-node RwLocks.
// Here insertion is batch synchronous (DESIGN.md §build): per batch
//   1. hnsw_search_kernel (mode 1)  build.rs:123-150  every node of the batch searches the frozen graph;
//   2. select_link_kernel           build.rs:104-110  select_neighbours_heuristic(M) + the node's own row,
//                                                     and emits one reverse-edge record per selected neighbour;
//   3. (records sorted by (layer, neighbour), stable => ascending inserted id inside a segment)
//   4. reverse_link_kernel          build.rs:111-118  per neighbour: push the new edges in ascending id,
//                                                     re-select to prune_m(mmax) whenever the list exceeds mmax.
// select_neighbours_heuristic (build.rs:57-95) is ONE device routine used by 2 and 4.
#pragma once
#include "common.cuh"
#include "hnsw_search.cuh"

namespace nidx {

constexpr int HB_THREADS = 256;
constexpr int HB_WARPS = HB_THREADS / 32;
constexpr int HB_MAX_CAND = 256;  // efC <= 256 (candidates of one select), mmax + 1 <= 256

struct HeurSmem {
    uint32_t* cand_id;   // [HB_MAX_CAND]
    float* cand_sim;     // [HB_MAX_CAND]
    unsigned char* state;  // [HB_MAX_CAND] 0 = untouched, 1 = kept, 2 = discarded
    uint32_t* sel_id;    // [HB_MAX_CAND]
    float* sel_sim;      // [HB_MAX_CAND]
    float* cache;        // [cache_cap][ld] kept vectors
    int cache_cap;
    int* s_fail;
    int* s_nsel;
};

__host__ __device__ __forceinline__ size_t hb_smem_bytes(int ld, int cache_cap) {
    return (size_t)HB_MAX_CAND * (4 + 4 + 4 + 4 + 1) + 64 + (size_t)cache_cap * ld * 4;
}

__device__ inline void hb_carve(HeurSmem& h, unsigned char* p, int ld, int cache_cap, int* s_ints) {
    h.cache = reinterpret_cast<float*>(p); p += (size_t)cache_cap * ld * 4;
    h.cand_id = reinterpret_cast<uint32_t*>(p); p += HB_MAX_CAND * 4;
    h.cand_sim = reinterpret_cast<float*>(p); p += HB_MAX_CAND * 4;
    h.sel_id = reinterpret_cast<uint32_t*>(p); p += HB_MAX_CAND * 4;
    h.sel_sim = reinterpret_cast<float*>(p); p += HB_MAX_CAND * 4;
    h.state = p;
    h.cache_cap = cache_cap;
    h.s_fail = &s_ints[0];
    h.s_nsel = &s_ints[1];
}

// build.rs:57-95.  Candidates (id, similarity to the new node) in h.cand_* [0, nc) in the given order.
// Result in h.sel_* [0, return value).  All threads of the CTA call this.
__device__ inline int select_neighbours_heuristic(const VecDev& V, HeurSmem& h, int nc, int k) {
    int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int ng = V.ld >> 2;
    for (int i = threadIdx.x; i < nc; i += blockDim.x) h.state[i] = 0;
    if (threadIdx.x == 0) *h.s_nsel = 0;
    __syncthreads();
    int nsel = 0;
    // the candidates are visited one after the other and each costs a dependent read of its 3 KB row: keep the next few rows on
    // their way into L2 (a warp per row, a lane per 128-byte line)
    constexpr int AHEAD = 4;
    const int lines = (V.ld * 4 + 127) >> 7;
    if (warp < AHEAD && warp < nc)
        for (int l = lane; l < lines; l += 32) prefetch_l2(reinterpret_cast<const char*>(V.vecs + (size_t)h.cand_id[warp] * V.ld) + (size_t)l * 128);
    for (int i = 0; i < nc && nsel < k; ++i) {  // 66-69: stop once k are kept
        uint32_t x = h.cand_id[i];
        float sim = h.cand_sim[i];
        if (threadIdx.x == 0) *h.s_fail = 0;
        if (warp == HB_WARPS - 1 && i + AHEAD < nc)
            for (int l = lane; l < lines; l += 32) prefetch_l2(reinterpret_cast<const char*>(V.vecs + (size_t)h.cand_id[i + AHEAD] * V.ld) + (size_t)l * 128);
        __syncthreads();
        const float4* xv = reinterpret_cast<const float4*>(V.vecs + (size_t)x * V.ld);
        float xn = V.sim != SIM_DOT ? V.norms[x] : 0.0f;
        for (int j = warp; j < nsel; j += HB_WARPS) {  // 72-75: sim(x, new) > sim(x, y) for all kept y
            uint32_t y = h.sel_id[j];
            const float4* yv = j < h.cache_cap ? reinterpret_cast<const float4*>(h.cache + (size_t)j * V.ld)
                                               : reinterpret_cast<const float4*>(V.vecs + (size_t)y * V.ld);
            float ab = warp_dot(xv, yv, ng, lane);
            float inter = sim_from_parts(V.sim, ab, xn, V.norms[y]);
            if (lane == 0 && !(sim > inter)) *h.s_fail = 1;
        }
        __syncthreads();
        bool keep = *h.s_fail == 0;
        if (keep) {
            if (nsel < h.cache_cap)
                for (int g = threadIdx.x; g < ng; g += blockDim.x) reinterpret_cast<float4*>(h.cache + (size_t)nsel * V.ld)[g] = xv[g];
            if (threadIdx.x == 0) { h.sel_id[nsel] = x; h.sel_sim[nsel] = sim; h.state[i] = 1; }
            nsel++;
        } else if (threadIdx.x == 0) {
            h.state[i] = 2;
        }
        __syncthreads();
    }
    if (nsel < k) {  // 84-92 keepPrunedConnections: best discarded first, then sort the whole list desc
        int need = k - nsel;
        for (int i = threadIdx.x; i < nc; i += blockDim.x) {
            if (h.state[i] != 2) continue;
            uint64_t key = make_key(h.cand_sim[i], h.cand_id[i], 0);
            int r = 0;
            for (int j = 0; j < nc; ++j) r += (h.state[j] == 2 && make_key(h.cand_sim[j], h.cand_id[j], 0) > key);
            if (r < need) { int pos = atomicAdd(h.s_nsel, 1); h.sel_id[nsel + pos] = h.cand_id[i]; h.sel_sim[nsel + pos] = h.cand_sim[i]; }
        }
        __syncthreads();
        int total = nsel + *h.s_nsel;
        // sort_unstable_by desc (ties: lower id first), via ranks into cand_* as scratch
        uint32_t my_id[ (HB_MAX_CAND + HB_THREADS - 1) / HB_THREADS ];
        float my_sim[ (HB_MAX_CAND + HB_THREADS - 1) / HB_THREADS ];
        int my_r[ (HB_MAX_CAND + HB_THREADS - 1) / HB_THREADS ];
        int cnt = 0;
        for (int i = threadIdx.x; i < total; i += blockDim.x, ++cnt) {
            uint64_t key = make_key(h.sel_sim[i], h.sel_id[i], 0);
            int r = 0;
            for (int j = 0; j < total; ++j) r += (make_key(h.sel_sim[j], h.sel_id[j], 0) > key) || (j < i && make_key(h.sel_sim[j], h.sel_id[j], 0) == key);
            my_id[cnt] = h.sel_id[i]; my_sim[cnt] = h.sel_sim[i]; my_r[cnt] = r;
        }
        __syncthreads();
        cnt = 0;
        for (int i = threadIdx.x; i < total; i += blockDim.x, ++cnt) { h.sel_id[my_r[cnt]] = my_id[cnt]; h.sel_sim[my_r[cnt]] = my_sim[cnt]; }
        __syncthreads();
        nsel = total;
    }
    return nsel;
}

struct BuildArgs {
    int n_work;                 // work items (node, layer) of this batch
    const uint32_t* w_pos;      // [n_work] position of the node in the insertion order
    const unsigned char* w_layer;  // [n_work]
    const uint32_t* order;      // insertion order (node ids)
    uint32_t batch_begin;       // first position of the batch in `order`
    int efC, M;
    const uint64_t* found;      // [batch][HS_MAX_LAYERS][efC]
    const int* found_count;     // [batch][HS_MAX_LAYERS]
    uint64_t* rev_key;          // [n_work * M]  (layer << 32 | neighbour), ~0 = none
    uint32_t* rev_x;            // [n_work * M]
    float* rev_sim;             // [n_work * M]
    int cache_cap;
};

// build.rs:104-110 for one (node, layer) per CTA.
__global__ void __launch_bounds__(HB_THREADS) select_link_kernel(VecDev V, GraphDev G, BuildArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_ints[4];
    HeurSmem h;
    hb_carve(h, smem, V.ld, a.cache_cap, s_ints);
    int w = blockIdx.x;
    uint32_t pos = a.w_pos[w];
    int layer = a.w_layer[w];
    uint32_t x = a.order[pos];
    uint32_t slot = pos - a.batch_begin;
    int nc = a.found_count[(size_t)slot * HS_MAX_LAYERS + layer];
    const uint64_t* f = a.found + ((size_t)slot * HS_MAX_LAYERS + layer) * a.efC;
    for (int i = threadIdx.x; i < nc; i += blockDim.x) { h.cand_id[i] = key_id(f[i]); h.cand_sim[i] = key_score(f[i]); }
    __syncthreads();
    int nsel = select_neighbours_heuristic(V, h, nc, a.M);
    uint32_t* row = G.row(x, layer);
    float* wrow = G.wrow(x, layer);
    int stride = G.stride(layer);
    for (int i = threadIdx.x; i < stride; i += blockDim.x) {
        row[i] = i < nsel ? h.sel_id[i] : NIL;
        wrow[i] = i < nsel ? h.sel_sim[i] : 0.0f;
    }
    for (int i = threadIdx.x; i < a.M; i += blockDim.x) {
        size_t r = (size_t)w * a.M + i;
        a.rev_key[r] = i < nsel ? (((uint64_t)layer << 32) | h.sel_id[i]) : ~0ull;
        a.rev_x[r] = x;
        a.rev_sim[r] = i < nsel ? h.sel_sim[i] : 0.0f;
    }
}

struct ReverseArgs {
    int n_rev;
    const uint64_t* key_sorted;   // [n_rev]
    const uint32_t* idx_sorted;   // [n_rev] index into rev_x / rev_sim
    const uint32_t* rev_x;
    const float* rev_sim;
    int cache_cap;
    const uint32_t* heads;         // compacted segment heads (indices into key_sorted)
    const unsigned int* n_heads;
    unsigned int* work_counter;
};

// Segment heads of the sorted reverse-edge records (first record of every (layer, neighbour) run), compacted so
// that reverse_link_kernel only spends CTAs on real work.
__global__ void collect_heads_kernel(const uint64_t* __restrict__ key_sorted, int n_rev, uint32_t* __restrict__ heads, unsigned int* __restrict__ n_heads) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    bool head = i < n_rev && key_sorted[i] != ~0ull && (i == 0 || key_sorted[i - 1] != key_sorted[i]);
    unsigned m = __ballot_sync(0xFFFFFFFFu, head);
    if (m) {
        int lane = threadIdx.x & 31;
        unsigned base = 0;
        if (lane == 0) base = atomicAdd(n_heads, (unsigned)__popc(m));
        base = __shfl_sync(0xFFFFFFFFu, base, 0);
        if (head) heads[base + __popc(m & ((1u << lane) - 1))] = (uint32_t)i;
    }
}

// build.rs:111-118: persistent CTAs pull (layer, neighbour) segments from the compacted head list.  The minimum of one CTA per
// SM keeps ptxas from trimming the kernel to 48 registers for occupancy (with spills, 5 % slower on an H100): the ~100 KB vector
// cache already allows only two CTAs per SM at d = 768.
__global__ void __launch_bounds__(HB_THREADS, 1) reverse_link_kernel(VecDev V, GraphDev G, ReverseArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_ints[4];
    __shared__ unsigned int s_work;
    HeurSmem h;
    hb_carve(h, smem, V.ld, a.cache_cap, s_ints);
    const unsigned int n_heads = *a.n_heads;
    while (true) {
        __syncthreads();
        if (threadIdx.x == 0) s_work = atomicAdd(a.work_counter, 1u);
        __syncthreads();
        unsigned int wi = s_work;
        if (wi >= n_heads) break;
        int i0 = (int)a.heads[wi];
        uint64_t key = a.key_sorted[i0];
        int layer = (int)(key >> 32);
        uint32_t y = (uint32_t)key;
        uint32_t* row = G.row(y, layer);
        float* wrow = G.wrow(y, layer);
        int stride = G.stride(layer), mmax = G.mmax(layer);
        // current list -> sel_* (the working list lives in sel_*, candidates are staged into cand_*)
        uint32_t mine = threadIdx.x < stride ? row[threadIdx.x] : NIL;  // rows are prefix-filled, stride <= 64
        if (mine != NIL) { h.sel_id[threadIdx.x] = mine; h.sel_sim[threadIdx.x] = wrow[threadIdx.x]; }
        int len = __syncthreads_count(mine != NIL);
        for (int i = i0; i < a.n_rev && a.key_sorted[i] == key; ++i) {
            uint32_t src = a.idx_sorted[i];
            __syncthreads();
            if (threadIdx.x == 0) { h.sel_id[len] = a.rev_x[src]; h.sel_sim[len] = a.rev_sim[src]; }  // other_edges.push((x, dist))
            len++;
            __syncthreads();
            if (len > mmax) {  // 115-117
                for (int j = threadIdx.x; j < len; j += blockDim.x) { h.cand_id[j] = h.sel_id[j]; h.cand_sim[j] = h.sel_sim[j]; }
                __syncthreads();
                len = select_neighbours_heuristic(V, h, len, mmax * 95 / 100);   // params.rs:29-31 prune_m
            }
        }
        __syncthreads();
        for (int j = threadIdx.x; j < stride; j += blockDim.x) {
            row[j] = j < len ? h.sel_id[j] : NIL;
            wrow[j] = j < len ? h.sel_sim[j] : 0.0f;
        }
    }
}

}  // namespace nidx
