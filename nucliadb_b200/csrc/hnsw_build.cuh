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
constexpr int HB_PAIR_LD = HS_MAX_ROW + 1;  // a full adjacency row plus the pushed edge

// lane-blocked dot of two rows that both live in shared memory (same arithmetic as warp_dot)
__device__ __forceinline__ float warp_dot_ss(const float4* __restrict__ a, const float4* __restrict__ b, int ngroups, int lane) {
    float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
    for (int g = lane; g < ngroups; g += 32) {
        float4 va = a[g], vb = b[g];
        ax = __fmaf_rn(va.x, vb.x, ax);
        ay = __fmaf_rn(va.y, vb.y, ay);
        az = __fmaf_rn(va.z, vb.z, az);
        aw = __fmaf_rn(va.w, vb.w, aw);
    }
    return butterfly_sum(__fadd_rn(__fadd_rn(ax, ay), __fadd_rn(az, aw)));
}

struct HeurSmem {
    uint32_t* cand_id;   // [HB_MAX_CAND]
    float* cand_sim;     // [HB_MAX_CAND]
    unsigned char* state;  // [HB_MAX_CAND] 0 = untouched, 1 = kept, 2 = discarded
    uint32_t* sel_id;    // [HB_MAX_CAND]
    float* sel_sim;      // [HB_MAX_CAND]
    float* cache;        // [cache_cap][ld] kept vectors (PRELOAD: all candidate vectors)
    float* pair;         // PRELOAD: [HB_PAIR_LD][HB_PAIR_LD] pairwise similarities
    unsigned char* sel_src;  // PRELOAD: candidate index of each kept entry
    int cache_cap;
    int* s_fail;
    int* s_nsel;
};

__host__ __device__ __forceinline__ size_t hb_smem_bytes(int ld, int cache_cap, bool preload = false) {
    return (size_t)HB_MAX_CAND * (4 + 4 + 4 + 4 + 1 + 1) + 64 + (size_t)cache_cap * ld * 4 + (preload ? (size_t)HB_PAIR_LD * HB_PAIR_LD * 4 : 0);
}

__device__ inline void hb_carve(HeurSmem& h, unsigned char* p, int ld, int cache_cap, int* s_ints) {
    h.cache = reinterpret_cast<float*>(p); p += (size_t)cache_cap * ld * 4;
    h.cand_id = reinterpret_cast<uint32_t*>(p); p += HB_MAX_CAND * 4;
    h.cand_sim = reinterpret_cast<float*>(p); p += HB_MAX_CAND * 4;
    h.sel_id = reinterpret_cast<uint32_t*>(p); p += HB_MAX_CAND * 4;
    h.sel_sim = reinterpret_cast<float*>(p); p += HB_MAX_CAND * 4;
    h.state = p; p += HB_MAX_CAND;
    h.sel_src = p; p += HB_MAX_CAND;
    h.pair = reinterpret_cast<float*>(p);   // only carved when the launch reserved it (preload)
    h.cache_cap = cache_cap;
    h.s_fail = &s_ints[0];
    h.s_nsel = &s_ints[1];
}

// build.rs:57-95.  Candidates (id, similarity to the new node) in h.cand_* [0, nc) in the given order.
// Result in h.sel_* [0, return value).  All threads of the CTA call this.
// PRELOAD (prune of a full adjacency list, nc <= mmax + 1): every candidate vector is staged in shared memory
// once (h.cache row i = candidate i), all nc*(nc-1)/2 pairwise similarities are computed in parallel into
// h.pair, and the sequential pick of build.rs:66-82 becomes a walk over that table by one warp -- same
// comparisons, same result, without one HBM round trip and two barriers per candidate.
template <bool PRELOAD>
__device__ inline int select_neighbours_heuristic(const VecDev& V, HeurSmem& h, int nc, int k) {
    int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int ng = V.ld >> 2;
    for (int i = threadIdx.x; i < nc; i += blockDim.x) h.state[i] = 0;
    if (threadIdx.x == 0) *h.s_nsel = 0;
    __syncthreads();
    int nsel = 0;
    if (PRELOAD) {
        for (int i = warp; i < nc; i += HB_WARPS) {   // one warp per candidate row: 3 KB coalesced, asynchronous (the rows of a warp overlap)
            const float4* src = reinterpret_cast<const float4*>(V.vecs + (size_t)h.cand_id[i] * V.ld);
            float4* dst = reinterpret_cast<float4*>(h.cache + (size_t)i * V.ld);
            for (int g = lane; g < ng; g += 32) cp_async16(dst + g, src + g);
        }
        cp_async_commit_wait_all();
        __syncthreads();
        // All pairwise similarities, register tiled: a warp takes a 4 x 4 block of (i, j) pairs, loads the eight rows' float4 groups
        // once per group and keeps the 16 pairs' four accumulators in registers -- a quarter of the shared-memory reads of one
        // dot per pair (the phase is bound by shared-memory bandwidth: 33 x 32 / 2 pairs x 6 KB).  Per pair the arithmetic is
        // exactly warp_dot_ss's (lane-blocked groups in increasing order, four FMA accumulators, the same butterfly): bit-identical.
        {
            const int nb = (nc + 3) >> 2;                 // blocks of four rows
            const int nblk = nb * (nb + 1) / 2;           // block pairs (ib >= jb)
            for (int bp = warp; bp < nblk; bp += HB_WARPS) {
                int ib = (int)((sqrtf(1.0f + 8.0f * (float)bp) - 1.0f) * 0.5f);
                while (ib * (ib + 1) / 2 > bp) --ib;
                while ((ib + 1) * (ib + 2) / 2 <= bp) ++ib;
                const int jb = bp - ib * (ib + 1) / 2;
                float acc[4][4][4];
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c2 = 0; c2 < 4; ++c2) { acc[r][c2][0] = 0.f; acc[r][c2][1] = 0.f; acc[r][c2][2] = 0.f; acc[r][c2][3] = 0.f; }
                const float4* rows_i[4];
                const float4* rows_j[4];
#pragma unroll
                for (int r = 0; r < 4; ++r) {
                    rows_i[r] = reinterpret_cast<const float4*>(h.cache + (size_t)min(ib * 4 + r, nc - 1) * V.ld);
                    rows_j[r] = reinterpret_cast<const float4*>(h.cache + (size_t)min(jb * 4 + r, nc - 1) * V.ld);
                }
                for (int g = lane; g < ng; g += 32) {
                    float4 va[4], vb[4];
#pragma unroll
                    for (int r = 0; r < 4; ++r) { va[r] = rows_i[r][g]; vb[r] = rows_j[r][g]; }
#pragma unroll
                    for (int r = 0; r < 4; ++r)
#pragma unroll
                        for (int c2 = 0; c2 < 4; ++c2) {
                            acc[r][c2][0] = __fmaf_rn(va[r].x, vb[c2].x, acc[r][c2][0]);
                            acc[r][c2][1] = __fmaf_rn(va[r].y, vb[c2].y, acc[r][c2][1]);
                            acc[r][c2][2] = __fmaf_rn(va[r].z, vb[c2].z, acc[r][c2][2]);
                            acc[r][c2][3] = __fmaf_rn(va[r].w, vb[c2].w, acc[r][c2][3]);
                        }
                }
#pragma unroll
                for (int r = 0; r < 4; ++r)
#pragma unroll
                    for (int c2 = 0; c2 < 4; ++c2) {
                        const int i = ib * 4 + r, j = jb * 4 + c2;
                        float ab = butterfly_sum(__fadd_rn(__fadd_rn(acc[r][c2][0], acc[r][c2][1]), __fadd_rn(acc[r][c2][2], acc[r][c2][3])));
                        if (lane == 0 && i < nc && j < i) {
                            float sv = sim_from_parts(V.sim, ab, V.norms[h.cand_id[i]], V.norms[h.cand_id[j]]);
                            h.pair[i * HB_PAIR_LD + j] = sv;
                            h.pair[j * HB_PAIR_LD + i] = sv;
                        }
                    }
            }
        }
        __syncthreads();
        if (warp == 0) {   // 66-82 on the table: lanes test the kept set in parallel
            int kept = 0;
            for (int i = 0; i < nc && kept < k; ++i) {
                float sim = h.cand_sim[i];
                bool bad = false;
                for (int j0 = 0; j0 < kept; j0 += 32) {
                    int j = j0 + lane;
                    bad = bad || (j < kept && !(sim > h.pair[i * HB_PAIR_LD + h.sel_src[j]]));
                }
                bad = __any_sync(0xFFFFFFFFu, bad);
                if (lane == 0) {
                    if (!bad) { h.sel_id[kept] = h.cand_id[i]; h.sel_sim[kept] = sim; h.sel_src[kept] = (unsigned char)i; h.state[i] = 1; }
                    else h.state[i] = 2;
                }
                __syncwarp();
                if (!bad) kept++;
            }
            if (lane == 0) *h.s_fail = kept;
        }
        __syncthreads();
        nsel = *h.s_fail;
    } else {
    // the candidates are visited one after the other and each costs a dependent read of its 3 KB row: keep the next few rows on
    // their way into L2 (a warp per row, a lane per 128-byte line)
    constexpr int AHEAD = 4;
    const int lines = (V.ld * 4 + 127) >> 7;
    if (warp < AHEAD && warp < nc)
        for (int l = lane; l < lines; l += 32) asm volatile("prefetch.global.L2 [%0];" :: "l"(reinterpret_cast<const char*>(V.vecs + (size_t)h.cand_id[warp] * V.ld) + (size_t)l * 128));
    for (int i = 0; i < nc && nsel < k; ++i) {  // 66-69: stop once k are kept
        uint32_t x = h.cand_id[i];
        float sim = h.cand_sim[i];
        if (threadIdx.x == 0) *h.s_fail = 0;
        if (warp == HB_WARPS - 1 && i + AHEAD < nc)
            for (int l = lane; l < lines; l += 32) asm volatile("prefetch.global.L2 [%0];" :: "l"(reinterpret_cast<const char*>(V.vecs + (size_t)h.cand_id[i + AHEAD] * V.ld) + (size_t)l * 128));
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
    int nsel = select_neighbours_heuristic<false>(V, h, nc, a.M);
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
    int preload;   // 1: the whole list (mmax + 1 vectors) fits in shared memory -> table-driven prune
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

// build.rs:111-118: persistent CTAs pull (layer, neighbour) segments from the compacted head list.
__global__ void __launch_bounds__(HB_THREADS) reverse_link_kernel(VecDev V, GraphDev G, ReverseArgs a) {
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
                len = a.preload ? select_neighbours_heuristic<true>(V, h, len, mmax * 95 / 100)   // params.rs:29-31 prune_m
                                : select_neighbours_heuristic<false>(V, h, len, mmax * 95 / 100);
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
