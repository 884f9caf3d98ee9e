// nidx_b200 — K2/K3: HNSW search for nidx_vector (sm_90a).
//
// One CTA walks one query (or, in build mode, one node to insert) through the graph:
//   HnswSearcher::layer_search      nidx/nidx_vector/src/hnsw/search.rs:242-304
//   HnswSearcher::search            search.rs:306-383  (descent with k=1, layer 0 with max(k, ef))
//   HnswSearcher::closest_up_nodes  search.rs:188-240  (filter / dedup aware expansion to k results)
//   NodeFilter::passes              search.rs:135-171
//   HnswBuilder::insert (search half) hnsw/build.rs:123-150
//
// Data structures per CTA, all in shared memory:
//   * ONE sorted list of 64-bit rank keys (score desc, id asc) with an "unexpanded" flag in bit 0.
//     It is the reference's two BinaryHeaps folded together: a candidate that is not among the best
//     `ef` results can never be expanded (popping it ends the search, search.rs:268-273), so the
//     candidates that matter are exactly the unexpanded members of the result list.
//   * an exact visited set (open-addressing hash of node ids) = the reference's FxHashSet;
//   * the query vector; up to 64 neighbour ids / keys of the node being expanded.
// Per expansion: warp 0 reads the adjacency row (one 128-byte line for M0=32) and filters it through
// the visited set; all warps compute one similarity each (3 KB coalesced, streamed past L1; the
// lane-blocked summation order of common.cuh makes scores bit-identical to the oracle's); the CTA
// merges the admitted keys into the list by rank (no sort).
#pragma once
#include <limits.h>

#include "common.cuh"

namespace nidx {

constexpr int HS_WARPS = 8;
constexpr int HS_THREADS = HS_WARPS * 32;
constexpr int HS_MAX_ROW = 64;      // stride of an adjacency row (M0 <= 64)
constexpr int HS_MAX_LAYERS = 8;    // found[] layers kept per inserted node (level > 7 has p < 1e-9)

struct SearchArgs {
    int mode;  // 0 = query (search.rs:306-383), 1 = build (build.rs:123-150)
    int nq;
    // query mode
    const float* queries;  // [nq][ld] zero padded
    const float* qnorms;   // [nq] (cosine)
    int k, ef0;            // ef0 = max(k, ef)
    float min_score;
    int with_duplicates, multi_vector;
    const uint64_t* filter;  // bitset over paragraphs (filter ∧ alive) or nullptr
    uint32_t* out_ids; float* out_scores; int* out_counts;
    // build mode
    const uint32_t* nodes;   // [nq]
    int efC;
    uint64_t* found;         // [nq][HS_MAX_LAYERS][efC] rank keys (flag bit 0)
    int* found_count;        // [nq][HS_MAX_LAYERS]
    // shared
    int hash_bits;           // visited table = 1 << hash_bits slots
    int list_cap;            // >= max(ef0, efC) and >= cu_cap
    int cu_cap;              // closest_up_nodes pending-candidate capacity
    unsigned int* work_counter;       // dynamic query scheduler (zeroed by the host)
    unsigned long long* counters;     // [0] similarities [1] expansions [2] visited overflows [3] cu overflows [4] RaBitQ estimates [5] exact similarities the sequential rerank_top needs
    // quantised walk (hnsw_rabitq.cuh; hnsw/search.rs:332-366 with SearchVector::RabitQ)
    const unsigned char* codes;       // [n][code_stride] vectors.quant records
    int code_stride;
    const uint32_t* planes;           // [nq][4][d/32] query bit planes
    const void* qparams;              // [nq] RabitqQueryParams
    uint32_t* gvisited;               // [grid][1 << gv_bits] layer-0 visited table in global memory (L2)
    int gv_bits;
    int last_k;                       // min(k * RERANKING_FACTOR, RERANKING_LIMIT)
};

// An exact visited set: open addressing over 1 << bits slots of node ids (NIL = free), linear probing.  Threads insert concurrently.
struct VisitedSet {
    uint32_t* slots;
    uint32_t mask;
    int bits;
    int limit;   // count at which inserts stop: a pass inserts at most one adjacency row, so the table stays below 15/16 full

    __device__ void init(uint32_t* s, int b) {
        slots = s; bits = b; mask = (1u << b) - 1;
        limit = (int)((15u << b) >> 4) - HS_MAX_ROW;
    }
    __device__ uint32_t slot(uint32_t y) const { return (y * 2654435761u) >> (32 - bits); }
    // Every thread of the CTA; 4 << bits bytes, 16-byte aligned.
    __device__ void clear() const {
        const uint4 e4 = make_uint4(NIL, NIL, NIL, NIL);
        for (uint32_t i = threadIdx.x; i < (mask + 1) / 4; i += blockDim.x) reinterpret_cast<uint4*>(slots)[i] = e4;
    }
    // True iff y was not in the set (and is now).  `count` is the number of ids the set held when the pass of inserts began: the
    // callers publish the new count only after the pass.  A full table reports "already visited" and sets `overflow`.
    __device__ bool insert(uint32_t y, int count, bool& overflow) const {
        if (count >= limit) { overflow = true; return false; }
        for (uint32_t h = slot(y);; h = (h + 1) & mask) {
            const uint32_t old = atomicCAS(&slots[h], NIL, y);
            if (old == NIL) return true;
            if (old == y) return false;
        }
    }

    // closest_up_nodes on top of the layer-0 walk's set (hs_closest_up<DEFER>): the ids it has reached carry MARK (ids < 2^31 - 1,
    // so y | MARK != NIL).  0 if y was reached before (or the table is full, as insert), 1 if y was not in the table, 2 if only
    // the layer-0 walk had visited it.
    static constexpr uint32_t MARK = 0x80000000u;
    __device__ int mark(uint32_t y, int count, bool& overflow) const {
        if (count >= limit) { overflow = true; return 0; }
        for (uint32_t h = slot(y);; h = (h + 1) & mask) {
            uint32_t old = atomicCAS(&slots[h], NIL, y | MARK);
            if (old == NIL) return 1;
            if (old == y) {
                old = atomicCAS(&slots[h], y, y | MARK);
                if (old == y) return 2;
            }
            if (old == (y | MARK)) return 0;
        }
    }
};

// What one expansion leaves for hs_merge and for the code after it.  There are two records, used by alternate hops (the parity of
// SearchCtx::hop), so that one can be reset while threads still read the other: hs_expand resets its own before its first barrier,
// rq_expand (whose atomics come before its barrier) the next hop's after it, and hs_reseed both.
struct HopRec {
    unsigned long long maxtodo;  // the largest admitted key: list entries above it keep their position in the merge
    int ntodo;                   // hs_expand: todo_key[0, ntodo) holds the scored neighbours, 0 for a refused one
    int nadmit;                  // admitted keys (rq_expand compacts them into todo_key[0, nadmit))
    int best_next;               // hs_merge's atomicMin: the first unexpanded entry of the merged list
    int pred;                    // rq_expand: list position of the predicted next candidate (-1: none)
    int nfresh;                  // rq_expand: neighbours not visited before
    int overflow;                // rq_expand: the visited set was full

    __device__ void clear() { maxtodo = 0; nadmit = 0; best_next = INT_MAX; nfresh = 0; overflow = 0; }
};

struct SearchCtx {
    float* qvec;
    uint64_t *A, *B;
    VisitedSet vis;       // the shared-memory visited set
    uint32_t* todo_id;
    uint64_t* todo_key;
    uint32_t* pref_row;   // [2][HS_MAX_ROW] speculatively prefetched adjacency rows (double buffered by hop parity)
    uint32_t* pref_node;  // [2] node each buffer belongs to (NIL = none)
    int *s_len, *s_best, *s_hash_count, *s_flag;
    unsigned long long* s_dropped;   // closest_up_nodes: the best key a full list has dropped (0: none)
    HopRec* hops;         // [2], by hop parity
    unsigned hop;         // expansions so far; hs_expand and rq_expand advance it at their end
    float qnorm;
    float qbound;                    // >= |q| (hs_query_bound), for the screen's error bound
    unsigned long long n_dist, n_expand, n_overflow;
    unsigned long long n_skip;       // similarities the screen settled without reading the f32 row

    __device__ HopRec& last_hop() const { return hops[(hop & 1u) ^ 1u]; }   // the record of the expansion that just ran
};

// An upper bound on |q| for the query in shared memory, the same in every thread: the squares are exact in f64 and the f64 sum
// of ld of them is within ld * 2^-53 of its value, which the factor 1 + 2^-20 covers (ld < 2^30).
__device__ inline float hs_query_bound(const float* q, int ld) {
    double s = 0.0;
    for (int i = threadIdx.x & 31; i < ld; i += 32) s = fma((double)q[i], (double)q[i], s);
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, off);
    return __double2float_ru(__dsqrt_ru(__dmul_ru(s, 1.0 + 0x1p-20)));
}

// The screen of a neighbour y of the layer search, given ah = warp_dot_h of its fp16 row and r = its hrec record: true when the
// exact key cannot exceed wkey, so the f32 row need not be read.
//   Let a be the f32 dot warp_dot_t computes and p the real dot <v, q>.  Both dots round each product term at most
//   m = dot_depth(ld) times, so |a - p| <= g_m * |v| |q| + ld * 2^-149 and |ah * 2^-e - <h', q>| <= g_m * |h'| |q| + ld * 2^-149 * 2^-e
//   + 2^-150 (g_m = m u / (1 - m u), u = 2^-24; 2^-149 per fused multiply-add for subnormal results; the scaling by 2^-e is exact
//   unless it underflows), with h' = h * 2^-e.  |<h', q> - p| <= rho |q|, rho = |h' - v| and |h'| <= |v| + rho.  Together:
//   |ah * 2^-e - a| <= |q| (rho + g_m (2 |v| + rho)) + 2^-149 (ld (1 + 2^-e) + 1) = |q| * err_q + err_abs (hs_half_kernel rounds
//   both up), and bnd below is rounded up again, so ab_up >= a.
//   sim_from_parts never decreases as ab grows (for the three similarities, the ab == 0 and zero-norm cases of cosine included;
//   ab_up >= +0 whenever a >= +0, so total_cmp's -0 < +0 cannot invert it) and make_key is monotone: key(a) <= key(ab_up) <= wkey.
//   The bound needs every partial sum finite: bnd >= 2^-20 |v| |q| (g_m >= 8u), so bnd <= 2^100 keeps both dots' partial sums
//   below 2^121.  A row with a non-finite element has err_q = +inf, a non-finite query gives a non-finite qbound, and an overflowed
//   fp16 dot is non-finite: all of these fail the test and read the f32 row.
__device__ __forceinline__ bool hs_screened_out(const VecDev& V, const SearchCtx& c, uint32_t y, float ah, float4 r, uint64_t wkey) {
    float a = __fmul_rn(ah, r.y);
    float bnd = __fmaf_ru(c.qbound, r.z, r.w);
    if (!(fabsf(a) <= 0x1p120f && bnd <= 0x1p100f)) return false;
    float s_up = sim_from_parts(V.sim, __fadd_ru(a, bnd), r.x, c.qnorm);
    return make_key(s_up, y, 1) <= wkey;
}

__host__ __device__ __forceinline__ size_t hs_smem_bytes(int ld, int list_cap, int hash_bits) {
    return (size_t)ld * 4 + (size_t)list_cap * 16 + ((size_t)4 << hash_bits) + HS_MAX_ROW * 12 + HS_MAX_ROW * 8 + 16 + 64;
}

// The CTA's shared state of a walk: the dynamic shared memory laid out as hs_smem_bytes counts it, from `p` on, and the shared
// scalars.  Returns the end of the layout, where the quantised walk lays out its own arrays.
__device__ inline unsigned char* hs_setup(SearchCtx& c, const SearchArgs& a, unsigned char* p, int ld) {
    __shared__ int s_ints[4];
    __shared__ HopRec s_hops[2];
    __shared__ unsigned long long s_drop;
    c.qvec = reinterpret_cast<float*>(p); p += (size_t)ld * 4;
    c.A = reinterpret_cast<uint64_t*>(p); p += (size_t)a.list_cap * 8;
    c.B = reinterpret_cast<uint64_t*>(p); p += (size_t)a.list_cap * 8;
    c.todo_key = reinterpret_cast<uint64_t*>(p); p += HS_MAX_ROW * 8;
    c.vis.init(reinterpret_cast<uint32_t*>(p), a.hash_bits); p += (size_t)4 << a.hash_bits;
    c.todo_id = reinterpret_cast<uint32_t*>(p); p += HS_MAX_ROW * 4;
    c.pref_row = reinterpret_cast<uint32_t*>(p); p += 2 * HS_MAX_ROW * 4;
    c.pref_node = reinterpret_cast<uint32_t*>(p); p += 16;
    c.s_len = &s_ints[0]; c.s_best = &s_ints[1]; c.s_hash_count = &s_ints[2]; c.s_flag = &s_ints[3];
    c.hops = s_hops;
    c.s_dropped = &s_drop;
    c.hop = 0;
    c.qnorm = 0.0f;
    c.n_dist = c.n_expand = c.n_overflow = c.n_skip = 0;
    return p;
}

// The dynamic scheduler: the CTA's next query in *q, false when every query has been taken.
__device__ inline bool hs_next_query(const SearchArgs& a, unsigned* q) {
    __shared__ unsigned s_work;
    __syncthreads();
    if (threadIdx.x == 0) s_work = atomicAdd(a.work_counter, 1u);
    __syncthreads();
    *q = s_work;
    return *q < (unsigned)a.nq;
}

// counters [0]-[3]: n_dist lives in lane 0 of every warp, the rest in thread 0
__device__ inline void hs_flush_counters(const SearchCtx& c, unsigned long long* counters) {
    if ((threadIdx.x & 31) == 0 && c.n_dist) atomicAdd(&counters[0], c.n_dist);
    if (threadIdx.x == 0) {
        if (c.n_expand) atomicAdd(&counters[1], c.n_expand);
        if (c.n_overflow & 0xFFFFFFFFull) atomicAdd(&counters[2], c.n_overflow & 0xFFFFFFFFull);
        if (c.n_overflow >> 32) atomicAdd(&counters[3], c.n_overflow >> 32);
    }
}

// Start a layer search (or closest_up_nodes) on the list in c.A: every entry unexpanded, the visited set `vis` = the list's ids,
// both hop records reset.  MARKED: the list's ids are marked (VisitedSet::mark), in the table as it stands when `keep`.
template <bool MARKED = false>
__device__ inline void hs_reseed(SearchCtx& c, const VisitedSet& vis, bool keep = false) {
    __syncthreads();
    if (!(MARKED && keep)) vis.clear();
    if (threadIdx.x == 0) {
        *c.s_hash_count = 0; *c.s_best = 0; *c.s_dropped = 0; c.pref_node[0] = NIL; c.pref_node[1] = NIL;
        c.hops[0].clear(); c.hops[1].clear();
    }
    __syncthreads();
    int len = *c.s_len;
    bool ov = false;
    for (int i = threadIdx.x; i < len; i += blockDim.x) {
        uint64_t key = c.A[i] | 1ull;
        c.A[i] = key;
        if (MARKED) vis.mark(key_id(key), 0, ov);
        else vis.insert(key_id(key), 0, ov);
    }
    __syncthreads();
    if (threadIdx.x == 0) *c.s_hash_count = len;
    __syncthreads();
}

// The node expanded next, unless a new neighbour outranks it, is the first unexpanded list entry after `best` (CU: entry 1, the
// next one once the popped candidate is dropped).  The last warp starts an asynchronous copy (cp.async) of its adjacency row into
// the other half of the double buffer while the hop works; the row's HBM latency then overlaps the hop's own loads.  The caller
// waits for the copy before the hop's last barrier.  Returns the entry's list position, -1 if there is none.
template <bool CU>
__device__ inline int hs_prefetch_next(const GraphDev& G, SearchCtx& c, int layer, int best, int len) {
    const int lane = threadIdx.x & 31;
    const int stride = G.stride(layer);
    int pred = -1;
    if (CU) {
        pred = len > 1 ? 1 : -1;
    } else {
        for (int i0 = best + 1; i0 < len && pred < 0; i0 += 32) {
            int i = i0 + lane;
            unsigned m = __ballot_sync(0xFFFFFFFFu, i < len && (c.A[i] & 1ull));
            if (m) pred = i0 + __ffs(m) - 1;
        }
    }
    uint32_t pnode = NIL;
    if (pred >= 0) {
        pnode = key_id(c.A[pred]);
        const uint32_t* row = G.row(pnode, layer);
        uint32_t* dst = c.pref_row + ((c.hop & 1u) ^ 1u) * HS_MAX_ROW;
        for (int e = lane; e < stride; e += 32) cp_async4(dst + e, row + e);
    }
    if (lane == 0) c.pref_node[(c.hop & 1u) ^ 1u] = pnode;
    return pred;
}

// Expand `node` (already chosen): gather unvisited neighbours (warp 0), score them (all warps).
// Admission: layer_search (search.rs:286) -- when the list holds `ef` entries only keys better than the
// worst survive; closest_up_nodes (search.rs:231) -- score >= min_score.
// Speculation: while warp 0 works, the last warp prefetches the row of the predicted next node (hs_prefetch_next).
// The hop's record: warp 0 resets it before the first barrier, the scoring after it adds the admitted keys.
// LEAN (the layer search's hot loop): the list length arrives in a register, so that hs_merge needs no barrier after thread 0 has
// published the new length -- three barriers per expansion instead of four.
// DEFER (CU, hs_closest_up<.., true>): visits are marked (VisitedSet::mark), and a neighbour only the layer-0 walk had visited is
// settled without its row.
template <bool CU, int NG, int W = HS_WARPS, bool LEAN = false, bool DEFER = false>
__device__ inline void hs_expand(const VecDev& V, const GraphDev& G, SearchCtx& c, uint32_t node, int layer, int ef, float min_score, int best, int len_in = -1) {
    int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int stride = G.stride(layer);
    unsigned cur = c.hop & 1u;
    HopRec& h = c.hops[cur];
    if (warp == 0) {
        const uint32_t* prow = c.pref_row + cur * HS_MAX_ROW;
        bool hit = c.pref_node[cur] == node;
        const uint32_t* row = G.row(node, layer);
        const int visited = *c.s_hash_count;
        int ntodo = 0;
        bool ov = false;
        for (int e0 = 0; e0 < stride; e0 += 32) {
            uint32_t y = NIL;
            if (e0 + lane < stride) y = hit ? prow[e0 + lane] : __ldg(row + e0 + lane);
            bool fresh;
            if (DEFER) {   // todo_id carries MARK for a neighbour to settle without its row
                const int m = y != NIL ? c.vis.mark(y, visited, ov) : 0;
                fresh = m != 0;
                if (m == 2) y |= VisitedSet::MARK;
            } else fresh = (y != NIL) && c.vis.insert(y, visited, ov);
            unsigned mask = __ballot_sync(0xFFFFFFFFu, fresh);
            if (fresh) c.todo_id[ntodo + __popc(mask & ((1u << lane) - 1))] = y;
            ntodo += __popc(mask);
        }
        if (__any_sync(0xFFFFFFFFu, ov) && lane == 0) c.n_overflow++;
        if (lane == 0) {
            h.ntodo = ntodo;
            *c.s_hash_count = visited + ntodo;
            h.best_next = INT_MAX;
            h.nadmit = 0;
            h.maxtodo = 0;
            c.n_expand++;
        }
    } else if (warp == W - 1) {
        hs_prefetch_next<CU>(G, c, layer, best, LEAN ? len_in : *c.s_len);
    }
    __syncthreads();
    int ntodo = h.ntodo, len = LEAN ? len_in : *c.s_len;
    uint64_t wkey = (!CU && len >= ef) ? c.A[len - 1] : 0;
    int ng = V.ld >> 2;
    auto finish = [&](int j, uint32_t y, float ab, float vnorm) {
        float s = sim_from_parts(V.sim, ab, vnorm, c.qnorm);
        uint64_t key = make_key(s, y, 1);
        bool admit = CU ? (s >= min_score) : (wkey == 0 || s > key_score(wkey));   // search.rs:286 compares scores: a tie with the worst is refused
        c.todo_key[j] = admit ? key : 0;
        if (admit) { atomicAdd(&h.nadmit, 1); atomicMax(&h.maxtodo, (unsigned long long)key); }
        c.n_dist++;
    };
    // Screen (layer search with a full list): a neighbour whose fp16 dot plus its error bound cannot beat wkey is rejected
    // without reading its f32 row (hs_screened_out); the others take the exact path below unchanged.
    const bool screen = !CU && wkey != 0 && V.hvecs != nullptr;
    auto skip = [&](int j) { c.todo_key[j] = 0; c.n_dist++; c.n_skip++; };
    const float4* qv = reinterpret_cast<const float4*>(c.qvec);
    auto frow = [&](uint32_t y) { return reinterpret_cast<const float4*>(V.vecs + (size_t)y * V.ld); };
    auto hrow = [&](uint32_t y) { return reinterpret_cast<const uint2*>(V.hvecs + (size_t)y * V.ldh); };
    // A warp's later rows (j + W, j + 2W, ...) are pulled into L2 while it works on its first one: their loads then cost an L2
    // hit instead of a second and third HBM round trip on the expansion's critical path (one prefetch per 128-byte line, a lane
    // each; no registers held, unlike a second row in flight).  Under the screen the row read first is the fp16 one.
    const int lines = screen ? (V.ldh * 2 + 127) >> 7 : (V.ld * 4 + 127) >> 7;
    for (int j = warp + W; j < ntodo; j += W) {
        if (DEFER && (c.todo_id[j] & VisitedSet::MARK)) continue;
        const char* rowp = screen ? reinterpret_cast<const char*>(hrow(c.todo_id[j])) : reinterpret_cast<const char*>(frow(c.todo_id[j]));
        for (int l = lane; l < lines; l += 32) prefetch_l2(rowp + (size_t)l * 128);
    }
    for (int j = warp; j < ntodo; j += W) {
        uint32_t y = c.todo_id[j];
        if (DEFER && (y & VisitedSet::MARK)) { if (lane == 0) skip(j); continue; }
        float vnorm;
        if (screen) {
            float4 r = __ldg(V.hrec + y);
            float ah = warp_dot_h<NG>(hrow(y), qv, ng, lane);
            if (hs_screened_out(V, c, y, ah, r, wkey)) { if (lane == 0) skip(j); continue; }
            vnorm = r.x;
        } else vnorm = V.sim != SIM_DOT ? __ldg(V.norms + y) : 0.0f;
        float ab = warp_dot_t<NG>(frow(y), qv, ng, lane);
        if (lane == 0) finish(j, y, ab, vnorm);
    }
    if (warp == W - 1) cp_async_commit_wait_all();
    c.hop++;
    __syncthreads();
}

// Merge the keys todo_key[0, ntodo) of the expansion that just ran (0 = refused; the rest is in its record, c.last_hop()) into
// the sorted list A -> B (rank merge, no sort), keep at most `cap`.
// CU: entry 0 (the popped candidate) is dropped.  Afterwards A/B are swapped and s_len/s_best updated.
// LEAN: `len_io` / `best_io` carry the list length and the next candidate in registers (every thread computes them); no barrier
// after thread 0's update of the shared copies, which only code outside the hot loop reads (after a barrier of its own).
template <bool CU, bool LEAN = false>
__device__ inline void hs_merge(SearchCtx& c, int cap, int best, int ntodo, int* len_io = nullptr, int* best_io = nullptr) {
    HopRec& h = c.last_hop();
    int len = LEAN ? *len_io : *c.s_len;
    int first = CU ? 1 : 0;
    int my_best = INT_MAX;
    const uint64_t maxtodo = h.maxtodo;
    const int nadmit = h.nadmit;            // final since the expansion's last barrier
    int* const bn = &h.best_next;
    for (int t = threadIdx.x; t < len - first + ntodo; t += blockDim.x) {
        uint64_t key;
        int p;
        if (t < len - first) {
            int i = t + first;
            key = c.A[i];
            if (!CU && i == best) key &= ~1ull;  // the entry just expanded
            int shift = 0;
            if (key < maxtodo)                      // entries above every admitted key keep their position
                for (int j = 0; j < ntodo; ++j) shift += (c.todo_key[j] > key);
            p = t + shift;
        } else {
            int j = t - (len - first);
            key = c.todo_key[j];
            if (key == 0) continue;
            int r = 0;
            for (int jj = 0; jj < ntodo; ++jj) r += (c.todo_key[jj] > key);
            int lo = first, hi = len;  // count of old keys greater than key (A sorted descending)
            while (lo < hi) {
                int mid = (lo + hi) >> 1;
                if (c.A[mid] > key) lo = mid + 1; else hi = mid;
            }
            p = r + (lo - first);
        }
        if (p < cap) {
            c.B[p] = key;
            if (key & 1ull) my_best = min(my_best, p);
        } else if (CU && p == cap && (key | 1ull) > *c.s_dropped) {
            *c.s_dropped = key | 1ull;             // the best key the full list drops (one thread per merge)
        }
    }
    // first unexpanded entry of the merged list: one shared-memory atomic per warp, not per entry
    my_best = __reduce_min_sync(0xFFFFFFFFu, my_best);
    if ((threadIdx.x & 31) == 0 && my_best != INT_MAX) atomicMin(bn, my_best);
    __syncthreads();
    int nl = len - first + nadmit;
    const bool over = nl > cap;
    if (over) nl = cap;
    const int nb = *bn;
    if (threadIdx.x == 0) {
        *c.s_len = nl;
        *c.s_best = nb;
    }
    uint64_t* t = c.A; c.A = c.B; c.B = t;
    if (LEAN) { *len_io = nl; *best_io = nb; }
    else __syncthreads();
}

// hnsw/search.rs:242-304 on the list held in shared memory.
template <int NG, int W = HS_WARPS>
__device__ inline void hs_layer_search(const VecDev& V, const GraphDev& G, SearchCtx& c, int layer, int ef) {
    int best = *c.s_best, len = *c.s_len;     // published by hs_reseed (behind its barrier); from here on in registers
    while (best < len) {
        uint64_t ckey = c.A[best];
        hs_expand<false, NG, W, true>(V, G, c, key_id(ckey), layer, ef, 0.0f, best, len);
        hs_merge<false, true>(c, ef, best, c.last_hop().ntodo, &len, &best);
    }
}

// NodeFilter::passes (search.rs:147-170) for the popped candidate; warp 0 only, result broadcast by the caller.
__device__ inline bool hs_passes(const VecDev& V, const SearchArgs& a, uint32_t node, float score, const uint32_t* acc_ids,
                                 const float* acc_scores, int nacc, int lane) {
    uint32_t p = V.paragraph_of ? V.paragraph_of[node] : node;
    if (a.filter && !((a.filter[p >> 6] >> (p & 63)) & 1)) return false;
    if (!a.with_duplicates) {  // RepCounter: exact byte equality with an accepted vector (search.rs:388-412)
        const float4* x = reinterpret_cast<const float4*>(V.vecs + (size_t)node * V.ld);
        for (int i = 0; i < nacc; ++i) {
            if (__float_as_uint(acc_scores[i]) != __float_as_uint(score)) continue;  // equal bytes => equal score
            const float4* y = reinterpret_cast<const float4*>(V.vecs + (size_t)acc_ids[i] * V.ld);
            bool same = true;
            for (int g = lane; g < (V.ld >> 2); g += 32) {
                float4 u = x[g], w = y[g];
                same = same && __float_as_uint(u.x) == __float_as_uint(w.x) && __float_as_uint(u.y) == __float_as_uint(w.y) &&
                       __float_as_uint(u.z) == __float_as_uint(w.z) && __float_as_uint(u.w) == __float_as_uint(w.w);
            }
            if (__all_sync(0xFFFFFFFFu, same)) return false;
        }
    }
    if (a.multi_vector) {
        for (int i = 0; i < nacc; ++i) {
            uint32_t ap = V.paragraph_of ? V.paragraph_of[acc_ids[i]] : acc_ids[i];
            if (ap == p) return false;
        }
    }
    return true;
}

// Whether closest_up_nodes may run on the kept layer-0 set (DEFER below), for the list the dense layer-0 walk left in c.A and
// its visited set in c.vis; every thread, before hs_reseed's barrier.  Only hnsw_search_kernel<NG, true> asks, which the host
// launches only when every pop is accepted (dense_walk) and the fp16 copy is attached.
//   The walk ends only when every list entry has been expanded, so every neighbour of a list entry is in its set, and one outside
//   the final list was refused (s <= worst, a float comparison), screened out or evicted: its key is at most make_key(b, y) with
//   b = s_w, the last entry's score (the worst only improves), or +0 when s_w = -0 (a float refusal lets +0 pass a worst of -0).
//   When every pop is accepted (no filter, duplicates allowed, one vector per paragraph, no NaN in the list; a NaN score is
//   never admitted) closest_up_nodes pops at most k entries and expands at most k - 1.  When moreover A[k-1] scores above b, one
//   of A[0, k) outranks every such neighbour at each pop, so none is ever popped or affects a pop: it can be settled without its
//   row.  Each expansion adds at most s0 ids to the table and s0 - 1 entries to the list, so the last two tests keep the table
//   below its insert limit and the list within cu_cap: no overflow, and no truncation that could differ from the f32 walk's.
__device__ inline bool hs_can_defer(const VecDev& V, const GraphDev& G, const SearchCtx& c, const SearchArgs& a) {
    const int len = *c.s_len;
    if (len != a.ef0) return false;
    const float top = key_score(c.A[0]), sw = key_score(c.A[len - 1]);
    if (top != top || sw != sw) return false;
    const float b = __float_as_uint(sw) == 0x80000000u ? 0.0f : sw;
    const int grow = (a.k - 1) * G.s0;
    return (uint32_t)(c.A[a.k - 1] >> 32) > ordered_bits(b) && *c.s_hash_count + grow <= c.vis.limit && len + grow <= a.cu_cap;
}

// hnsw/search.rs:188-240.  Results go straight to out_ids/out_scores (already descending).
// DEFER: closest_up_nodes' visits are marked in the table, and `keep` (hs_can_defer) keeps the layer-0 walk's set under them, so a
// neighbour is new exactly when the reference's BitSet says so, and a new neighbour the layer-0 walk had visited is counted as a
// similarity settled without its row (as the screen's) and not listed.  Without `keep` the table is cleared first and no
// neighbour is settled, as without DEFER: one walk serves both cases, so the kernel carries one copy of it.
template <int NG, int W = HS_WARPS, bool DEFER = false>
__device__ inline int hs_closest_up(const VecDev& V, const GraphDev& G, SearchCtx& c, const SearchArgs& a, uint32_t* out_ids, float* out_scores,
                                    bool keep = false) {
    int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    hs_reseed<DEFER>(c, c.vis, keep);
    int nacc = 0;
    bool lost = false;
    while (true) {
        int len = *c.s_len;
        // The reference's candidate heap is unbounded; this list keeps its best cu_cap entries.  A dropped entry changes the result
        // only if it would be popped: when it outranks the list's head (or the list is empty) and passes min_score.  Counted once.
        const unsigned long long dropped = *c.s_dropped;
        if (!lost && dropped && (len == 0 || (c.A[0] | 1ull) < dropped) && !(key_score(dropped) < a.min_score)) {
            lost = true;
            if (threadIdx.x == 0) c.n_overflow += 1ull << 32;
        }
        if (len == 0) break;
        uint64_t ckey = c.A[0];
        float score = key_score(ckey);
        uint32_t node = key_id(ckey);
        if (score < a.min_score) break;  // 206
        __syncthreads();
        if (warp == 0) {
            bool pass = !(score != score) && hs_passes(V, a, node, score, out_ids, out_scores, nacc, lane);
            if (lane == 0) {
                *c.s_flag = pass;
                if (pass) { out_ids[nacc] = node; out_scores[nacc] = score; }
            }
        }
        __syncthreads();
        nacc += *c.s_flag;
        if (nacc == a.k) break;  // 214
        hs_expand<true, NG, W, false, DEFER>(V, G, c, node, 0, 0, a.min_score, 0);
        hs_merge<true>(c, a.cu_cap, 0, c.last_hop().ntodo);
    }
    return nacc;
}

// The tail of HnswSearcher::search for query q: closest_up_nodes on the list in c.A (search.rs:369-375), the final stable sort
// (search.rs:381) and the NIL padding of the outputs.  L0: closest_up_nodes may defer (hnsw_search_kernel<NG, true>).
template <int NG, int W = HS_WARPS, bool L0 = false>
__device__ inline void hs_emit_results(const VecDev& V, const GraphDev& G, SearchCtx& c, const SearchArgs& a, unsigned int q) {
    uint32_t* oi = a.out_ids + (size_t)q * a.k;
    float* os = a.out_scores + (size_t)q * a.k;
    int nacc = hs_closest_up<NG, W, L0>(V, G, c, a, oi, os, L0 && hs_can_defer(V, G, c, a));
    __syncthreads();
    // search.rs:381 `filtered_result.sort_by(|a, b| b.1.total_cmp(&a.1))`: stable, descending.
    // (closest_up_nodes can accept a late-found neighbour that outranks earlier results.)
    {
        uint32_t* tid = reinterpret_cast<uint32_t*>(c.B);
        float* tsc = reinterpret_cast<float*>(c.B) + a.k;
        for (int i = threadIdx.x; i < nacc; i += blockDim.x) { tid[i] = oi[i]; tsc[i] = os[i]; }
        __syncthreads();
        for (int i = threadIdx.x; i < nacc; i += blockDim.x) {
            uint32_t oi_bits = ordered_bits(tsc[i]);
            int r = 0;
            for (int j = 0; j < nacc; ++j) {
                uint32_t oj = ordered_bits(tsc[j]);
                r += (oj > oi_bits) || (oj == oi_bits && j < i);
            }
            oi[r] = tid[i];
            os[r] = tsc[i];
        }
        __syncthreads();
    }
    for (int i = nacc + threadIdx.x; i < a.k; i += blockDim.x) { oi[i] = NIL; os[i] = 0.0f; }
    if (threadIdx.x == 0) a.out_counts[q] = nacc;
}

// HS_WARPS = 8 warps per CTA, one row per warp in flight, 4 CTAs per SM (528 queries resident on 132 SMs).
// DEFER: closest_up_nodes may settle neighbours on the kept layer-0 set (hs_can_defer).  The host launches it only for queries
// whose pops are all accepted (no filter, duplicates allowed, one vector per paragraph) with the fp16 copy attached; every other
// walk, and the build, runs the kernel without it.
template <int NG, bool DEFER = false>
__global__ void __launch_bounds__(HS_THREADS, 4) hnsw_search_kernel(VecDev V, GraphDev G, SearchArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    SearchCtx c;
    hs_setup(c, a, smem, V.ld);
    int lane = threadIdx.x & 31;
    int ng = V.ld >> 2;

    unsigned q;
    while (hs_next_query(a, &q)) {
        const float* qsrc;
        uint32_t self = NIL;
        if (a.mode == 0) { qsrc = a.queries + (size_t)q * V.ld; c.qnorm = V.sim != SIM_DOT ? a.qnorms[q] : 0.0f; }
        else { self = a.nodes[q]; qsrc = V.vecs + (size_t)self * V.ld; c.qnorm = V.sim != SIM_DOT ? V.norms[self] : 0.0f; }
        for (int i = threadIdx.x; i < ng; i += blockDim.x) reinterpret_cast<float4*>(c.qvec)[i] = reinterpret_cast<const float4*>(qsrc)[i];
        __syncthreads();
        if (V.hvecs) c.qbound = hs_query_bound(c.qvec, V.ld);

        // entry point: similarity + single-entry list (search.rs:256-261)
        if (threadIdx.x < 32) {
            uint32_t ep = G.entry_node;
            float ab = warp_dot_t<NG>(reinterpret_cast<const float4*>(V.vecs + (size_t)ep * V.ld), reinterpret_cast<const float4*>(c.qvec), ng, lane);
            if (lane == 0) {
                c.A[0] = make_key(finish_similarity(V, ab, ep, c.qnorm), ep, 1);
                *c.s_len = 1;
                c.n_dist++;
            }
        }
        __syncthreads();

        int top = a.mode == 1 ? (int)G.level[self] : -1;
        for (int layer = (int)G.entry_layer; layer >= 0; --layer) {
            int ef;
            if (a.mode == 0) ef = layer == 0 ? a.ef0 : 1;
            else ef = layer <= top ? a.efC : 1;
            hs_reseed(c, c.vis);
            hs_layer_search<NG>(V, G, c, layer, ef);
            __syncthreads();
            if (a.mode == 1 && layer <= top && layer < HS_MAX_LAYERS) {
                int len = *c.s_len;
                uint64_t* dst = a.found + ((size_t)q * HS_MAX_LAYERS + layer) * a.efC;
                for (int i = threadIdx.x; i < len; i += blockDim.x) dst[i] = c.A[i];
                if (threadIdx.x == 0) a.found_count[(size_t)q * HS_MAX_LAYERS + layer] = len;
            }
            // next layer's entry points: the list as it stands -- a single node above the insertion
            // layers and for queries (ef == 1, search.rs:323-328), all efC results once inside the
            // node's layers (build.rs:142-150).  Scores to the same query do not change, so they are
            // not recomputed; hs_reseed() marks them unexpanded and seeds the visited set.
            __syncthreads();
        }

        // a node that rises above the current top layer (only on graph reuse, nidx_vec_extend_hnsw) finds nothing up there
        if (a.mode == 1 && threadIdx.x == 0)
            for (int layer = (int)G.entry_layer + 1; layer <= top && layer < HS_MAX_LAYERS; ++layer) a.found_count[(size_t)q * HS_MAX_LAYERS + layer] = 0;

        if (a.mode == 0) hs_emit_results<NG, HS_WARPS, DEFER>(V, G, c, a, q);
    }
    hs_flush_counters(c, a.counters);
    // [6] = f32 rows read for a similarity (n_skip lives in lane 0 of every warp, as n_dist)
    if (lane == 0 && c.n_dist) atomicAdd(&a.counters[6], c.n_dist - c.n_skip);
}

}  // namespace nidx
