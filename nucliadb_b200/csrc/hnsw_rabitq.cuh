// nidx_b200 — K5b: the HNSW walk with a RaBitQ query (sm_90a).  The reference's production path for Dot indexes that
// carry 1-bit codes:
//   nidx/nidx_vector/src/segment.rs:506-513       the query becomes SearchVector::RabitQ when the store has vectors.quant
//   nidx/nidx_vector/src/hnsw/search.rs:306-383   HnswSearcher::search: the walk ranks by the ESTIMATE (similarity_upper_bound().score,
//                                                 segment.rs:339-348), layer 0 asks for min(k * 100, 2000) nodes (search.rs:332-337),
//                                                 rerank_top re-scores them exactly (rabitq.rs:222-244), closest_up_nodes and the
//                                                 final sort run on exact similarities (search.rs:355-381)
//   nidx/nidx_vector/src/vector_types/rabitq.rs:166-218   QueryVector::dot / similarity: 4 bit planes AND + POPC against the code
//
// One CTA per query (dynamic fetch, like hnsw_search_kernel, whose list / merge / closest_up code is reused).  What changes:
//   * an expansion costs 32 codes of 112 bytes instead of 32 rows of 3 KB, so it is one warp's work: lane = neighbour.  The lane
//     issues its code loads and its visited-set atomicCAS together -- codes of already visited neighbours are fetched for nothing
//     (3.6 KB per expansion), but the two dependent latencies become one;
//   * layer 0 keeps a 1 000-entry list (the reference's k * 100) and visits ~10-20 k nodes: the visited set of that layer is
//     an open-addressing table in GLOBAL memory (one slice per resident CTA, L2 resident); upper layers and closest_up_nodes
//     keep the shared-memory set;
//   * rerank_top keeps the reference's SEQUENTIAL semantics (a candidate is evaluated iff `best.len() < k || best_k < upper
//     bound` at its turn): chunks of 64 candidates are filtered against the state at the start of the chunk (a superset), their
//     exact similarities are computed by the eight warps, one thread replays the reference's loop.
// Estimates, error bounds and exact similarities are bit-identical to the oracle's (oracle/rabitq.hpp, hnsw_search_rabitq).
#pragma once
#include "hnsw_search.cuh"
#include "rabitq.cuh"

namespace nidx {

constexpr int RQ_RC = 64;   // rerank chunk
constexpr int RQ_TCH = 16;  // code chunks (16 bytes) whose query-plane words are kept transposed in shared memory (d <= 1984)

__host__ __device__ __forceinline__ size_t rq_smem_bytes(int ld, int d, int list_cap, int hash_bits, int k) {
    return hs_smem_bytes(ld, list_cap, hash_bits) + (size_t)4 * (d / 32) * 4 + (size_t)RQ_TCH * 64 + (size_t)RQ_RC * 12 + (size_t)(k + 1) * 8 + 64 + 16;
}

struct RqCtx {
    const uint32_t* planes;   // shared memory, [4][nw]
    const uint32_t* planes_t; // shared memory, [RQ_TCH][4 planes][4 words]: plane words by code chunk (16-byte aligned)
    int nw;
    float low, delta, root_dim;
    uint32_t sum_quantized;
    VisitedSet gvis;          // layer 0: this CTA's slice of the global visited table
    unsigned long long n_quant, n_rerank;
    unsigned long long n_gvis_overflow;   // hops whose insert the full global table refused
};

// rabitq.rs:166-218: the float tail of QueryVector::similarity from the integer dot product -> (estimate, error bound)
__device__ __forceinline__ void rq_finish(const RqCtx& r, uint32_t idot, uint32_t dqo_bits, uint32_t sum_bits, float& estimate, float& error) {
    float dot = (float)idot;
    float dqo = __uint_as_float(dqo_bits);
    float t1 = __fmul_rn(__fdiv_rn(__fmul_rn(2.0f, r.delta), r.root_dim), dot);
    float t2 = __fdiv_rn(__fmul_rn(__fmul_rn(2.0f, r.low), (float)sum_bits), r.root_dim);
    float t3 = __fdiv_rn(__fmul_rn(r.delta, (float)r.sum_quantized), r.root_dim);
    float t4 = __fmul_rn(r.low, r.root_dim);
    float dqq = __fsub_rn(__fsub_rn(__fadd_rn(t1, t2), t3), t4);
    estimate = __fdiv_rn(dqq, dqo);
    float dd = __fmul_rn(dqo, dqo);
    error = __fdiv_rn(__fmul_rn(__fsqrt_rn(__fdiv_rn(__fsub_rn(1.0f, dd), dd)), RABITQ_EPSILON), r.root_dim);
}

// weighted popcount of one 16-byte chunk of a code against the four query bit planes (words -2, -1 of chunk 0 are the header)
__device__ __forceinline__ uint32_t rq_chunk_dot(const RqCtx& r, int ch, uint4 w) {
    if (ch < RQ_TCH) {   // the four planes' words that face this chunk, contiguous (zero where the chunk holds the header or padding)
        const uint4* pt = reinterpret_cast<const uint4*>(r.planes_t) + ch * 4;
        const uint4 p0 = pt[0], p1 = pt[1], p2 = pt[2], p3 = pt[3];
        uint32_t d0 = __popc(p0.x & w.x) + __popc(p0.y & w.y) + __popc(p0.z & w.z) + __popc(p0.w & w.w);
        uint32_t d1 = __popc(p1.x & w.x) + __popc(p1.y & w.y) + __popc(p1.z & w.z) + __popc(p1.w & w.w);
        uint32_t d2 = __popc(p2.x & w.x) + __popc(p2.y & w.y) + __popc(p2.z & w.z) + __popc(p2.w & w.w);
        uint32_t d3 = __popc(p3.x & w.x) + __popc(p3.y & w.y) + __popc(p3.z & w.z) + __popc(p3.w & w.w);
        return d0 + d1 * 2 + d2 * 4 + d3 * 8;
    }
    uint32_t ws[4] = {w.x, w.y, w.z, w.w};
    uint32_t d0 = 0, d1 = 0, d2 = 0, d3 = 0;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
        int i = ch * 4 + t - 2;
        if (i >= 0 && i < r.nw) {
            uint32_t s = ws[t];
            d0 += __popc(r.planes[i] & s);
            d1 += __popc(r.planes[r.nw + i] & s);
            d2 += __popc(r.planes[2 * r.nw + i] & s);
            d3 += __popc(r.planes[3 * r.nw + i] & s);
        }
    }
    return d0 + d1 * 2 + d2 * 4 + d3 * 8;   // exact integer arithmetic: any summation order gives the reference's value
}

// One thread, one code (16-byte aligned, `stride` bytes, zero padded).  The chunk loads are issued eight at a time BEFORE any of
// them is consumed: a code costs one HBM latency, not one per 16 bytes.
__device__ __forceinline__ void rq_estimate(const RqCtx& r, const unsigned char* __restrict__ code, int stride, float& estimate, float& error) {
    const uint4* c4 = reinterpret_cast<const uint4*>(code);
    uint32_t idot = 0, dqo_bits = 0, sum_bits = 0;
    const int nchunks = stride >> 4;
    for (int c0 = 0; c0 < nchunks; c0 += 8) {
        uint4 w[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) w[j] = c0 + j < nchunks ? __ldg(c4 + c0 + j) : make_uint4(0, 0, 0, 0);
        if (c0 == 0) { dqo_bits = w[0].x; sum_bits = w[0].y; }
#pragma unroll
        for (int j = 0; j < 8; ++j) if (c0 + j < nchunks) idot += rq_chunk_dot(r, c0 + j, w[j]);
    }
    rq_finish(r, idot, dqo_bits, sum_bits, estimate, error);
}

// Expand `node` ranking by the estimate.  The whole CTA works on one adjacency row: EIGHT (8 warps) or FOUR (4 warps) LANES PER
// NEIGHBOUR, 32 neighbours per pass.  Lane j of a group loads 16-byte chunk j (j + 8, ...) of the neighbour's code -- the 112 bytes of a
// 768-d code arrive as seven adjacent 16-byte requests of one warp instruction -- and takes its weighted popcount; three
// shuffles add the eight partial sums (integers: exact in any order).  The group's first lane tests the visited set (global
// table: the atomicCAS and the code loads are in flight together, codes of visited neighbours are fetched for nothing) and
// finishes the estimate.  Admitted keys are compacted into todo_key[0 .. nadmit) (their order does not matter: hs_merge ranks
// by key).  The last warp first prefetches the adjacency row of the predicted next candidate (hs_prefetch_next) and publishes its
// list position (HopRec::pred) for the caller's nothing-admitted fast path.
// The hop's record collects the counts; thread 0 folds them after the barrier and resets the other record for the next hop, so no
// extra barrier is needed to reset them (hs_reseed resets both before a layer search's first hop).
template <bool GLOBAL_VIS, int W>
__device__ inline void rq_expand(const GraphDev& G, SearchCtx& c, const SearchArgs& a, RqCtx& r, uint32_t node, int layer, int ef, int best) {
    // LPN lanes per neighbour, so that the CTA covers one adjacency row of 32 per pass: 8 lanes (one 16-byte chunk each per 128 bytes
    // of code) with 8 warps, 4 lanes (two chunks each) with 4 warps -- the float tail of the estimate then runs once per warp for
    // eight neighbours instead of four.
    constexpr int LPN = W >= 8 ? 8 : 4;
    constexpr int CPL = 8 / LPN;         // chunks per lane and 128-byte block of code
    constexpr int NPG = W * 32 / LPN;    // neighbours per pass (32)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int sub = lane & (LPN - 1);
    const int stride = G.stride(layer);
    const unsigned cur = c.hop & 1u;
    HopRec& h = c.hops[cur];
    const VisitedSet& vis = GLOBAL_VIS ? r.gvis : c.vis;
    const int len = *c.s_len;
    const bool full = len >= ef;
    const float wscore = full ? key_score(c.A[len - 1]) : 0.0f;
    const int visited = *c.s_hash_count;       // stable during the expansion (thread 0 updates it after the barrier)
    const int nchunks = a.code_stride >> 4;
    if (warp == W - 1) {
        const int pred = hs_prefetch_next<false>(G, c, layer, best, len);
        if (lane == 0) h.pred = pred;
    }
    const uint32_t* prow = c.pref_row + cur * HS_MAX_ROW;
    const bool hit = c.pref_node[cur] == node;
    const uint32_t* row = G.row(node, layer);
    for (int e0 = 0; e0 < stride; e0 += NPG) {
        // every global request of the pass (code chunks, visited-set CAS) is in flight before anything is consumed
        const int e = e0 + (int)(threadIdx.x / LPN);
        uint32_t y = NIL;
        if (e < stride) y = hit ? prow[e] : __ldg(row + e);
        const bool valid = y != NIL;
        bool fresh = false, ov = false;
        const uint4* c4 = reinterpret_cast<const uint4*>(a.codes + (size_t)(valid ? y : 0) * a.code_stride);
        uint4 w[2][CPL];                 // the first 256 bytes of code (d <= 1984); longer codes loop below
        auto load_chunks = [&]() {
#pragma unroll
            for (int blk = 0; blk < 2; ++blk)
#pragma unroll
                for (int cc = 0; cc < CPL; ++cc) {
                    const int ch = blk * 8 + sub * CPL + cc;
                    w[blk][cc] = ch < nchunks ? __ldg(c4 + ch) : make_uint4(0, 0, 0, 0);
                }
        };
#pragma unroll
        for (int blk = 0; blk < 2; ++blk)
#pragma unroll
            for (int cc = 0; cc < CPL; ++cc) w[blk][cc] = make_uint4(0, 0, 0, 0);
        if (GLOBAL_VIS && valid) load_chunks();
        if (valid && sub == 0) fresh = vis.insert(y, visited, ov);
        if (!GLOBAL_VIS) {
            fresh = __shfl_sync(0xFFFFFFFFu, fresh, lane & ~(LPN - 1));
            if (fresh) load_chunks();
        }
        uint32_t idot = 0;
        if (valid && (GLOBAL_VIS || fresh)) {
#pragma unroll
            for (int blk = 0; blk < 2; ++blk)
#pragma unroll
                for (int cc = 0; cc < CPL; ++cc) {
                    const int ch = blk * 8 + sub * CPL + cc;
                    if (ch < nchunks) idot += rq_chunk_dot(r, ch, w[blk][cc]);
                }
            for (int base = 16; base < nchunks; base += 8)
#pragma unroll
                for (int cc = 0; cc < CPL; ++cc) {
                    const int ch = base + sub * CPL + cc;
                    if (ch < nchunks) idot += rq_chunk_dot(r, ch, __ldg(c4 + ch));
                }
        }
#pragma unroll
        for (int off = 1; off < LPN; off <<= 1) idot += __shfl_xor_sync(0xFFFFFFFFu, idot, off);
        if (sub == 0 && fresh) {
            float est, err;
            rq_finish(r, idot, w[0][0].x, w[0][0].y, est, err);       // chunk 0 starts with the code's header (dot_quant_original, sum_bits)
            uint64_t key = make_key(est, y, 1);
            if (!full || est > wscore) {                                  // layer_search (search.rs:286): a SCORE above the worst of a full list (a tie is refused whatever the ids)
                c.todo_key[atomicAdd(&h.nadmit, 1)] = key;
                atomicMax(&h.maxtodo, (unsigned long long)key);
            }
        }
        unsigned mf = __ballot_sync(0xFFFFFFFFu, sub == 0 && fresh);
        if (lane == 0 && mf) atomicAdd(&h.nfresh, __popc(mf));
        if (ov) h.overflow = 1;
    }
    if (warp == W - 1) {
        cp_async_commit_wait_all();
        if (GLOBAL_VIS) {
            // The predicted next node's adjacency row is in shared memory now: pull its neighbours' codes and visited-table slots
            // into L2 while this hop's merge runs (3.6 KB + 32 lines per hop; wasted when the prediction fails).
            __syncwarp();
            const uint32_t* nrow = c.pref_row + (cur ^ 1u) * HS_MAX_ROW;
            if (c.pref_node[cur ^ 1u] != NIL)
                for (int e = lane; e < stride; e += 32) {
                    uint32_t y2 = nrow[e];
                    if (y2 != NIL) {
                        const unsigned char* cp = a.codes + (size_t)y2 * a.code_stride;
                        prefetch_l2(cp);
                        if (((uintptr_t)cp & 127) + a.code_stride > 128) prefetch_l2(cp + 128 - ((uintptr_t)cp & 127));
                        prefetch_l2(&r.gvis.slots[r.gvis.slot(y2)]);
                    }
                }
        }
    }
    c.hop++;
    __syncthreads();
    if (threadIdx.x == 0) {
        *c.s_hash_count = visited + h.nfresh;
        c.n_expand++;
        r.n_quant += h.nfresh;
        if (h.overflow) { c.n_overflow++; if (GLOBAL_VIS) r.n_gvis_overflow++; }
        c.hops[cur ^ 1u].clear();
    }
}

template <bool GLOBAL_VIS, int W>
__device__ inline void rq_layer_search(const GraphDev& G, SearchCtx& c, const SearchArgs& a, RqCtx& r, int layer, int ef) {
    while (true) {
        int best = *c.s_best, len = *c.s_len;
        if (best >= len) break;
        uint64_t ckey = c.A[best];
        rq_expand<GLOBAL_VIS, W>(G, c, a, r, key_id(ckey), layer, ef, best);
        const HopRec& h = c.last_hop();
        if (h.nadmit == 0) {
            // nothing admitted (the common case once the list is full): the list only loses the expanded flag of `best`, and the
            // next candidate is the first unexpanded entry after it -- the one the prefetching warp has just located.
            if (threadIdx.x == 0) {    // (every thread read *s_best before rq_expand's barrier and this record is not touched until the next one)
                c.A[best] &= ~1ull;
                int pred = h.pred;
                *c.s_best = pred >= 0 ? pred : len;
            }
            __syncthreads();
            continue;
        }
        hs_merge<false>(c, ef, best, h.nadmit);
    }
}

// W warps per CTA: 8 (4 CTAs per SM, 592 queries resident) or 4 (7 CTAs per SM: a batch of 1024 is resident at once -- the walk is
// bound by the ~1 000 dependent hops of a query, so queries in flight, not warps per query, set the throughput).
template <int NG, int W = HS_WARPS>
__global__ void __launch_bounds__(W * 32, W == HS_WARPS ? 4 : 7) hnsw_rabitq_kernel(VecDev V, GraphDev G, SearchArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_wtot[RQ_RC / 32], s_total, s_hlen;
    __shared__ float s_best_k;
    SearchCtx c;
    RqCtx r;
    unsigned char* p = hs_setup(c, a, smem, V.ld);
    uint64_t* heap = reinterpret_cast<uint64_t*>(p); p += (size_t)(a.k + 1) * 8;          // rerank_top's `best`, rank keys, descending
    uint32_t* planes = reinterpret_cast<uint32_t*>(p); p += (size_t)4 * (V.d / 32) * 4;
    p = smem + (((size_t)(p - smem) + 15) & ~(size_t)15);
    uint32_t* planes_t = reinterpret_cast<uint32_t*>(p); p += (size_t)RQ_TCH * 64;
    uint32_t* surv_id = reinterpret_cast<uint32_t*>(p); p += RQ_RC * 4;
    float* surv_up = reinterpret_cast<float*>(p); p += RQ_RC * 4;
    float* surv_real = reinterpret_cast<float*>(p);
    r.planes = planes; r.planes_t = planes_t; r.nw = V.d / 32; r.root_dim = __fsqrt_rn((float)V.d);
    r.gvis.init(a.gvisited + ((size_t)blockIdx.x << a.gv_bits), a.gv_bits);
    r.n_quant = r.n_rerank = r.n_gvis_overflow = 0;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ng = V.ld >> 2;
    const RabitqQueryParams* qparams = reinterpret_cast<const RabitqQueryParams*>(a.qparams);

    unsigned q;
    while (hs_next_query(a, &q, a.nq)) {
        const float* qsrc = a.queries + (size_t)q * V.ld;
        for (int i = threadIdx.x; i < ng; i += blockDim.x) reinterpret_cast<float4*>(c.qvec)[i] = reinterpret_cast<const float4*>(qsrc)[i];
        for (int i = threadIdx.x; i < 4 * r.nw; i += blockDim.x) planes[i] = a.planes[(size_t)q * 4 * r.nw + i];
        for (int i = threadIdx.x; i < RQ_TCH * 16; i += blockDim.x) {      // [chunk][plane][t]: word 4 * chunk - 2 + t of the plane
            int ch = i >> 4, kpl = (i >> 2) & 3, wi = ch * 4 + (i & 3) - 2;
            planes_t[i] = (wi >= 0 && wi < r.nw) ? a.planes[(size_t)q * 4 * r.nw + kpl * r.nw + wi] : 0u;
        }
        RabitqQueryParams qp = qparams[q];
        r.low = qp.low; r.delta = qp.delta; r.sum_quantized = qp.sum_quantized;
        __syncthreads();

        // entry point: similarity_upper_bound(ep, query).score = the estimate (search.rs:256-261)
        if (threadIdx.x == 0) {
            uint32_t ep = G.entry_node;
            float est, err;
            rq_estimate(r, a.codes + (size_t)ep * a.code_stride, a.code_stride, est, err);
            c.A[0] = make_key(est, ep, 1);
            *c.s_len = 1;
            r.n_quant++;
        }
        __syncthreads();
        for (int layer = (int)G.entry_layer; layer > 0; --layer) {   // search.rs:321-327: one best node per upper layer
            hs_reseed(c, c.vis);
            rq_layer_search<false, W>(G, c, a, r, layer, 1);
            __syncthreads();
        }
        hs_reseed(c, r.gvis);
        rq_layer_search<true, W>(G, c, a, r, 0, a.last_k);             // search.rs:335-345
        __syncthreads();

        // ---- rerank_top (rabitq.rs:222-244) over the list, best estimate first ----
        const int len = *c.s_len;
        if (threadIdx.x == 0) { s_hlen = 0; s_best_k = 0.0f; }
        __syncthreads();
        for (int c0 = 0; c0 < len; c0 += RQ_RC) {
            int hlen = s_hlen;
            float best_k = s_best_k;
            bool pass = false;
            uint32_t id = NIL;
            float up = 0.0f;
            if (threadIdx.x < RQ_RC) {
                int i = c0 + (int)threadIdx.x;
                if (i < len) {
                    id = key_id(c.A[i]);
                    float est, err;
                    rq_estimate(r, a.codes + (size_t)id * a.code_stride, a.code_stride, est, err);
                    up = __fadd_rn(est, err);                               // EstimatedScore::new_with_error
                    pass = hlen < a.k || best_k < up;
                }
                unsigned m = __ballot_sync(0xFFFFFFFFu, pass);
                if (lane == 0) s_wtot[warp] = __popc(m);
            }
            __syncthreads();
            if (threadIdx.x < RQ_RC) {
                unsigned m = __ballot_sync(0xFFFFFFFFu, pass);
                int base = 0;
                for (int w = 0; w < warp; ++w) base += s_wtot[w];
                if (pass) { int pos = base + __popc(m & ((1u << lane) - 1)); surv_id[pos] = id; surv_up[pos] = up; }
                if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < RQ_RC / 32; ++w) t += s_wtot[w]; s_total = t; }
            }
            __syncthreads();
            int total = s_total;
            for (int s = warp; s < total; s += W) {                         // exact similarities (Dot) of the survivors
                float ab = warp_dot_t<NG>(reinterpret_cast<const float4*>(V.vecs + (size_t)surv_id[s] * V.ld), reinterpret_cast<const float4*>(c.qvec), ng, lane);
                if (lane == 0) { surv_real[s] = ab; c.n_dist++; }
            }
            __syncthreads();
            if (threadIdx.x == 0) {                                          // the reference's loop, in order
                for (int s = 0; s < total; ++s) {
                    if (hlen < a.k || best_k < surv_up[s]) {
                        r.n_rerank++;
                        float real = surv_real[s];
                        if (real >= a.min_score && (hlen < a.k || best_k < real)) {
                            uint64_t key = make_key(real, surv_id[s], 0);
                            int i = hlen;
                            while (i > 0 && heap[i - 1] < key) { heap[i] = heap[i - 1]; --i; }
                            heap[i] = key;
                            if (hlen < a.k) ++hlen;          // else the worst (last) entry falls off
                            best_k = key_score(heap[hlen - 1]);
                        }
                    }
                }
                s_hlen = hlen;
                s_best_k = best_k;
            }
            __syncthreads();
        }
        // reranked (exact, descending) -> the list; closest_up_nodes + final sort on exact similarities (search.rs:369-381)
        {
            int hlen = s_hlen;
            for (int i = threadIdx.x; i < hlen; i += blockDim.x) c.A[i] = heap[i];
            if (threadIdx.x == 0) *c.s_len = hlen;
            __syncthreads();
        }
        hs_emit_results<NG, W>(V, G, c, a, q);
    }
    hs_flush_counters(c, a.counters);
    if (threadIdx.x == 0) {
        if (r.n_quant) atomicAdd(&a.counters[4], r.n_quant);
        if (r.n_rerank) atomicAdd(&a.counters[5], r.n_rerank);
        if (r.n_gvis_overflow) atomicAdd(&a.counters[7], r.n_gvis_overflow);
    }
}

}  // namespace nidx
