// nidx_b200 — K5: RaBitQ 1-bit quantisation for nidx_vector (sm_90a).  First slice of SURVEY §8f rank 1:
// encoding, the estimator and the quantised exact scan; the quantised HNSW walk is the next step.
//
//   nidx/nidx_vector/src/vector_types/rabitq.rs:75-106    EncodedVector::encode    -> rabitq_encode_kernel
//   rabitq.rs:124-157                                     QueryVector::from_vector -> rabitq_query_kernel
//   rabitq.rs:166-218                                     QueryVector::dot / similarity (estimate, error) -> rabitq_estimate_kernel
//   rabitq.rs:222-244 + segment.rs:581-608                rerank_top over the brute-force candidates -> rabitq_rerank_kernel
// Only for Dot similarity and dimension % 64 == 0 (config.rs:170-173).  The code of a vector is the reference's
// vectors.quant record, [f32 dot_quant_original][u32 sum_bits][dim/8 sign bits], padded to a 16-byte stride in HBM:
// 104 -> 112 bytes at d = 768 against 3 072 bytes of f32, i.e. 27x less HBM traffic per candidate.
// All float arithmetic is written with *_rn intrinsics in the reference's order, so estimates and error bounds are
// bit-identical to the oracle's (oracle/rabitq.hpp).
#pragma once
#include "common.cuh"

namespace nidx {

constexpr float RABITQ_EPSILON = 1.9f;   // rabitq.rs:30
constexpr int RQ_MAX_WORDS32 = 128;      // d <= 4096

__host__ __device__ __forceinline__ int rabitq_stride(int d) { return ((d / 8 + 8) + 15) / 16 * 16; }

// one warp per vector
__global__ void rabitq_encode_kernel(VecDev V, unsigned char* __restrict__ codes, int stride) {
    __shared__ uint32_t bits[8][RQ_MAX_WORDS32];
    int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint64_t v = (uint64_t)blockIdx.x * 8 + warp;
    int nw = V.d / 32;
    for (int i = lane; i < nw; i += 32) bits[warp][i] = 0;
    __syncwarp();
    if (v >= V.n) return;
    float root_dim = __fsqrt_rn((float)V.d);
    float pos = __fdiv_rn(1.0f, root_dim), neg = __fdiv_rn(-1.0f, root_dim);
    const float4* a = reinterpret_cast<const float4*>(V.vecs + v * (size_t)V.ld);
    float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
    uint32_t nbits = 0;
    for (int g = lane; g < (V.d >> 2); g += 32) {   // lane-blocked order: dot_ordered(v, v_repr)
        float4 x = a[g];
        uint32_t nib = (x.x > 0.0f ? 1u : 0u) | (x.y > 0.0f ? 2u : 0u) | (x.z > 0.0f ? 4u : 0u) | (x.w > 0.0f ? 8u : 0u);
        ax = __fmaf_rn(x.x, x.x > 0.0f ? pos : neg, ax);
        ay = __fmaf_rn(x.y, x.y > 0.0f ? pos : neg, ay);
        az = __fmaf_rn(x.z, x.z > 0.0f ? pos : neg, az);
        aw = __fmaf_rn(x.w, x.w > 0.0f ? pos : neg, aw);
        nbits += __popc(nib);
        if (nib) atomicOr(&bits[warp][g >> 3], nib << ((g & 7) * 4));   // element i = 4g + c -> bit i % 32 of word i / 32
    }
    float dqo = butterfly_sum(__fadd_rn(__fadd_rn(ax, ay), __fadd_rn(az, aw)));
    for (int off = 16; off >= 1; off >>= 1) nbits += __shfl_xor_sync(0xFFFFFFFFu, nbits, off);
    __syncwarp();
    uint32_t* out = reinterpret_cast<uint32_t*>(codes + v * (size_t)stride);
    if (lane == 0) { out[0] = __float_as_uint(dqo); out[1] = nbits; }
    for (int i = lane; i < nw; i += 32) out[2 + i] = bits[warp][i];
    for (int i = 2 + nw + lane; i < stride / 4; i += 32) out[i] = 0;
}

struct RabitqQueryParams {
    float low, delta;
    uint32_t sum_quantized;
    uint32_t pad;
};

// one warp per query: 4 bit planes of the 4-bit scalar quantisation + (low, delta, sum_quantized)
__global__ void rabitq_query_kernel(const float* __restrict__ queries, int ld, int d, int nq, uint32_t* __restrict__ planes /* [nq][4][d/32] */,
                                    RabitqQueryParams* __restrict__ params) {
    __shared__ uint32_t bits[8][4][RQ_MAX_WORDS32];
    int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int q = blockIdx.x * 8 + warp;
    int nw = d / 32;
    for (int p = 0; p < 4; ++p)
        for (int i = lane; i < nw; i += 32) bits[warp][p][i] = 0;
    __syncwarp();
    if (q >= nq) return;
    const float* x = queries + (size_t)q * ld;
    float lo = x[0], hi = x[0];
    for (int i = lane; i < d; i += 32) { float v = x[i]; lo = v < lo ? v : lo; hi = v > hi ? v : hi; }
    for (int off = 16; off >= 1; off >>= 1) {
        float l2 = __shfl_xor_sync(0xFFFFFFFFu, lo, off), h2 = __shfl_xor_sync(0xFFFFFFFFu, hi, off);
        lo = l2 < lo ? l2 : lo;
        hi = h2 > hi ? h2 : hi;
    }
    hi = __fadd_rn(hi, 0.00001f);
    float delta = __fdiv_rn(__fsub_rn(hi, lo), 16.0f);
    uint32_t sum = 0;
    for (int i = lane; i < d; i += 32) {
        float f = __fdiv_rn(__fsub_rn(x[i], lo), delta);
        uint32_t wq = f >= 0.0f ? __float2uint_rz(f) : 0u;   // `as u64`
        sum += wq;
#pragma unroll
        for (int p = 0; p < 4; ++p)
            if ((wq >> p) & 1u) atomicOr(&bits[warp][p][i >> 5], 1u << (i & 31));
    }
    for (int off = 16; off >= 1; off >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, off);
    __syncwarp();
    for (int p = 0; p < 4; ++p)
        for (int i = lane; i < nw; i += 32) planes[((size_t)q * 4 + p) * nw + i] = bits[warp][p][i];
    if (lane == 0) params[q] = RabitqQueryParams{lo, delta, sum, 0};
}

// rabitq.rs:166-218 for one (query, vector): popcounts over 32-bit words (same sums as the reference's u64 words)
__device__ __forceinline__ void rabitq_similarity(const uint32_t* __restrict__ code, const uint32_t* __restrict__ planes, int nw, float low, float delta,
                                                  uint32_t sum_quantized, float root_dim, float& estimate, float& error) {
    uint32_t d0 = 0, d1 = 0, d2 = 0, d3 = 0;
    for (int i = 0; i < nw; ++i) {
        uint32_t s = code[2 + i];
        d0 += __popc(planes[i] & s);
        d1 += __popc(planes[nw + i] & s);
        d2 += __popc(planes[2 * nw + i] & s);
        d3 += __popc(planes[3 * nw + i] & s);
    }
    float dot = (float)(d0 + d1 * 2 + d2 * 4 + d3 * 8);
    float dqo = __uint_as_float(code[0]);
    float sum_bits = (float)code[1];
    float t1 = __fmul_rn(__fdiv_rn(__fmul_rn(2.0f, delta), root_dim), dot);
    float t2 = __fdiv_rn(__fmul_rn(__fmul_rn(2.0f, low), sum_bits), root_dim);
    float t3 = __fdiv_rn(__fmul_rn(delta, (float)sum_quantized), root_dim);
    float t4 = __fmul_rn(low, root_dim);
    float dqq = __fsub_rn(__fsub_rn(__fadd_rn(t1, t2), t3), t4);
    estimate = __fdiv_rn(dqq, dqo);
    float dd = __fmul_rn(dqo, dqo);
    error = __fdiv_rn(__fmul_rn(__fsqrt_rn(__fdiv_rn(__fsub_rn(1.0f, dd), dd)), RABITQ_EPSILON), root_dim);
}

// grid (vector chunks of 256, queries); one thread per vector; the query's planes in shared memory
__global__ void __launch_bounds__(256) rabitq_estimate_kernel(const unsigned char* __restrict__ codes, int stride, uint32_t n, int d,
                                                              const uint32_t* __restrict__ planes, const RabitqQueryParams* __restrict__ params,
                                                              float* __restrict__ est, float* __restrict__ err) {
    __shared__ uint32_t pl[4 * RQ_MAX_WORDS32];
    int q = blockIdx.y, nw = d / 32;
    for (int i = threadIdx.x; i < 4 * nw; i += blockDim.x) pl[i] = planes[(size_t)q * 4 * nw + i];
    __syncthreads();
    uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= n) return;
    RabitqQueryParams p = params[q];
    float e, r;
    rabitq_similarity(reinterpret_cast<const uint32_t*>(codes + (size_t)v * stride), pl, nw, p.low, p.delta, p.sum_quantized, __fsqrt_rn((float)d), e, r);
    est[(size_t)q * n + v] = e;
    err[(size_t)q * n + v] = r;
}

// rerank_top (rabitq.rs:222-244) over the candidates of the quantised exact scan (segment.rs:581-608), with the
// reference's SEQUENTIAL semantics: candidates in address order, the exact similarity is evaluated iff
// `best.len() < k || best_k < upper_bound` at that point of the scan.  A chunk of 4096 candidates is filtered in
// parallel against the state at the start of the chunk (a superset: best_k only grows), the survivors' exact
// similarities are computed by the warps, and one thread replays the reference's loop over the survivors.
constexpr int RR_THREADS = 256, RR_PER = 16, RR_CHUNK = RR_THREADS * RR_PER;

__host__ __device__ __forceinline__ size_t rr_smem_bytes(int ld, int k) { return (size_t)ld * 4 + (size_t)RR_CHUNK * 12 + (size_t)(k + 1) * 8 + 64; }

__global__ void __launch_bounds__(RR_THREADS) rabitq_rerank_kernel(VecDev V, const float* __restrict__ queries, const float* __restrict__ est,
                                                                   const float* __restrict__ err, const uint64_t* __restrict__ bits, float min_score,
                                                                   int k, uint32_t* __restrict__ out_ids, float* __restrict__ out_scores,
                                                                   int* __restrict__ out_counts, unsigned long long* __restrict__ exact_evals) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_warp_tot[8], s_total, s_hlen;
    __shared__ float s_best_k;
    unsigned char* p = smem;
    float* qv = reinterpret_cast<float*>(p); p += (size_t)V.ld * 4;
    uint64_t* heap = reinterpret_cast<uint64_t*>(p); p += (size_t)(k + 1) * 8;   // rank keys, descending
    uint32_t* surv_id = reinterpret_cast<uint32_t*>(p); p += RR_CHUNK * 4;
    float* surv_up = reinterpret_cast<float*>(p); p += RR_CHUNK * 4;
    float* surv_real = reinterpret_cast<float*>(p);
    int q = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int ng = V.ld >> 2;
    for (int i = threadIdx.x; i < ng; i += blockDim.x) reinterpret_cast<float4*>(qv)[i] = reinterpret_cast<const float4*>(queries + (size_t)q * V.ld)[i];
    if (threadIdx.x == 0) { s_hlen = 0; s_best_k = 0.0f; }
    __syncthreads();
    const float* qe = est + (size_t)q * V.n;
    const float* qr = err + (size_t)q * V.n;
    unsigned long long evals = 0;
    for (uint32_t c0 = 0; c0 < V.n; c0 += RR_CHUNK) {
        int hlen = s_hlen;
        float best_k = s_best_k;
        // phase 1: candidates of this thread (16 consecutive addresses) that the sequential scan could evaluate
        uint32_t mask = 0;
        float ups[RR_PER];
#pragma unroll
        for (int u = 0; u < RR_PER; ++u) {
            uint32_t v = c0 + threadIdx.x * RR_PER + u;
            ups[u] = 0.0f;
            if (v < V.n && (!bits || ((bits[v >> 6] >> (v & 63)) & 1))) {
                float up = __fadd_rn(qe[v], qr[v]);   // EstimatedScore::new_with_error
                ups[u] = up;
                if (up >= min_score && (hlen < k || best_k < up)) mask |= 1u << u;
            }
        }
        int cnt = __popc(mask), x = cnt;
        for (int off = 1; off < 32; off <<= 1) { int y = __shfl_up_sync(0xFFFFFFFFu, x, off); if (lane >= off) x += y; }
        if (lane == 31) s_warp_tot[warp] = x;
        __syncthreads();
        int base = 0;
        for (int w = 0; w < warp; ++w) base += s_warp_tot[w];
        if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < 8; ++w) t += s_warp_tot[w]; s_total = t; }
        int pos = base + x - cnt;
#pragma unroll
        for (int u = 0; u < RR_PER; ++u)
            if (mask & (1u << u)) { surv_id[pos] = c0 + threadIdx.x * RR_PER + u; surv_up[pos] = ups[u]; ++pos; }
        __syncthreads();
        int total = s_total;
        // phase 2: exact similarities of the survivors (Dot)
        for (int s = warp; s < total; s += RR_THREADS / 32) {
            float ab = warp_dot(reinterpret_cast<const float4*>(V.vecs + (size_t)surv_id[s] * V.ld), reinterpret_cast<const float4*>(qv), ng, lane);
            if (lane == 0) surv_real[s] = ab;
        }
        __syncthreads();
        // phase 3: the reference's loop, in order
        if (threadIdx.x == 0) {
            for (int s = 0; s < total; ++s) {
                if (hlen < k || best_k < surv_up[s]) {
                    ++evals;
                    float real = surv_real[s];
                    if (real >= min_score && (hlen < k || best_k < real)) {
                        uint64_t key = make_key(real, surv_id[s], 0);
                        int i = hlen;
                        while (i > 0 && heap[i - 1] < key) { heap[i] = heap[i - 1]; --i; }
                        heap[i] = key;
                        if (hlen < k) ++hlen;          // else the worst (last) entry falls off
                        best_k = key_score(heap[hlen - 1]);
                    }
                }
            }
            s_hlen = hlen;
            s_best_k = best_k;
        }
        __syncthreads();
    }
    int hlen = s_hlen;
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        out_ids[(size_t)q * k + i] = i < hlen ? key_id(heap[i]) : NIL;
        out_scores[(size_t)q * k + i] = i < hlen ? key_score(heap[i]) : 0.0f;
    }
    if (threadIdx.x == 0) {
        out_counts[q] = hlen;
        if (exact_evals) exact_evals[q] = evals;
    }
}

}  // namespace nidx
