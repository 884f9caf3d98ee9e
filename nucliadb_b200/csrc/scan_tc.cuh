// nidx_b200 — K1 (batched): exact-scan scores on the Hopper tensor cores (wgmma, sm_90a).
//
// A batch of queries against a block of stored vectors IS a dense GEMM (scores = Q · Vᵀ), the one place on the
// nidx_vector path where tensor cores apply (segment.rs:581-597 evaluated for many queries at once).  To stay
// inside the 1e-5 similarity tolerance with f32 inputs the product is computed as a 3xTF32 split:
//     x = x_hi + x_lo,  x_hi = x with the low 13 mantissa bits cleared (exact in TF32),  x_lo = x - x_hi (exact in f32)
//     q·v ≈ q_hi·v_hi + q_hi·v_lo + q_lo·v_hi            (the dropped q_lo·v_lo term is < 2^-22 relative)
// accumulated in f32 in registers.  The tensor core does not round its f32 accumulator like an f32 add does, so a single
// accumulator drifts at d = 768; the sum is spread over four accumulators -- three take the hi·hi products round-robin,
// one takes the two small cross terms -- that are added in f32 by the epilogue.  This path is only used on request
// (NIDX_B200_SCAN=tensor3x); large batches take the filter + refine path of scan_tc2.cuh.
//
// One CTA = one 128-query × TC_N-vector tile of the score matrix, two warpgroups of 64 query rows each.
//   * operands go global -> registers -> split hi/lo -> shared memory in the canonical K-major no-swizzle layout
//     (8-row × 16-byte core matrices):
//         byte offset(row r, 16-byte k-chunk c) = c * LBO + (r / 8) * 128 + (r % 8) * 16,   SBO = 128
//     LBO is padded by 16 bytes so that the 8 k-chunks a quarter-warp stores fall into different banks;
//   * each warpgroup issues wgmma.mma_async m64nTC_Nk8 tf32 (K = 8 per instruction), three per k-step (hi·hi, hi·lo,
//     lo·hi), into four register accumulators (4 x 32 f32 per thread);
//   * two shared-memory stages plus a register stage: the global loads of k-block i+1 are issued before the MMAs of
//     k-block i, its split + stores overlap those MMAs;
//   * epilogue: the accumulator fragments are summed, scaled (cosine) and written to scores[q][v].
#pragma once
#include "common.cuh"

namespace nidx {

constexpr int TC_M = 128;        // queries per tile (two warpgroups x wgmma M = 64)
constexpr int TC_N = 64;         // vectors per tile (wgmma N)
constexpr int TC_KB = 32;        // floats per k-block (8 chunks of 16 bytes = 4 MMA k-steps of K = 8)
constexpr int TC_THREADS = 256;
constexpr int TC_CHUNKS = TC_KB / 4;
constexpr uint32_t TC_LBO_A = (TC_M / 8) * 128 + 16;   // bytes between k-chunks of the A (query) tile, padded
constexpr uint32_t TC_LBO_B = (TC_N / 8) * 128 + 16;
constexpr uint32_t TC_A_BYTES = TC_CHUNKS * TC_LBO_A;  // one of {hi, lo} of one stage
constexpr uint32_t TC_B_BYTES = TC_CHUNKS * TC_LBO_B;
constexpr uint32_t TC_STAGE_BYTES = 2 * TC_A_BYTES + 2 * TC_B_BYTES;
constexpr size_t TC_SMEM_BYTES = 2 * TC_STAGE_BYTES + 1024;

// wgmma shared-memory matrix descriptor: start >> 4 [0,14), LBO >> 4 [16,30), SBO >> 4 [32,46), layout [62,64)
// (0 = no swizzle, 1 = 128-byte swizzle)
__device__ __forceinline__ uint64_t wg_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout) {
    return (uint64_t)((smem_addr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes & 0x3FFFFu) >> 4) << 16) | ((uint64_t)((sbo_bytes & 0x3FFFFu) >> 4) << 32) |
           ((uint64_t)layout << 62);
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// keeps the compiler from moving accesses of the accumulator registers across the asynchronous MMAs
__device__ __forceinline__ void wg_fence_regs(float (&d)[32]) {
#pragma unroll
    for (int i = 0; i < 32; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}
// d[64 x 64] (+)= A[64 x 8] · B[64 x 8]ᵀ, tf32 operands from shared memory, f32 accumulator fragment d[32] per thread:
// d[4j + e] holds row (warp % 4) * 16 + lane / 4 + 8 * (e / 2), column 8j + 2 (lane % 4) + e % 2.
__device__ __forceinline__ void wg_mma_64x64_tf32(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void mbar_init(uint64_t* mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(mbar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* mbar, uint32_t parity) {
    uint32_t addr = (uint32_t)__cvta_generic_to_shared(mbar);
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
                 :: "r"(addr), "r"(parity) : "memory");
}

// split x into the TF32-exact head and the f32 remainder
__device__ __forceinline__ void tc_split(float x, float& hi, float& lo) {
    hi = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
    lo = __fsub_rn(x, hi);
}

// A [rows][TC_KB] block (row stride ld floats, rows beyond n_rows read as zero) moves in two steps so that the
// global loads of the next k-block are in flight while the tensor core works: tc_fetch -> registers (4 consecutive
// rows x 8 chunks per warp: 128-byte coalesced reads), tc_store -> split hi/lo -> shared (conflict-free thanks to
// the padded LBO).
template <int ROWS>
__device__ __forceinline__ void tc_fetch(const float* __restrict__ src, uint64_t row0, uint64_t n_rows, int ld, int k0, float4 (&regs)[ROWS * TC_CHUNKS / TC_THREADS]) {
#pragma unroll
    for (int u = 0; u < ROWS * TC_CHUNKS / TC_THREADS; ++u) {
        int i = u * TC_THREADS + threadIdx.x;
        int r = i / TC_CHUNKS, c = i % TC_CHUNKS;
        regs[u] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (row0 + r < n_rows) regs[u] = ldg_stream(reinterpret_cast<const float4*>(src + (row0 + r) * (size_t)ld + k0) + c);
    }
}
template <int ROWS, uint32_t LBO>
__device__ __forceinline__ void tc_store(const float4 (&regs)[ROWS * TC_CHUNKS / TC_THREADS], unsigned char* hi_tile, unsigned char* lo_tile) {
#pragma unroll
    for (int u = 0; u < ROWS * TC_CHUNKS / TC_THREADS; ++u) {
        int i = u * TC_THREADS + threadIdx.x;
        int r = i / TC_CHUNKS, c = i % TC_CHUNKS;
        float4 v = regs[u], h, l;
        tc_split(v.x, h.x, l.x); tc_split(v.y, h.y, l.y); tc_split(v.z, h.z, l.z); tc_split(v.w, h.w, l.w);
        uint32_t off = (uint32_t)c * LBO + (uint32_t)(r >> 3) * 128u + (uint32_t)(r & 7) * 16u;
        *reinterpret_cast<float4*>(hi_tile + off) = h;
        *reinterpret_cast<float4*>(lo_tile + off) = l;
    }
}

// grid: (vector tiles, query tiles).  queries: [nq][ld] zero padded; ld % TC_KB == 0.
__global__ void __launch_bounds__(TC_THREADS, 1) scan_scores_tc_kernel(VecDev V, const float* __restrict__ queries, const float* __restrict__ qnorms, int nq,
                                                                       float* __restrict__ scores) {
    extern __shared__ __align__(128) unsigned char tc_smem[];
    unsigned char* smem = tc_smem;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = warp >> 2;
    uint64_t v0 = (uint64_t)blockIdx.x * TC_N;
    int q0 = blockIdx.y * TC_M;

    // acc[0..2]: hi·hi round-robin, acc[3]: the cross terms; all start at zero, so every MMA accumulates
    float acc[4][32];
#pragma unroll
    for (int g = 0; g < 4; ++g)
#pragma unroll
        for (int i = 0; i < 32; ++i) acc[g][i] = 0.0f;

    int n_kb = V.ld / TC_KB;
    uint32_t smem_u32 = (uint32_t)__cvta_generic_to_shared(smem);
    // register stages: k-blocks kb+1 and kb+2 are in flight while k-block kb is split, stored and multiplied
    float4 ra[2][TC_M * TC_CHUNKS / TC_THREADS], rb[2][TC_N * TC_CHUNKS / TC_THREADS];
    tc_fetch<TC_M>(queries, (uint64_t)q0, (uint64_t)nq, V.ld, 0, ra[0]);
    tc_fetch<TC_N>(V.vecs, v0, (uint64_t)V.n, V.ld, 0, rb[0]);
    if (n_kb > 1) {
        tc_fetch<TC_M>(queries, (uint64_t)q0, (uint64_t)nq, V.ld, TC_KB, ra[1]);
        tc_fetch<TC_N>(V.vecs, v0, (uint64_t)V.n, V.ld, TC_KB, rb[1]);
    }
    int step = 0;   // k-step counter: step % 3 picks the hi·hi accumulator
#pragma unroll 1
    for (int kb = 0; kb < n_kb; ++kb) {
        int st = kb & 1;
        // the tensor core must be done with this stage's previous contents (k-block kb - 2) in every warp
        wg_wait<1>();
        __syncthreads();
        unsigned char* stage = smem + (size_t)st * TC_STAGE_BYTES;
        unsigned char *a_hi = stage, *a_lo = stage + TC_A_BYTES, *b_hi = stage + 2 * TC_A_BYTES, *b_lo = stage + 2 * TC_A_BYTES + TC_B_BYTES;
        if (st == 0) { tc_store<TC_M, TC_LBO_A>(ra[0], a_hi, a_lo); tc_store<TC_N, TC_LBO_B>(rb[0], b_hi, b_lo); }
        else         { tc_store<TC_M, TC_LBO_A>(ra[1], a_hi, a_lo); tc_store<TC_N, TC_LBO_B>(rb[1], b_hi, b_lo); }
        if (kb + 2 < n_kb) {   // refill the register stage just consumed: two iterations to land
            if (st == 0) { tc_fetch<TC_M>(queries, (uint64_t)q0, (uint64_t)nq, V.ld, (kb + 2) * TC_KB, ra[0]); tc_fetch<TC_N>(V.vecs, v0, (uint64_t)V.n, V.ld, (kb + 2) * TC_KB, rb[0]); }
            else         { tc_fetch<TC_M>(queries, (uint64_t)q0, (uint64_t)nq, V.ld, (kb + 2) * TC_KB, ra[1]); tc_fetch<TC_N>(V.vecs, v0, (uint64_t)V.n, V.ld, (kb + 2) * TC_KB, rb[1]); }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy stores -> visible to the tensor core (async proxy)
        __syncthreads();
        uint32_t sbase = smem_u32 + (uint32_t)st * TC_STAGE_BYTES + (uint32_t)wg * (64 / 8) * 128;   // this warpgroup's 64 query rows
        uint32_t bbase = smem_u32 + (uint32_t)st * TC_STAGE_BYTES + 2 * TC_A_BYTES;
#pragma unroll
        for (int g = 0; g < 4; ++g) wg_fence_regs(acc[g]);
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < TC_KB / 8; ++ks, ++step) {   // K = 8 per instruction = 2 chunks
            uint32_t ka = (uint32_t)(2 * ks) * TC_LBO_A, kbo = (uint32_t)(2 * ks) * TC_LBO_B;
            uint64_t d_ahi = wg_desc(sbase + ka, TC_LBO_A, 128, 0), d_alo = wg_desc(sbase + TC_A_BYTES + ka, TC_LBO_A, 128, 0);
            uint64_t d_bhi = wg_desc(bbase + kbo, TC_LBO_B, 128, 0), d_blo = wg_desc(bbase + TC_B_BYTES + kbo, TC_LBO_B, 128, 0);
            wg_mma_64x64_tf32(acc[3], d_alo, d_bhi, 1);
            wg_mma_64x64_tf32(acc[3], d_ahi, d_blo, 1);
            int m = step % 3;   // warp-uniform: the accumulator is picked by a branch, registers cannot be indexed
            if (m == 0) wg_mma_64x64_tf32(acc[0], d_ahi, d_bhi, 1);
            else if (m == 1) wg_mma_64x64_tf32(acc[1], d_ahi, d_bhi, 1);
            else wg_mma_64x64_tf32(acc[2], d_ahi, d_bhi, 1);
        }
        wg_commit();
#pragma unroll
        for (int g = 0; g < 4; ++g) wg_fence_regs(acc[g]);
    }
    wg_wait<0>();
#pragma unroll
    for (int g = 0; g < 4; ++g) wg_fence_regs(acc[g]);

    // epilogue.  Cosine: ab * (1/|q|) * (1/|v|) with simsimd's edge cases (zero norms, ab == 0, clamp) -- two multiplies
    // per score instead of a division.
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        int qrow = q0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * h;
        if (qrow >= nq) continue;
        float qn = V.sim == SIM_COSINE ? qnorms[qrow] : 0.0f;
        float inv_qn = qn > 0.0f ? __frcp_rn(qn) : 0.0f;
        float* out = scores + (size_t)qrow * V.n;
#pragma unroll
        for (int j = 0; j < TC_N / 8; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                int i = 4 * j + 2 * h + e;
                uint64_t v = v0 + 8 * j + 2 * (lane & 3) + e;
                if (v >= V.n) continue;
                float ab = __fadd_rn(__fadd_rn(__fadd_rn(acc[0][i], acc[1][i]), acc[2][i]), acc[3][i]);
                float sc = ab;
                if (V.sim == SIM_COSINE) {
                    float vn = __ldg(V.norms + v);
                    float ivn = vn > 0.0f ? __frcp_rn(vn) : 0.0f;
                    if (inv_qn == 0.0f && ivn == 0.0f) sc = 1.0f;          // both norms zero: distance 0
                    else if (ab == 0.0f) sc = 0.0f;                       // distance 1
                    else {
                        float dist = __fsub_rn(1.0f, __fmul_rn(__fmul_rn(ab, inv_qn), ivn));
                        sc = __fsub_rn(1.0f, dist > 0.0f ? dist : 0.0f);
                    }
                }
                out[v] = sc;
            }
    }
}

}  // namespace nidx
