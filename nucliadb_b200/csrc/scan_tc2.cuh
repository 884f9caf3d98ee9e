// nidx_b200 — K1 (batched): the exact scan for a large query batch as FILTER (tensor cores) + REFINE (bit-exact).
//
// brute_force_search (nidx/nidx_vector/src/segment.rs:569-623) evaluated for a batch of queries is a dense GEMM,
// scores = Q · Vᵀ -- the one place on the nidx_vector path where the tensor cores apply.  The product is needed only to
// find each query's top-k, so it is computed ONCE in TF32 (f32 operands straight from the stored rows, f32 accumulation) as a
// filter with a rigorous error bound, never written to HBM, and only the few survivors are re-scored with the lane-blocked f32
// arithmetic of common.cuh.  Ids AND scores are therefore bit-identical to the small-batch kernel and to the oracle.
//
// The bound, for ld = the padded row length (the tensor cores' internal summation order and rounding are not documented, so the
// accumulation is taken as the worst case: a sequential f32 sum rounded toward zero, unit 2^-23; products of tf32 operands are
// exact in f32).  With S = sum |q_i v_i| <= |q| |v|:
//   operands   |tf32(q_i) tf32(v_i) - q_i v_i| <= (2^-9 + 2^-20) |q_i v_i|   (truncation to 10 mantissa bits: < 2^-10 per factor)
//   accumulate <= (ld - 1) 2^-23 / (1 - ld 2^-23) (1 + 2^-10)^2 S              (any summation tree of ld terms)
//   exact dot  <= dot_depth(ld) 2^-24 S <= 2^-18 S                             (the lane-blocked f32 score it is compared with)
//   cosine     the epilogue's four rn roundings (frcp_rn of both norms, two products) and the exact score's (division, two
//              subtractions) add < 2^-21; stored norms are within 2^-22 of |q|, |v|
//   subnormal  all of the above holds for normal f32 values only.  With |q|, |v| (cosine: every non-zero row) or |q|, max|v| (dot)
//              >= TC2_MIN_NORM = 2^-40, an operand, product or partial sum that is subnormal -- or flushed to zero, which the PTX
//              ISA leaves open for tf32 -- errs by < 2^-126 absolute, ld 2^-126 (1 + |q| + |v|) in all, < 2^-33 of |q| |v| at ld <= 4096
// Up to ld = 4096 all but the operand term stay below 65 2^-23, so |approx - exact| <= eps(ld) S with
//   eps(ld) = max(2.2e-3, 2^-9 + 2^-20 + (ld + 64) 2^-23)   (tc2_eps: 2.2e-3 up to ld = 1999, 2.45e-3 at 4096)
// as a cosine score, or eps(ld) |q| max|v| as a dot product.  tests/test_scan_filter_bound.py checks it against a model of the
// filter, and shows that 2.2e-3 alone fails at d = 4096.  Outside the bound the query or the segment takes the exact scan:
// a segment with a non-finite norm or (cosine) a non-zero row with |v| < TC2_MIN_NORM (api.cu, max_norm_kernel); a query with
// |q| or max|v| below TC2_MIN_NORM, |q| max|v| above 2^126 or not finite (so no tf32 sum or exact dot overflows), or a non-finite tau.
//   Let tau = the k-th largest APPROXIMATE score of a query over the
//   eligible vectors: every member of the true top-k has approx >= tau - 2 eps.  Each CTA keeps, per query row, the best
//   TC2_L approximate scores of ITS share of the vectors (a list in registers); the k best approximations overall are in
//   those lists (at most k - 1 entries of a share rank above any of them, and L >= k), so tau is known exactly from the
//   lists; survivors = list entries with approx >= tau - 2 eps.  A list that is full and whose smallest entry is still
//   >= tau - 2 eps may have dropped a survivor: OVERFLOW, the query is then scanned exactly (rare).
//
// scan_tc_filter_kernel: persistent CTAs; a CTA serves ONE 128-query block (slot s of grid / n_qblocks slots) and walks the
// vector chunks s, s + slots, ...; the CTAs of one slot run together and share every chunk (L2 reuse).  Warp-specialised:
//   warpgroup 0      TMA producer (one thread): cp.async.bulk.tensor (128-byte swizzle) of a 128 x 32-float query tile and a
//                    128 x 32-float vector tile per stage into a 4-stage mbarrier ring (32 KB per stage);
//   warpgroups 1, 2  consumers, 64 query rows each: wgmma.mma_async m64n128k8 tf32 from the stage (four per stage), f32
//                    accumulators in registers; every consumer warp releases the stage when its MMAs have read it.  The
//                    accumulators then go to a per-warpgroup score tile in shared memory and the same 128 threads run the
//                    epilogue with thread = (query row, column half): cosine scaling, eligibility bit, running top-L of the
//                    row's half in REGISTERS (unsorted + its minimum), fed through a per-row staging area in shared memory so
//                    that the (warp-wide) list update runs once per ~8-16 candidates of the busiest row, not once per column.
// scan_tc_refine_kernel: one CTA per query: overflow test, tau, survivors, exact re-scoring (one warp per survivor),
//   min_score, top-k -- or the exact scan of the whole segment for an overflowed query.
#pragma once
#include <cuda.h>

#include "common.cuh"
#include "topk.cuh"

namespace nidx {

constexpr int TC2_M = 128;            // queries per block (two consumer warpgroups x wgmma M = 64)
constexpr int TC2_N = 128;            // vectors per tile (wgmma N)
constexpr int TC2_KB = 32;            // floats per k-block = one 128-byte swizzle row
constexpr int TC2_STAGES = 4;
constexpr int TC2_TILES = 16;         // vector tiles per chunk
constexpr int TC2_CHUNK = TC2_N * TC2_TILES;   // 2048 vectors
constexpr int TC2_L = 24;             // candidates kept per (query, chunk)
constexpr int TC2_KMAX = 16;          // the filter path serves k <= TC2_KMAX
constexpr int TC2_CONSUMERS = 2;      // consumer warpgroups: query rows 64 c .. 64 c + 63
constexpr int TC2_THREADS = (1 + TC2_CONSUMERS) * 128;
constexpr int TC2_ROWS = TC2_M / TC2_CONSUMERS;   // query rows per consumer warpgroup
constexpr int TC2_TILE_LD = TC2_N + 1;           // score tile row stride (floats): a warp reading one column of 32 rows hits 32 banks
constexpr uint32_t TC2_A_BYTES = TC2_M * 128, TC2_B_BYTES = TC2_N * 128, TC2_STAGE_BYTES = TC2_A_BYTES + TC2_B_BYTES;
constexpr int TC2_STAGE_ROWS = 12;    // staged candidates per (query row, column half) between two merges into the register list
constexpr int TC2_LISTS = 2;          // candidate lists per query row and CTA (one per column half of every tile)
constexpr size_t TC2_SMEM_BYTES = 1024 /* alignment slack */ + (size_t)TC2_STAGES * TC2_STAGE_BYTES +
                                  (size_t)TC2_CONSUMERS * TC2_ROWS * TC2_TILE_LD * 4 /* score tiles */ + TC2_CONSUMERS * TC2_N * 4 /* 1/|v| */ +
                                  TC2_CONSUMERS * (TC2_N / 32) * 4 /* eligibility */ + (size_t)TC2_STAGE_ROWS * TC2_M * TC2_LISTS * 8 /* staging */ + 256;
static_assert(TC2_SMEM_BYTES <= 227 * 1024, "the filter kernel's shared memory exceeds a Hopper block's 227 KB");
constexpr float TC2_EPS = 2.2e-3f;
constexpr float TC2_MIN_NORM = 0x1p-40f;   // far from the subnormal range: see the header comment
constexpr int TC2_SURV_CAP = 512;     // survivors per query the refine kernel re-scores; more => exact scan
// eps(ld) of the header comment
__host__ __device__ __forceinline__ float tc2_eps(int ld) { return fmaxf(TC2_EPS, 0x1p-9f + 0x1p-20f + (float)(ld + 64) * 0x1p-23f); }

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
__device__ __forceinline__ void mbar_init(uint64_t* mbar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(mbar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* mbar, uint32_t parity) {
    uint32_t addr = (uint32_t)__cvta_generic_to_shared(mbar);
    asm volatile("{\n\t.reg .pred p;\n\tWAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra DONE_%=;\n\tbra WAIT_%=;\n\tDONE_%=:\n\t}"
                 :: "r"(addr), "r"(parity) : "memory");
}

__device__ __forceinline__ uint64_t tc2_desc(uint32_t smem_addr) {
    // K-major, SWIZZLE_128B: LBO unused (16 B), SBO = 8 rows x 128 B = 1024 B
    return wg_desc(smem_addr, 16, 1024, 1);
}
// d[64 x 128] (+)= A[64 x 8] · B[128 x 8]ᵀ, tf32 operands from shared memory, f32 accumulator fragment d[64] per thread:
// d[4j + e] (j = 0..15) holds row (warp % 4) * 16 + lane / 4 + 8 * (e / 2), column 8j + 2 (lane % 4) + e % 2.
__device__ __forceinline__ void wg_mma_64x128_tf32(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]),
          "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]),
          "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),
          "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]),
          "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
          "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate)
        : "memory");
}
__device__ __forceinline__ void wg_fence_regs64(float (&d)[64]) {
#pragma unroll
    for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i]) :: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* mbar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"((uint32_t)__cvta_generic_to_shared(mbar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* mbar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"((uint32_t)__cvta_generic_to_shared(mbar)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* mbar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 :: "r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(map), "r"(c0), "r"(c1), "r"((uint32_t)__cvta_generic_to_shared(mbar)) : "memory");
}

struct Tc2Args {
    int nq, n_qblocks, n_chunks, slots;   // slots = CTAs per query block (1 when there are more query blocks than CTAs)
    const float* qnorms;          // [nq] (cosine)
    const uint64_t* bits;         // eligibility (alive & filter) per vector, or nullptr
    float* cand_score;            // [nq][slots * TC2_LISTS][TC2_L] approx scores, unsorted, -inf padded
    uint32_t* cand_id;            // [nq][slots * TC2_LISTS][TC2_L]
    unsigned int* work_counter;
};

// The (query block, chunk) sequence of a CTA -- the same in both roles.  n_qblocks <= gridDim: CTA c serves block c % n_qblocks
// as slot c / n_qblocks (CTAs beyond n_qblocks * slots idle); else one slot and CTA c serves blocks c, c + gridDim, ...
struct Tc2Sched {
    int g0, gstride, slot, slots;
    __device__ Tc2Sched(const Tc2Args& a) {
        slots = a.slots;
        if (a.n_qblocks <= (int)gridDim.x) { g0 = (int)blockIdx.x % a.n_qblocks; slot = (int)blockIdx.x / a.n_qblocks; gstride = a.n_qblocks; if (slot >= slots) g0 = a.n_qblocks; }
        else { g0 = (int)blockIdx.x; slot = 0; gstride = (int)gridDim.x; }
    }
};

__global__ void __launch_bounds__(TC2_THREADS, 1) scan_tc_filter_kernel(const __grid_constant__ CUtensorMap map_q, const __grid_constant__ CUtensorMap map_v,
                                                                        VecDev V, Tc2Args a) {
    extern __shared__ unsigned char tc2_raw[];
    __shared__ uint64_t full[TC2_STAGES], empty[TC2_STAGES];
    unsigned char* smem = reinterpret_cast<unsigned char*>(((uintptr_t)tc2_raw + 1023) & ~(uintptr_t)1023);   // SWIZZLE_128B tiles: 1024-byte aligned
    unsigned char* stages = smem;
    float* tiles = reinterpret_cast<float*>(smem + (size_t)TC2_STAGES * TC2_STAGE_BYTES);         // [consumer][64][TC2_TILE_LD]
    float* inv_vn = tiles + TC2_CONSUMERS * TC2_ROWS * TC2_TILE_LD;                                // [consumer][128]
    uint32_t* elig = reinterpret_cast<uint32_t*>(inv_vn + TC2_CONSUMERS * TC2_N);                  // [consumer][4]
    float* stg_sc = reinterpret_cast<float*>(elig + TC2_CONSUMERS * (TC2_N / 32));                 // [TC2_STAGE_ROWS][2 * 128] staged scores ...
    uint32_t* stg_id = reinterpret_cast<uint32_t*>(stg_sc + TC2_STAGE_ROWS * TC2_M * TC2_LISTS);   // ... and ids of the epilogue threads
    const int warp = __shfl_sync(0xFFFFFFFFu, (int)threadIdx.x >> 5, 0), lane = threadIdx.x & 31;   // warp-uniform for the compiler
    const int n_kb = V.ld / TC2_KB;
    const Tc2Sched sch(a);

    if (threadIdx.x == 0) {
        for (int s = 0; s < TC2_STAGES; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], 4 * TC2_CONSUMERS); }   // one arrive per consumer warp
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (warp < 4) {
        // ===== TMA producer =====
        asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");   // registers go to the consumers: 128 x 40 + 256 x 232 <= 64 K
        if (threadIdx.x == 0) {
            uint32_t st = 0, ph = 0;
            for (int qb = sch.g0; qb < a.n_qblocks; qb += sch.gstride)
                for (int ch = sch.slot; ch < a.n_chunks; ch += sch.slots)
                    for (int t = 0; t < TC2_TILES; ++t) {
                        int v0 = ch * TC2_CHUNK + t * TC2_N;
                        if ((uint32_t)v0 >= V.n) break;
                        for (int kb = 0; kb < n_kb; ++kb) {
                            mbar_wait(&empty[st], ph ^ 1);
                            mbar_expect_tx(&full[st], TC2_STAGE_BYTES);
                            unsigned char* sa = stages + (size_t)st * TC2_STAGE_BYTES;
                            tma_load_2d(sa, &map_q, kb * TC2_KB, qb * TC2_M, &full[st]);
                            tma_load_2d(sa + TC2_A_BYTES, &map_v, kb * TC2_KB, v0, &full[st]);
                            if (++st == TC2_STAGES) { st = 0; ph ^= 1; }
                        }
                    }
        }
    } else {
        // ===== consumers: MMA, then epilogue with thread = (query row, column half) =====
        asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
        const int c = (warp >> 2) - 1;                          // consumer warpgroup: query rows 64 c .. 64 c + 63
        const int et = threadIdx.x - 128 * (c + 1);             // 0 .. 127
        const int rl = et & (TC2_ROWS - 1), half = et >> 6;     // row of this warpgroup's 64, column half of every tile
        const int row = c * TC2_ROWS + rl;                      // query row of the block
        const int srow = half * TC2_M + row;                    // this thread's column of the staging area
        float* tile = tiles + c * TC2_ROWS * TC2_TILE_LD;
        float* ivn_c = inv_vn + c * TC2_N;
        uint32_t* elig_c = elig + c * (TC2_N / 32);
        const uint32_t bar_id = 1 + c;                          // named barrier of this warpgroup's 128 threads
        const uint32_t sbase = (uint32_t)__cvta_generic_to_shared(stages);
        uint32_t st = 0, ph = 0;
        for (int qb = sch.g0; qb < a.n_qblocks; qb += sch.gstride) {
            int q = qb * TC2_M + row;
            float inv_qn = 1.0f;
            if (V.sim == SIM_COSINE) { float qn = q < a.nq ? a.qnorms[q] : 0.0f; inv_qn = qn > 0.0f ? __frcp_rn(qn) : 0.0f; }
            // the row's best TC2_L approximate scores over this CTA's share: unsorted, with the minimum and where it sits
            float ls[TC2_L];
            uint32_t li[TC2_L];
#pragma unroll
            for (int i = 0; i < TC2_L; ++i) { ls[i] = -INFINITY; li[i] = NIL; }
            int cnt = 0, minpos = 0, n_st = 0;
            float thr = -INFINITY;       // scores <= thr cannot enter the list (-inf until it is full)
            // Candidates that beat the row's threshold are first appended to a per-row staging area in shared memory ([slot][row]: the
            // lanes of a warp hit 32 different banks) and merged into the register list only when some row's area is nearly full: the
            // list update -- ~70 predicated instructions, executed by the whole warp whenever ANY lane needs it -- then runs a few
            // dozen times per row share instead of once per column.  Staged entries keep their column order and are re-tested against
            // the up-to-date threshold at merge time, so the list ends up exactly as if every column had been merged at once.
            auto merge_staged = [&]() {
                for (int t = 0; t < n_st; ++t) {
                    const float sc = stg_sc[t * (TC2_M * TC2_LISTS) + srow];
                    if (sc > thr) {
                        const uint32_t id = stg_id[t * (TC2_M * TC2_LISTS) + srow];
                        const int pos = cnt < TC2_L ? cnt : minpos;
#pragma unroll
                        for (int i = 0; i < TC2_L; ++i) if (i == pos) { ls[i] = sc; li[i] = id; }   // static indices: predicated moves
                        if (cnt < TC2_L) ++cnt;
                        if (cnt == TC2_L) {
                            float m = ls[0];
                            int mp = 0;
#pragma unroll
                            for (int i = 1; i < TC2_L; ++i) if (ls[i] < m) { m = ls[i]; mp = i; }
                            thr = m; minpos = mp;
                        }
                    }
                }
                n_st = 0;
            };
            for (int ch = sch.slot; ch < a.n_chunks; ch += sch.slots)
                for (int t = 0; t < TC2_TILES; ++t) {
                    int v0 = ch * TC2_CHUNK + t * TC2_N;
                    if ((uint32_t)v0 >= V.n) break;
                    // MMA: this warpgroup's 64 rows x 128 vectors over all k-blocks; a stage is released as soon as the MMAs
                    // issued after it have been waited for (one wgmma group in flight behind the newest)
                    float acc[64];
                    wg_fence_regs64(acc);
                    wg_fence();
                    uint32_t prev = 0;
                    for (int kb = 0; kb < n_kb; ++kb) {
                        mbar_wait(&full[st], ph);
                        uint32_t sa = sbase + st * TC2_STAGE_BYTES + (uint32_t)c * (TC2_ROWS * 128), sb = sbase + st * TC2_STAGE_BYTES + TC2_A_BYTES;
#pragma unroll
                        for (int ks = 0; ks < TC2_KB / 8; ++ks)    // K = 8 tf32 = 32 bytes inside the 128-byte swizzle row
                            wg_mma_64x128_tf32(acc, tc2_desc(sa + ks * 32), tc2_desc(sb + ks * 32), (kb | ks) != 0);
                        wg_commit();
                        if (kb > 0) {
                            wg_wait<1>();
                            if (lane == 0) mbar_arrive(&empty[prev]);
                        }
                        prev = st;
                        if (++st == TC2_STAGES) { st = 0; ph ^= 1; }
                    }
                    wg_wait<0>();
                    wg_fence_regs64(acc);
                    if (lane == 0) mbar_arrive(&empty[prev]);
                    // the previous tile's epilogue is done with the score tile and the column data
                    asm volatile("bar.sync %0, 128;" :: "r"(bar_id) : "memory");
#pragma unroll
                    for (int j = 0; j < TC2_N / 8; ++j)
#pragma unroll
                        for (int e = 0; e < 4; ++e)
                            tile[((warp & 3) * 16 + (lane >> 2) + 8 * (e >> 1)) * TC2_TILE_LD + 8 * j + 2 * (lane & 3) + (e & 1)] = acc[4 * j + e];
                    // per-tile column data: 1 / |v| (cosine) and the eligibility bits
                    {
                        uint32_t v = (uint32_t)v0 + et;
                        float ivn = 1.0f;
                        if (V.sim == SIM_COSINE) { float vn = v < V.n ? __ldg(V.norms + v) : 0.0f; ivn = vn > 0.0f ? __frcp_rn(vn) : 0.0f; }
                        ivn_c[et] = ivn;
                    }
                    if (et < TC2_N / 32) {
                        uint32_t w = 0xFFFFFFFFu;
                        uint32_t vb = (uint32_t)v0 + et * 32;
                        if (a.bits) w = vb < V.n ? reinterpret_cast<const uint32_t*>(a.bits)[vb >> 5] : 0u;
                        if (vb + 32 > V.n) w &= vb < V.n ? (0xFFFFFFFFu >> (32 - (V.n - vb))) : 0u;   // columns beyond the segment
                        elig_c[et] = w;
                    }
                    asm volatile("bar.sync %0, 128;" :: "r"(bar_id) : "memory");
                    for (int c0 = half * (TC2_N / TC2_LISTS); c0 < (half + 1) * (TC2_N / TC2_LISTS); c0 += 32) {
                        const uint32_t ew = q < a.nq ? elig_c[c0 >> 5] : 0u;
                        const float* trow = tile + rl * TC2_TILE_LD + c0;
#pragma unroll
                        for (int j = 0; j < 32; ++j) {
                            float sc = trow[j];
                            if (V.sim == SIM_COSINE) sc = sc * inv_qn * ivn_c[c0 + j];
                            const bool pass = ((ew >> j) & 1u) && sc > thr;
                            if (pass) {                                   // predicated stores: the row's staging area, in column order
                                stg_sc[n_st * (TC2_M * TC2_LISTS) + srow] = sc;
                                stg_id[n_st * (TC2_M * TC2_LISTS) + srow] = (uint32_t)v0 + c0 + j;
                                ++n_st;
                            }
                            if ((j & 3) == 3 && __any_sync(0xFFFFFFFFu, n_st > TC2_STAGE_ROWS - 4)) merge_staged();
                        }
                    }
                }
            merge_staged();
            if (q < a.nq) {
                float* os = a.cand_score + (((size_t)q * a.slots + sch.slot) * TC2_LISTS + half) * TC2_L;
                uint32_t* oi = a.cand_id + (((size_t)q * a.slots + sch.slot) * TC2_LISTS + half) * TC2_L;
#pragma unroll
                for (int i = 0; i < TC2_L; ++i) { os[i] = ls[i]; oi[i] = li[i]; }
            }
        }
    }
}

// One CTA per query.  dynamic smem: ld floats (query) + cap keys (top-k buffer) + survivors.
__host__ __device__ __forceinline__ size_t tc2_refine_smem(int ld, int cap) { return (size_t)ld * 4 + (size_t)cap * 8 + (size_t)TC2_SURV_CAP * 4 + 64; }

__global__ void __launch_bounds__(256) scan_tc_refine_kernel(VecDev V, const float* __restrict__ queries, const float* __restrict__ qnorms, int n_lists,
                                                             const float* __restrict__ cand_score, const uint32_t* __restrict__ cand_id,
                                                             const uint64_t* __restrict__ bits, float max_vnorm, float min_score, int k, int cap,
                                                             uint32_t* __restrict__ out_ids, float* __restrict__ out_scores, int* __restrict__ out_counts,
                                                             unsigned long long* __restrict__ stats /* [0] survivors [1] overflowed queries */) {
    extern __shared__ __align__(16) unsigned char rf_smem[];
    __shared__ int tk_count;
    __shared__ uint64_t tk_thr;
    __shared__ int s_overflow, s_nsurv;
    float* qv = reinterpret_cast<float*>(rf_smem);
    uint64_t* tk_buf = reinterpret_cast<uint64_t*>(rf_smem + (size_t)V.ld * 4);
    uint32_t* surv = reinterpret_cast<uint32_t*>(tk_buf + cap);
    const int q = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ng = V.ld >> 2;
    for (int i = threadIdx.x; i < ng; i += blockDim.x) reinterpret_cast<float4*>(qv)[i] = reinterpret_cast<const float4*>(queries + (size_t)q * V.ld)[i];
    const float qn = V.sim == SIM_COSINE ? qnorms[q] : 0.0f;
    // eps of this query: cosine scores are scale free; a dot product scales with both norms
    float eps = tc2_eps(V.ld), qabs = qn;
    if (V.sim != SIM_COSINE) {
        float s = 0.0f;
        for (int i = lane; i < V.d; i += 32) { float x = queries[(size_t)q * V.ld + i]; s += x * x; }
        for (int off = 16; off >= 1; off >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, off);
        qabs = sqrtf(s);
        eps *= qabs * max_vnorm;
    }
    const float margin = 2.0f * eps;
    // a query outside the bound (header comment) is scanned exactly: NaN / inf elements, a tiny query or segment (subnormal
    // products), or sums that may overflow
    const bool out_of_bound = !(qabs >= TC2_MIN_NORM) || !(max_vnorm >= TC2_MIN_NORM) || !(qabs * max_vnorm <= 0x1p126f);
    if (threadIdx.x == 0) { s_overflow = out_of_bound ? 1 : 0; s_nsurv = 0; }
    BlockTopK tk;
    tk.init(tk_buf, &tk_count, &tk_thr, k, cap);
    const float* cs = cand_score + (size_t)q * n_lists * TC2_L;
    const uint32_t* ci = cand_id + (size_t)q * n_lists * TC2_L;
    // 1. tau = k-th largest approximate score among all candidates
    const int total = n_lists * TC2_L;
    for (int base = 0; base < total; base += blockDim.x) {
        int i = base + threadIdx.x;
        uint64_t key = 0;
        if (i < total && ci[i] != NIL) key = make_key(cs[i], (uint32_t)i, 0);
        tk.offer(key);
    }
    int c = tk.finish();
    const float tau = c >= k ? key_score(tk_buf[k - 1]) : -INFINITY;
    if (threadIdx.x == 0 && (tau == INFINITY || isnan(tau - margin))) s_overflow = 1;
    __syncthreads();
    // 2. overflow test per list: full (no NIL entry), and its smallest entry still within the margin of tau
    for (int l = threadIdx.x; l < n_lists; l += blockDim.x) {
        float mn = INFINITY;
        bool full = true;
        for (int i = 0; i < TC2_L; ++i) { full &= ci[(size_t)l * TC2_L + i] != NIL; mn = fminf(mn, cs[(size_t)l * TC2_L + i]); }
        if (full && mn >= tau - margin) s_overflow = 1;
    }
    // 3. survivors
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
        if (ci[i] != NIL && cs[i] >= tau - margin) {
            int pos = atomicAdd(&s_nsurv, 1);
            if (pos < TC2_SURV_CAP) surv[pos] = ci[i];
        }
    }
    __syncthreads();
    const bool exact_all = s_overflow || s_nsurv > TC2_SURV_CAP;
    const int nsurv = exact_all ? (int)V.n : s_nsurv;
    if (threadIdx.x == 0 && stats) { atomicAdd(&stats[0], (unsigned long long)(exact_all ? 0 : nsurv)); if (exact_all) atomicAdd(&stats[1], 1ull); }
    // 4. exact scores (lane-blocked arithmetic: bit-identical to scan_scores_kernel), min_score, top-k
    tk.init(tk_buf, &tk_count, &tk_thr, k, cap);
    for (int base = 0; base < nsurv; base += blockDim.x) {
        // one warp per candidate, 8 candidates per round, keys offered by lane 0 of each warp in a full-block round
        uint64_t mykey = 0;
        for (int w8 = 0; w8 < 32; ++w8) {            // 32 sub-rounds x 8 warps = 256 candidates per offer round
            int i = base + w8 * 8 + warp;
            uint64_t key = 0;
            if (i < nsurv) {
                uint32_t v = exact_all ? (uint32_t)i : surv[i];
                bool ok = !exact_all || !bits || ((bits[v >> 6] >> (v & 63)) & 1);
                if (ok) {
                    float ab = warp_dot(reinterpret_cast<const float4*>(V.vecs + (size_t)v * V.ld), reinterpret_cast<const float4*>(qv), ng, lane);
                    float s = sim_from_parts(V.sim, ab, V.norms[v], qn);
                    if (s >= min_score) key = make_key(s, v, 0);
                }
            }
            if (lane == w8) mykey = key;             // lane w8 of warp `warp` carries candidate base + w8 * 8 + warp
        }
        tk.offer(mykey);
    }
    c = tk.finish();
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        out_ids[(size_t)q * k + i] = i < c ? key_id(tk_buf[i]) : NIL;
        out_scores[(size_t)q * k + i] = i < c ? key_score(tk_buf[i]) : 0.0f;
    }
    if (threadIdx.x == 0 && out_counts) out_counts[q] = c;
}

}  // namespace nidx
