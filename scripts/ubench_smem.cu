// Micro-benchmark of the shared-memory scatter primitives a BM25 accumulate can be built from (sm_90a).
// Not part of the product: it decides the design of bm25 (DESIGN.md §BM25): how many random-address
// accumulations per clock per SM do (a) ATOMS, (b) plain LDS+STS by an owning warp, (c) MATCH.ANY give?
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o /tmp/ubench_smem scripts/ubench_smem.cu && /tmp/ubench_smem
#include <cstdio>
#include <cstdint>
#include <cuda_runtime.h>

constexpr int WORDS = 12288;   // 48 KB of u32 accumulators per CTA
constexpr int ITERS = 2048;

__device__ __forceinline__ uint32_t next(uint32_t& s) { s ^= s << 13; s ^= s >> 17; s ^= s << 5; return s; }

template <int MODE>
__global__ void __launch_bounds__(256) k(uint32_t* gacc, uint32_t gwords, unsigned long long* out_cycles, uint32_t* sink) {
    extern __shared__ uint32_t acc[];
    unsigned char* tag = reinterpret_cast<unsigned char*>(acc + WORDS);
    for (int i = threadIdx.x; i < WORDS; i += blockDim.x) acc[i] = 0;
    __syncthreads();
    uint32_t s = (blockIdx.x * 256 + threadIdx.x) * 2654435761u + 12345u;
    uint32_t keep = 0;
    int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // warp-private sub-range for the ownership modes
    uint32_t wbase = warp * (WORDS / 8), wspan = WORDS / 8;
    long long t0 = clock64();
#pragma unroll 4
    for (int it = 0; it < ITERS; ++it) {
        uint32_t r = next(s);
        uint32_t idx = r % WORDS;
        uint32_t widx = wbase + (r % wspan);
        uint32_t v = (r >> 20) | 1u;
        if (MODE == 0) keep += idx + v;
        if (MODE == 1) atomicAdd(&acc[idx], v);
        if (MODE == 2) keep += atomicAdd(&acc[idx], v) == 0;
        if (MODE == 3) { uint32_t o = acc[widx]; acc[widx] = o + v; }
        if (MODE == 4) { unsigned m = __match_any_sync(0xFFFFFFFFu, widx); keep += m; }
        if (MODE == 5) atomicAdd(reinterpret_cast<float*>(acc) + idx, 1.0f);
        if (MODE == 6) atomicAdd(&gacc[(r ^ (r << 9)) % gwords], v);
        if (MODE == 7) {   // warp-owned range, lanes may collide: tag, verify, winners add, losers retry
            bool pending = true;
            while (__any_sync(0xFFFFFFFFu, pending)) {
                if (pending) tag[widx] = (unsigned char)lane;
                __syncwarp();
                bool win = pending && tag[widx] == (unsigned char)lane;
                if (win) { uint32_t o = acc[widx]; acc[widx] = o + v; pending = false; }
                __syncwarp();
            }
        }
        if (MODE == 8) {   // warp-owned range + MATCH.ANY: the lowest lane of every group adds the group's sum
            unsigned m = __match_any_sync(0xFFFFFFFFu, widx);
            if (m == (1u << lane)) { uint32_t o = acc[widx]; acc[widx] = o + v; }
            else {   // rare: serialise the group
                unsigned todo = m;
                while (todo) {
                    int l = __ffs(todo) - 1;
                    if (l == lane) { uint32_t o = acc[widx]; acc[widx] = o + v; }
                    __syncwarp(m);
                    todo &= todo - 1;
                }
            }
        }
        if (MODE == 9) { uint32_t o = acc[idx]; keep += o; }          // LDS only, random
        if (MODE == 10) { acc[idx] = v; }                             // STS only, random
    }
    long long t1 = clock64();
    if (lane == 0) atomicMax(out_cycles, (unsigned long long)(t1 - t0));
    if (keep == 0xDEADBEEF) sink[0] = keep;
    __syncthreads();
    if (threadIdx.x == 0) sink[1 + (blockIdx.x & 7)] = acc[blockIdx.x % WORDS];
}

template <int MODE>
void run(const char* name, int ctas_per_sm, int sms, uint32_t* gacc, uint32_t gwords, unsigned long long* d_cyc, uint32_t* sink, double base_cpw) {
    size_t smem = WORDS * 4 + WORDS;
    cudaFuncSetAttribute(k<MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    int grid = sms * ctas_per_sm;
    cudaMemset(d_cyc, 0, 8);
    k<MODE><<<grid, 256, smem>>>(gacc, gwords, d_cyc, sink);   // warm
    cudaMemset(d_cyc, 0, 8);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0); cudaEventCreate(&e1);
    cudaEventRecord(e0);
    k<MODE><<<grid, 256, smem>>>(gacc, gwords, d_cyc, sink);
    cudaEventRecord(e1);
    cudaError_t err = cudaDeviceSynchronize();
    float ms = 0;
    cudaEventElapsedTime(&ms, e0, e1);
    unsigned long long cyc = 0;
    cudaMemcpy(&cyc, d_cyc, 8, cudaMemcpyDeviceToHost);
    double warp_instr_per_sm = (double)ctas_per_sm * 8 * ITERS;
    double cpw = (double)cyc / warp_instr_per_sm;       // SM cycles per warp-level op (all warps of the SM interleaved)
    printf("%-34s ctas/sm=%d  %8.3f ms  max-cycles=%9llu  cycles/warp-op/SM=%7.2f  (minus index loop %6.2f)  ops/clk/SM=%6.2f  %s\n", name, ctas_per_sm, ms, cyc, cpw,
           cpw - base_cpw, 32.0 / cpw, err == cudaSuccess ? "" : cudaGetErrorString(err));
}

int main() {
    cudaDeviceProp p;
    cudaGetDeviceProperties(&p, 0);
    int sms = p.multiProcessorCount;
    printf("%s, %d SMs\n", p.name, sms);
    uint32_t gwords = 5u << 20;   // 20 MB
    uint32_t *gacc, *sink;
    unsigned long long* d_cyc;
    cudaMalloc(&gacc, (size_t)gwords * 4);
    cudaMemset(gacc, 0, (size_t)gwords * 4);
    cudaMalloc(&sink, 64);
    cudaMalloc(&d_cyc, 8);
    for (int c : {1, 2, 4}) {
        run<0>("index loop only", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<1>("ATOMS.ADD u32 (no return)", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<2>("ATOMS.ADD u32 (return used)", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<3>("LDS+IADD+STS warp-owned range", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<4>("MATCH.ANY only", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<5>("ATOMS.ADD f32", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<6>("RED.global u32 (20 MB, L2)", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<7>("tag-verify RMW", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<8>("MATCH.ANY + RMW", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<9>("LDS only", c, sms, gacc, gwords, d_cyc, sink, 0);
        run<10>("STS only", c, sms, gacc, gwords, d_cyc, sink, 0);
    }
    return 0;
}
