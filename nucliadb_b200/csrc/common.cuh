// nidx_b200 — shared device helpers (sm_90a).
//
// The similarity arithmetic of nidx_vector (vector_types/dense_f32.rs:29-39 over simsimd) is done
// in ONE fixed summation order everywhere ("lane-blocked", DESIGN.md §kernels): lane l of a warp
// owns the float4 groups g with g % 32 == l, visited in increasing g, four fused-multiply-add
// accumulators per lane (one per component), lane value (ax+ay)+(az+aw), xor-butterfly 16,8,4,2,1.
// All arithmetic uses the *_rn intrinsics so nvcc can neither contract nor reassociate it.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace nidx {

constexpr uint32_t NIL = 0xFFFFFFFFu;
constexpr int SIM_DOT = 0, SIM_COSINE = 1, SIM_L2 = 2;   // L2: an extension (the reference has Dot and Cosine only, config.rs:33-37)

struct VecDev {
    const float* vecs;    // [n][ld] f32, ld % 4 == 0, rows 16-byte aligned, zero padded
    const float* norms;   // [n] sqrt(dot_ordered(v, v)); read for cosine and L2
    const uint32_t* paragraph_of;  // [n] or nullptr (identity)
    uint32_t n;
    int d, ld, sim;
    // The HNSW walk's screening copy (hs_half_kernel), or nullptr: the walk then reads every neighbour's f32 row.
    const __half* hvecs;  // [n][ldh] fp16(v * 2^e_row), ldh = ld rounded up to 8 (16-byte rows), zero padded
    const float4* hrec;   // [n] {norms[i], 2^-e_row, err_q, err_abs}: |screen dot - exact dot| <= |q| * err_q + err_abs
    int ldh;
};

// Rounding depth of one product term in the lane-blocked dot (warp_dot / warp_dot_t / warp_dot_h): ceil(ngroups / 32) fused
// multiply-adds in its lane's accumulator, two adds combining the four accumulators, five butterfly adds.
__host__ __device__ __forceinline__ int dot_depth(int ld) { return (ld / 4 + 31) / 32 + 7; }

struct GraphDev {
    uint32_t n;
    int M, M0, s0, su;
    const uint8_t* level;
    uint32_t entry_node, entry_layer;
    uint32_t* adj0; float* w0;           // [n][s0]
    const uint64_t* upper_off;           // [n]
    uint32_t* adjU; float* wU;           // [rows][su]
    __device__ __forceinline__ uint32_t* row(uint32_t node, int layer) const {
        return layer == 0 ? adj0 + (size_t)node * s0 : adjU + (upper_off[node] + (uint64_t)(layer - 1)) * su;
    }
    __device__ __forceinline__ float* wrow(uint32_t node, int layer) const {
        return layer == 0 ? w0 + (size_t)node * s0 : wU + (upper_off[node] + (uint64_t)(layer - 1)) * su;
    }
    __device__ __forceinline__ int stride(int layer) const { return layer == 0 ? s0 : su; }
    __device__ __forceinline__ int mmax(int layer) const { return layer == 0 ? M0 : M; }
};

// f32::total_cmp-compatible monotone key (hnsw/search.rs:90-93).
__device__ __forceinline__ uint32_t ordered_bits(float f) {
    uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float from_ordered_bits(uint32_t o) {
    uint32_t u = (o & 0x80000000u) ? (o & 0x7FFFFFFFu) : ~o;
    return __uint_as_float(u);
}
// 64-bit rank key: higher score first, then lower id first; bit 0 is a free flag
// ("not yet expanded" in the search lists).  ids < 2^31.
__device__ __forceinline__ uint64_t make_key(float score, uint32_t id, uint32_t flag) {
    return ((uint64_t)ordered_bits(score) << 32) | (uint64_t)(((0x7FFFFFFFu - id) << 1) | (flag & 1u));
}
__device__ __forceinline__ uint32_t key_id(uint64_t k) { return 0x7FFFFFFFu - ((uint32_t)k >> 1); }
__device__ __forceinline__ float key_score(uint64_t k) { return from_ordered_bits((uint32_t)(k >> 32)); }
__device__ __forceinline__ uint32_t key_flag(uint64_t k) { return (uint32_t)k & 1u; }

__device__ __forceinline__ float4 ldg_stream(const float4* p) {
    float4 r;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}

__device__ __forceinline__ float butterfly_sum(float v) {
#pragma unroll
    for (int off = 16; off >= 1; off >>= 1) v = __fadd_rn(v, __shfl_xor_sync(0xFFFFFFFFu, v, off));
    return v;
}

// Lane-blocked dot of a global row `a` (streamed) with `b` (shared or global), both [ngroups] float4.
// All 32 lanes of the warp call this; every lane returns the full sum.
__device__ __forceinline__ float warp_dot(const float4* __restrict__ a, const float4* __restrict__ b, int ngroups, int lane) {
    float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
    for (int base = 0; base < ngroups; base += 256) {
        float4 va[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            int g = base + j * 32 + lane;
            va[j] = g < ngroups ? ldg_stream(a + g) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            int g = base + j * 32 + lane;
            if (g < ngroups) {
                float4 vb = b[g];
                ax = __fmaf_rn(va[j].x, vb.x, ax);
                ay = __fmaf_rn(va[j].y, vb.y, ay);
                az = __fmaf_rn(va[j].z, vb.z, az);
                aw = __fmaf_rn(va[j].w, vb.w, aw);
            }
        }
    }
    return butterfly_sum(__fadd_rn(__fadd_rn(ax, ay), __fadd_rn(az, aw)));
}

// Same arithmetic, compile-time row length: NG float4 groups per lane (ld == NG * 128 floats).  No
// predication, immediate load offsets; NG == 0 falls back to the run-time loop above.
template <int NG>
__device__ __forceinline__ float warp_dot_t(const float4* __restrict__ a, const float4* __restrict__ b, int ngroups, int lane) {
    if constexpr (NG == 0) {
        return warp_dot(a, b, ngroups, lane);
    } else {
        float4 va[NG];
#pragma unroll
        for (int j = 0; j < NG; ++j) va[j] = ldg_stream(a + j * 32 + lane);
        float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
#pragma unroll
        for (int j = 0; j < NG; ++j) {
            float4 vb = b[j * 32 + lane];
            ax = __fmaf_rn(va[j].x, vb.x, ax);
            ay = __fmaf_rn(va[j].y, vb.y, ay);
            az = __fmaf_rn(va[j].z, vb.z, az);
            aw = __fmaf_rn(va[j].w, vb.w, aw);
        }
        return butterfly_sum(__fadd_rn(__fadd_rn(ax, ay), __fadd_rn(az, aw)));
    }
}

__device__ __forceinline__ uint2 ldg_stream2(const uint2* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}

// warp_dot_t's lane-blocked order over an fp16 row `a` ([ngroups] groups of four halves, 8-byte loads, widened to f32 in
// registers -- exactly) against the f32 `b`: the same dot_depth(), so the same rounding-error bound as the f32 dot.
template <int NG>
__device__ __forceinline__ float warp_dot_h(const uint2* __restrict__ a, const float4* __restrict__ b, int ngroups, int lane) {
    float ax = 0.f, ay = 0.f, az = 0.f, aw = 0.f;
    auto acc = [&](uint2 h, float4 vb) {
        float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&h.x)), hi = __half22float2(*reinterpret_cast<const __half2*>(&h.y));
        ax = __fmaf_rn(lo.x, vb.x, ax);
        ay = __fmaf_rn(lo.y, vb.y, ay);
        az = __fmaf_rn(hi.x, vb.z, az);
        aw = __fmaf_rn(hi.y, vb.w, aw);
    };
    if constexpr (NG == 0) {
        for (int g = lane; g < ngroups; g += 32) acc(ldg_stream2(a + g), b[g]);
    } else {
        uint2 va[NG];
#pragma unroll
        for (int j = 0; j < NG; ++j) va[j] = ldg_stream2(a + j * 32 + lane);
#pragma unroll
        for (int j = 0; j < NG; ++j) acc(va[j], b[j * 32 + lane]);
    }
    return butterfly_sum(__fadd_rn(__fadd_rn(ax, ay), __fadd_rn(az, aw)));
}

__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gmem_src) {
    unsigned s = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gmem_src));
}
__device__ __forceinline__ void cp_async_commit_wait_all() {
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_all;" ::: "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" :: "l"(p)); }

// dense_f32.rs:29-33 with simsimd's edge cases; na, nb = precomputed ordered norms.
__device__ __forceinline__ float cosine_from_parts(float ab, float na, float nb) {
    if (na == 0.0f && nb == 0.0f) return 1.0f;
    if (ab == 0.0f) return 0.0f;
    float c = __fdiv_rn(ab, __fmul_rn(na, nb));
    float dist = __fsub_rn(1.0f, c);
    if (!(dist > 0.0f)) dist = 0.0f;
    return __fsub_rn(1.0f, dist);
}

// L2 as a similarity (higher = closer): -|a - b|^2 = 2 ab - (|a|^2 + |b|^2), from the same ordered dot and the stored norms
// (|x|^2 is taken as rn(|x| * |x|), the same on the oracle's side), so it ranks like every other similarity here.
__device__ __forceinline__ float l2_from_parts(float ab, float na, float nb) {
    return __fsub_rn(__fmul_rn(2.0f, ab), __fadd_rn(__fmul_rn(na, na), __fmul_rn(nb, nb)));
}
__device__ __forceinline__ float sim_from_parts(int sim, float ab, float na, float nb) {
    return sim == SIM_COSINE ? cosine_from_parts(ab, na, nb) : (sim == SIM_L2 ? l2_from_parts(ab, na, nb) : ab);
}
__device__ __forceinline__ float finish_similarity(const VecDev& V, float ab, uint32_t x, float qnorm) {
    return V.sim == SIM_DOT ? ab : sim_from_parts(V.sim, ab, V.norms[x], qnorm);
}

}  // namespace nidx
