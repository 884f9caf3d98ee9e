// ORACLE — TEST INFRASTRUCTURE ONLY.  Nothing under nucliadb_b200/ (the product) may
// include, link or call this.  Only tests/, __graft_entry__.smoke() and bench.py's
// cpu_baseline / --impl reference legs use it, as the checker / the CPU baseline.
//
// CPU restatement of the distance arithmetic of nidx_vector:
//   nidx/nidx_vector/src/vector_types/dense_f32.rs:29-39   cosine_similarity = 1 - simsimd cos distance
//                                                          dot_similarity    = simsimd dot
//   nidx/nidx_vector/src/utils.rs:20-23                    normalize_vector
//
// The arithmetic itself lives in the third-party crate simsimd 6.5.16 (nidx/Cargo.lock:4552),
// which is NOT in the reference tree.  Restated from its published algorithm [recalled]:
//   dot:  ab = sum a_i*b_i                     (f32 lanes, backend-specific order)
//   cos:  ab, a2, b2 accumulated together; distance =
//           0                          if a2 == 0 && b2 == 0
//           1                          if ab == 0
//           max(0, 1 - ab/(sqrt(a2)*sqrt(b2)))   otherwise
//         (simsimd uses rsqrt + Newton on some backends; last-ulp differences per host)
// simsimd picks its summation order per CPU backend at run time, so the reference's low-order
// bits are host dependent and its own tests only pin 1e-2 (dense_f32.rs:66-84).  The oracle
// therefore fixes ONE summation order ("lane-blocked", below) and documents it; a second,
// f64-accumulated variant is provided to show the order is within 1e-6 of exact.
//
// Lane-blocked order (the same order the CUDA kernels use, so scores are bit-identical):
//   32 lanes; lane l owns the float4 groups g with g % 32 == l (elements 4g..4g+3), visited in
//   increasing g; four independent fused-multiply-add accumulators per lane (one per float4
//   component); lane value = (ax + ay) + (az + aw); lanes combined by an xor butterfly with
//   offsets 16, 8, 4, 2, 1 (v[l] += v[l ^ off]).  Rows are zero padded to a multiple of 4.
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>

namespace nidx_oracle {

enum Similarity : int { SIM_DOT = 0, SIM_COSINE = 1, SIM_L2 = 2 };   // L2: an extension, the reference has none (config.rs:33-37)

// Lane 0's value of the xor butterfly (v[l] += v[l ^ off] for off = 16, 8, 4, 2, 1).  Lane 0 only ever consumes lanes below
// `off`, whose values are v[l] + v[l + off] with the operands in that order: the halving tree below is the same arithmetic
// with 31 additions instead of 160.
static inline float butterfly32(float v[32]) {
    for (int off = 16; off >= 1; off >>= 1)
        for (int l = 0; l < off; ++l) v[l] = v[l] + v[l + off];
    return v[0];
}

// dot(a, b) in the lane-blocked order.  acc[k] (k = 4*lane + component) accumulates the elements
// i with i % 128 == k in increasing i -- the same thing as "lane l owns groups g % 32 == l",
// written so that gcc vectorises it (8 zmm accumulators).  Zero padding is a no-op for fma.
static inline float dot_ordered(const float* __restrict a, const float* __restrict b, int d) {
    alignas(64) float acc[128];
    for (int k = 0; k < 128; ++k) acc[k] = 0.0f;
    int full = d / 128 * 128;
    for (int i = 0; i < full; i += 128)
        for (int k = 0; k < 128; ++k) acc[k] = __builtin_fmaf(a[i + k], b[i + k], acc[k]);
    for (int k = 0; k < d - full; ++k) acc[k] = __builtin_fmaf(a[full + k], b[full + k], acc[k]);
    float v[32];
    for (int l = 0; l < 32; ++l) v[l] = (acc[4 * l] + acc[4 * l + 1]) + (acc[4 * l + 2] + acc[4 * l + 3]);
    return butterfly32(v);
}

static inline double dot_f64(const float* a, const float* b, int d) {
    double s = 0;
    for (int i = 0; i < d; ++i) s += (double)a[i] * (double)b[i];
    return s;
}

// sqrt(sum a_i^2) in the lane-blocked order: the per-vector norm the kernels precompute at open().
static inline float norm_ordered(const float* a, int d) { return std::sqrt(dot_ordered(a, a, d)); }

// dense_f32.rs:29-33 with simsimd's edge cases.  na, nb are norm_ordered(a), norm_ordered(b).
static inline float cosine_from_parts(float ab, float na, float nb) {
    if (na == 0.0f && nb == 0.0f) return 1.0f;  // distance 0
    if (ab == 0.0f) return 0.0f;                // distance 1
    float c = ab / (na * nb);
    float dist = 1.0f - c;
    if (!(dist > 0.0f)) dist = 0.0f;            // simsimd clamps the distance at 0
    return 1.0f - dist;
}

static inline float similarity(int sim, const float* a, float na, const float* b, float nb, int d) {
    float ab = dot_ordered(a, b, d);
    if (sim == SIM_L2) return 2.0f * ab - (na * na + nb * nb);   // -|a - b|^2 from the ordered dot and the norms (csrc/common.cuh l2_from_parts)
    return sim == SIM_COSINE ? cosine_from_parts(ab, na, nb) : ab;
}

// utils.rs:20-23: magnitude = sqrt(fold(0.0, acc + x.powi(2))) in f32, sequential; out = x / magnitude.
static inline void normalize_vector(const float* in, float* out, int d) {
    float acc = 0.0f;
    for (int i = 0; i < d; ++i) acc = acc + in[i] * in[i];
    float mag = std::sqrt(acc);
    for (int i = 0; i < d; ++i) out[i] = in[i] / mag;
}

// f32::total_cmp key: monotone map f32 -> u32 (hnsw/search.rs:90-93 orders Cnx by total_cmp).
static inline uint32_t ordered_bits(float f) {
    uint32_t u;
    std::memcpy(&u, &f, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
// Total order used by oracle AND kernels wherever the reference's order under exactly equal
// scores is unspecified (BinaryHeap / sort_unstable): higher score first, then lower id first.
static inline uint64_t rank_key(float score, uint32_t id) {
    return ((uint64_t)ordered_bits(score) << 32) | (uint64_t)(0xFFFFFFFFu - id);
}

}  // namespace nidx_oracle
