// Host restatement of the HNSW walk's fp16 screen, in the kernels' arithmetic and summation order:
//   the encoder and its record (api.cu hs_half_kernel), the lane-blocked f32 dot (common.cuh warp_dot_t), the fp16 dot
//   (warp_dot_h), the query bound (hnsw_search.cuh hs_query_bound) and the test itself (hs_screened_out).
// Directed roundings (__fmaf_ru, __fadd_ru, __double2float_ru, ...) are done under fesetround(FE_UPWARD); build with
// -frounding-math -ffp-contract=off.
#include <algorithm>
#include <cfenv>
#include <cmath>
#include <cstdint>
#include <cstring>

namespace {

const int SIM_COSINE = 1, SIM_L2 = 2;

struct Up {   // round toward +inf while alive
    Up() { std::fesetround(FE_UPWARD); }
    ~Up() { std::fesetround(FE_TONEAREST); }
};
float fmaf_ru(float a, float b, float c) { Up u; return std::fma(a, b, c); }
float fadd_ru(float a, float b) { Up u; volatile float r = a + b; return r; }
float d2f_ru(double x) { Up u; volatile float r = (float)x; return r; }
double dsqrt_ru(double x) { Up u; return std::sqrt(x); }
double dmul_ru(double a, double b) { Up u; volatile double r = a * b; return r; }

int dot_depth(int ld) { return (ld / 4 + 31) / 32 + 7; }

// lane l owns the groups of four g = l, l + 32, ...; four fused accumulators; (ax + ay) + (az + aw); butterfly 16, 8, 4, 2, 1
float lane_dot(const float* a, const float* b, int ld) {
    float lanes[32];
    for (int l = 0; l < 32; ++l) {
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int g = l; g < ld / 4; g += 32)
            for (int c = 0; c < 4; ++c) acc[c] = std::fma(a[4 * g + c], b[4 * g + c], acc[c]);
        lanes[l] = (acc[0] + acc[1]) + (acc[2] + acc[3]);
    }
    for (int off = 16; off >= 1; off >>= 1) {
        float t[32];
        for (int l = 0; l < 32; ++l) t[l] = lanes[l] + lanes[l ^ off];
        std::memcpy(lanes, t, sizeof(t));
    }
    return lanes[0];
}

float cosine_from_parts(float ab, float na, float nb) {
    if (na == 0.0f && nb == 0.0f) return 1.0f;
    if (ab == 0.0f) return 0.0f;
    float c = ab / (na * nb);
    float dist = 1.0f - c;
    if (!(dist > 0.0f)) dist = 0.0f;
    return 1.0f - dist;
}
float sim_from_parts(int sim, float ab, float na, float nb) {
    if (sim == SIM_COSINE) return cosine_from_parts(ab, na, nb);
    if (sim == SIM_L2) return 2.0f * ab - (na * na + nb * nb);
    return ab;
}
uint32_t ordered_bits(float f) {
    uint32_t u;
    std::memcpy(&u, &f, 4);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// hs_half_kernel for one row: h[ld] (as f32, exact) and rec = {norm, 2^-e, err_q, err_abs}
void encode(const float* v, int ld, float* h, float rec[4]) {
    float m = 0.0f;
    bool finite = true;
    for (int k = 0; k < ld; ++k) { finite = finite && std::isfinite(v[k]); m = std::fmax(m, std::fabs(v[k])); }
    int e = 0;
    if (finite && m > 0.0f) { int ex; std::frexp(m, &ex); e = std::min(15 - ex, 126); }
    const float up = std::ldexp(1.0f, e), down = std::ldexp(1.0f, -e);
    const double slack = 1.0 + 0x1p-20, mu = dot_depth(ld) * 0x1p-24, gm = mu / (1.0 - mu);
    double r2 = 0.0, v2 = 0.0;
    for (int k = 0; k < ld; ++k) {
        h[k] = (float)(_Float16)(v[k] * up);
        double dd = (double)h[k] * (double)down - (double)v[k];
        r2 = std::fma(dd, dd, r2);
        v2 = std::fma((double)v[k], (double)v[k], v2);
    }
    double rho = std::sqrt(r2 * slack), vn = std::sqrt(v2 * slack);
    double eq = (rho + gm * (2.0 * vn + rho)) * slack;
    double ea = 0x1p-149 * ((double)ld * (1.0 + (double)down) + 1.0) * slack;
    rec[0] = std::sqrt(lane_dot(v, v, ld));
    rec[1] = down;
    rec[2] = finite ? d2f_ru(eq) : INFINITY;
    rec[3] = d2f_ru(ea);
}

float query_bound(const float* q, int ld) {
    double s = 0.0;
    for (int k = 0; k < ld; ++k) s = std::fma((double)q[k], (double)q[k], s);
    return d2f_ru(dsqrt_ru(dmul_ru(s, 1.0 + 0x1p-20)));
}

}  // namespace

extern "C" {

// For n rows v[n][ld] (ld % 4 == 0) against one query: the exact f32 similarity and the screen's upper bound.  screened[i] = 1
// when the screen would be allowed to reject row i (finite bound, finite fp16 dot), i.e. when s_up[i] must rank >= s_exact[i].
// Returns the number of violations: screenable rows with ab_up < ab or ordered(s_up) < ordered(s_exact).
int screen_rows(const float* v, int n, int ld, const float* q, int sim, float* s_exact, float* s_up, float* ab_exact, float* ab_up, int* screened) {
    float* h = new float[ld];
    const float qn = std::sqrt(lane_dot(q, q, ld)), qb = query_bound(q, ld);
    int bad = 0;
    for (int i = 0; i < n; ++i) {
        const float* row = v + (size_t)i * ld;
        float rec[4];
        encode(row, ld, h, rec);
        float ab = lane_dot(row, q, ld);
        float a = lane_dot(h, q, ld) * rec[1];
        float bnd = fmaf_ru(qb, rec[2], rec[3]);
        screened[i] = std::fabs(a) <= 0x1p120f && bnd <= 0x1p100f;
        float up = screened[i] ? fadd_ru(a, bnd) : NAN;
        ab_exact[i] = ab;
        ab_up[i] = up;
        s_exact[i] = sim_from_parts(sim, ab, rec[0], qn);
        s_up[i] = screened[i] ? sim_from_parts(sim, up, rec[0], qn) : NAN;
        if (screened[i] && (!(ab <= up) || ordered_bits(s_up[i]) < ordered_bits(s_exact[i]))) ++bad;
    }
    delete[] h;
    return bad;
}

}
