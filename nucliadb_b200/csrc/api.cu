// nidx_b200 — C ABI (include/nidx_b200.h) over the CUDA kernels.  Host side of the hot path:
// what nidx_vector's OpenSegment / HnswBuilder and the tantivy collector call do on the CPU in the
// reference is orchestrated here on one GPU.  No CPU fallback: every entry point needs a device.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cfloat>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/nidx_b200.h"
#include "bm25.cuh"
#include "graph.cuh"
#include "phrase.cuh"
#include "prefilter.cuh"
#include "common.cuh"
#include "hnsw_build.cuh"
#include "hnsw_search.cuh"
#include "hnsw_rabitq.cuh"
#include "rabitq.cuh"
#include "rank_fusion.cuh"
#include "scan.cu"
#include "scan_tc2.cuh"
#include "segment_io.hpp"
#include "shard.cuh"
#include "suggest.cuh"
#include "topk.cuh"

using namespace nidx;

// ---------------------------------------------------------------------------------------------
static thread_local std::string g_err;
static std::atomic<uint64_t> g_launches{0};

static int fail(int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    g_err = buf;
    return code;
}
#define CU(expr)                                                                                              \
    do {                                                                                                      \
        cudaError_t e__ = (expr);                                                                             \
        if (e__ != cudaSuccess) return fail(NIDX_ECUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
    } while (0)
#define LAUNCHED() (g_launches.fetch_add(1, std::memory_order_relaxed))

static int next_pow2(int x) { int p = 1; while (p < x) p <<= 1; return p; }
static int ilog2(int x) { int b = 0; while ((1 << b) < x) ++b; return b; }

// The owner of every device allocation: move-only, freed when it is destroyed, released or allocated again.  Sizes are in bytes.
// alloc() takes exactly the size asked for (segment arrays, whose sizes include the padding kernels read into), ensure() grows
// with slack (per-call scratch), try_alloc() reports a failure to its caller only (an allocation with a fallback).  It converts to
// the raw pointer that kernels and copies take.
template <class T>
struct DevArray {
    T* p = nullptr;
    size_t cap = 0;
    DevArray() = default;
    DevArray(DevArray&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DevArray& operator=(DevArray&& o) noexcept {
        if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
        return *this;
    }
    ~DevArray() { release(); }
    operator T*() const { return p; }
    template <class U> U* as() const { return reinterpret_cast<U*>(p); }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    cudaError_t try_alloc(size_t bytes) {
        release();
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) cap = bytes;
        else { p = nullptr; (void)cudaGetLastError(); }   // not left for the next cudaGetLastError() to report
        return e;
    }
    int alloc(size_t bytes) {
        cudaError_t e = try_alloc(bytes);
        return e == cudaSuccess ? 0 : fail(NIDX_ECUDA, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(e));
    }
    int ensure(size_t bytes) {
        if (bytes <= cap || try_alloc(bytes + bytes / 4 + 256) == cudaSuccess) return 0;
        return alloc(bytes);
    }
};
using DevBuf = DevArray<unsigned char>;
#define ENSURE(buf, bytes) do { int r__ = (buf).ensure(bytes); if (r__) return r__; } while (0)
#define ALLOC(buf, bytes) do { int r__ = (buf).alloc(bytes); if (r__) return r__; } while (0)

// Per-call scratch; a segment keeps a pool so concurrent searches do not share one.
struct Workspace {
    DevBuf queries, qnorms, stage, scores, partial, filter, misc, sched, facets, phrases, prefilter, rerun;
    cudaEvent_t done = nullptr;
    cudaStream_t last_stream = nullptr;
    bool busy = false;
    ~Workspace() { if (done) cudaEventDestroy(done); }
};

struct WorkspacePool {
    std::mutex mu;
    std::vector<Workspace*> all;
    // A free workspace last used on this stream (stream order protects it), else one whose last call has completed, else a new one
    // (up to MAX_POOL: calls issued from one host thread on alternating streams then overlap on the device instead of the second
    // waiting for the first one's buffers), else the host waits for a free one's last call.
    static constexpr size_t MAX_POOL = 8;
    Workspace* acquire(cudaStream_t stream) {
        std::lock_guard<std::mutex> g(mu);
        Workspace* pick = nullptr;
        for (Workspace* w : all)
            if (!w->busy && w->last_stream == stream) { pick = w; break; }
        if (!pick) {
            for (Workspace* w : all)
                if (!w->busy && (!w->done || cudaEventQuery(w->done) == cudaSuccess)) { pick = w; break; }
            (void)cudaGetLastError();   // cudaErrorNotReady from a query is not an error: do not leave it for the next cudaGetLastError()
        }
        if (!pick && all.size() >= MAX_POOL)
            for (Workspace* w : all)
                if (!w->busy) { cudaEventSynchronize(w->done); pick = w; break; }
        if (!pick) {
            pick = new Workspace();
            cudaEventCreateWithFlags(&pick->done, cudaEventDisableTiming);
            all.push_back(pick);
        }
        pick->busy = true;
        return pick;
    }
    void release(Workspace* w, cudaStream_t stream) {
        cudaEventRecord(w->done, stream);
        std::lock_guard<std::mutex> g(mu);
        w->last_stream = stream;
        w->busy = false;
    }
    ~WorkspacePool() { for (Workspace* w : all) delete w; }
};
struct WsGuard {
    WorkspacePool& pool; Workspace* w; cudaStream_t s;
    WsGuard(WorkspacePool& p, cudaStream_t st) : pool(p), w(p.acquire(st)), s(st) {}
    ~WsGuard() { pool.release(w, s); }
};

// Workspaces of the calls that belong to no segment, per device
static WorkspacePool* plan_pool(int device) {
    static std::mutex mu;
    static WorkspacePool* pools[64] = {nullptr};
    std::lock_guard<std::mutex> g(mu);
    if (device < 0 || device >= 64) return nullptr;
    if (!pools[device]) pools[device] = new WorkspacePool();
    return pools[device];
}

// The `mem` contract of include/nidx_b200.h for one call.  in() and out() hand out a device pointer for each caller buffer: the
// caller's own on the device path, else a 16-byte-aligned slice of one staging buffer that place() lays out (uploading the host
// inputs) and finish() copies back (then synchronises the stream, once).  A NULL output gets a scratch slice that is never copied
// back; a NULL input stays NULL.  Inputs and outputs may lie on different sides (host queries, device outputs).  On the device path
// nothing is copied, set or synchronised here.
struct Stage {
    cudaStream_t stream;
    bool qhost, ohost;
    struct Slot { void* var; const void* in; void* out; size_t bytes; void* dev; };   // var: the caller's T* to point at the slice
    std::vector<Slot> slots;
    size_t total = 0;
    Stage(cudaStream_t s, bool qh, bool oh) : stream(s), qhost(qh), ohost(oh) {}
    void add(void* var, const void* in, void* out, size_t bytes) {
        slots.push_back({var, in, out, bytes, nullptr});
        total += (bytes + 15) / 16 * 16;
    }
    template <class T> void in(const T* src, size_t n, const T** dev) {
        *dev = src;
        if (qhost && src) add(dev, src, nullptr, n * sizeof(T));
    }
    template <class T> void out(T* dst, size_t n, T** dev) {
        *dev = dst;
        if (ohost || !dst) add(dev, nullptr, ohost ? dst : nullptr, n * sizeof(T));
    }
    int place(DevBuf& buf) {
        ENSURE(buf, total);
        unsigned char* p = buf.as<unsigned char>();
        for (Slot& s : slots) {
            s.dev = p;
            p += (s.bytes + 15) / 16 * 16;
            memcpy(s.var, &s.dev, sizeof(void*));
            if (s.in && s.bytes) CU(cudaMemcpyAsync(s.dev, s.in, s.bytes, cudaMemcpyHostToDevice, stream));
        }
        return 0;
    }
    // sync: synchronise on the device path too (a call that reads a count back)
    int finish(bool sync = false) {
        if (ohost)
            for (const Slot& s : slots)
                if (s.out && s.bytes) CU(cudaMemcpyAsync(s.out, s.dev, s.bytes, cudaMemcpyDeviceToHost, stream));
        if (ohost || sync) CU(cudaStreamSynchronize(stream));
        return 0;
    }
};

struct nidx_vec_segment {
    nidx_vec_config cfg;
    uint64_t n = 0;
    int d = 0, ld = 0;
    int sm_count = 0;
    DevArray<float> d_vecs;
    DevArray<float> d_norms;
    DevArray<uint32_t> d_par_of;
    DevArray<uint32_t> d_par_first;
    uint32_t n_par = 0;
    DevArray<uint64_t> d_alive;
    uint64_t alive_count = 0;         // set bits of d_alive (counted in nidx_vec_set_alive): `matching` of an unfiltered search
    DevArray<uint64_t> d_par_keys;    // [n_par] caller-supplied paragraph keys for the cross-segment de-duplication (shard.cuh)
    struct InvIndex {                 // one inverted index (inverted_index/fst_index.rs + map.rs): sorted keys on the host, postings in HBM
        std::vector<unsigned char> key_bytes;
        std::vector<uint64_t> key_off, post_off;
        DevArray<uint32_t> d_post;
        DevArray<uint64_t> d_post_off;  // post_off in HBM, for the prefilter hand-off (nidx_vec_prefilter_bits)
        uint32_t n_keys = 0;
    } inv[2];
    // graph
    bool has_graph = false;
    std::vector<uint8_t> h_level;
    DevArray<uint8_t> d_level;
    uint32_t entry_node = 0, entry_layer = 0;
    int s0 = 0, su = 0;
    uint64_t upper_rows = 0;
    DevArray<uint32_t> d_adj0; DevArray<float> d_w0;
    DevArray<uint64_t> d_upper_off;
    DevArray<uint32_t> d_adjU; DevArray<float> d_wU;
    float max_norm = 0.0f;              // max |v| (error bound of the tensor-core filter for Dot)
    bool tc_rows_ok = false;            // every row meets the filter's bound (max_norm_kernel): else batches take the exact scan
    CUtensorMap map_v;                  // TMA descriptor of the vector block (scan_tc2.cuh), built on first use
    bool map_v_ready = false;
    std::mutex map_mu;
    DevArray<unsigned char> d_quant;    // RaBitQ codes [n][quant_stride] (vectors.quant records, padded)
    int quant_stride = 0;
    DevArray<unsigned long long> d_counters;   // [8] the build's counters
    std::atomic<unsigned long long*> last_counters{nullptr};   // counters of the LAST search call (they live in that call's workspace: concurrent
                                                               // searches never add into each other's), read by nidx_vec_counters*
    DevArray<unsigned int> d_work_counter;
    cudaEvent_t ev_k0 = nullptr, ev_k1 = nullptr;  // around the dominant kernel of the last search (bench roofline)
    WorkspacePool pool;
    // fp16 screening copy of the vectors for the HNSW walk (hs_half_kernel), made once by ensure_half_copy
    DevArray<__half> d_hvecs;
    DevArray<float4> d_hrec;
    int ldh = 0;
    bool half_decided = false;          // the copy was made, or was found not to fit (the walk then reads f32 rows only)
    std::mutex half_mu;

    ~nidx_vec_segment() {
        if (ev_k0) cudaEventDestroy(ev_k0);
        if (ev_k1) cudaEventDestroy(ev_k1);
    }

    VecDev vdev() const {
        VecDev v;
        v.vecs = d_vecs; v.norms = d_norms; v.paragraph_of = d_par_of; v.n = (uint32_t)n; v.d = d; v.ld = ld; v.sim = cfg.similarity;
        v.hvecs = nullptr; v.hrec = nullptr; v.ldh = 0;   // the HNSW walks attach the screening copy (attach_half_copy)
        return v;
    }
    GraphDev gdev() const {
        GraphDev g;
        g.n = (uint32_t)n; g.M = cfg.m; g.M0 = cfg.m0; g.s0 = s0; g.su = su; g.level = d_level;
        g.entry_node = entry_node; g.entry_layer = entry_layer;
        g.adj0 = d_adj0; g.w0 = d_w0; g.upper_off = d_upper_off; g.adjU = d_adjU; g.wU = d_wU;
        return g;
    }
};

static int stride0_for(int M0) { return (M0 + 31) / 32 * 32; }
static int strideU_for(int M) { return (M + 15) / 16 * 16; }

static void free_graph(nidx_vec_segment* s) {
    s->d_level.release(); s->d_adj0.release(); s->d_w0.release(); s->d_upper_off.release(); s->d_adjU.release(); s->d_wU.release();
    s->has_graph = false;
}

// Allocate graph storage for the given levels (ram_hnsw.rs:88-107: every node in layers 0..=level,
// entry point in the top layer -- lowest id there).
static int alloc_graph(nidx_vec_segment* s, const uint8_t* level) {
    free_graph(s);
    uint64_t n = s->n;
    s->h_level.assign(level, level + n);
    std::vector<uint64_t> off(n ? n : 1);
    uint64_t rows = 0;
    uint32_t top = 0;
    for (uint64_t i = 0; i < n; ++i) { off[i] = rows; rows += level[i]; top = std::max<uint32_t>(top, level[i]); }
    s->upper_rows = rows;
    s->entry_layer = top;
    s->entry_node = 0;
    for (uint64_t i = 0; i < n; ++i) if (level[i] == top) { s->entry_node = (uint32_t)i; break; }
    s->s0 = stride0_for(s->cfg.m0);
    s->su = strideU_for(s->cfg.m);
    size_t n0 = (size_t)n * s->s0, nu = (size_t)std::max<uint64_t>(rows, 1) * s->su;
    ALLOC(s->d_level, std::max<uint64_t>(n, 1));
    ALLOC(s->d_adj0, n0 * 4 + 16);
    ALLOC(s->d_w0, n0 * 4 + 16);
    ALLOC(s->d_upper_off, std::max<uint64_t>(n, 1) * 8);
    ALLOC(s->d_adjU, nu * 4);
    ALLOC(s->d_wU, nu * 4);
    CU(cudaMemcpy(s->d_level, level, n, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_upper_off, off.data(), n * 8, cudaMemcpyHostToDevice));
    CU(cudaMemset(s->d_adj0, 0xFF, n0 * 4));
    CU(cudaMemset(s->d_w0, 0, n0 * 4));
    CU(cudaMemset(s->d_adjU, 0xFF, nu * 4));
    CU(cudaMemset(s->d_wU, 0, nu * 4));
    return 0;
}

// out[0] = bits of max |v|; out[1] = 1 if some row is outside the tensor-core filter's bound (scan_tc2.cuh): a non-finite norm, or
// (cosine) a row with a non-zero element whose norm is below TC2_MIN_NORM.  Rows are read only for such tiny norms.
__global__ void max_norm_kernel(VecDev V, uint64_t n, unsigned int* __restrict__ out) {
    float m = 0.0f;
    bool bad = false;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        const float nv = V.norms[i];
        m = fmaxf(m, nv);
        if (!(nv <= FLT_MAX)) bad = true;
        else if (V.sim == SIM_COSINE && nv < TC2_MIN_NORM)
            for (int j = 0; j < V.ld && !bad; ++j) bad = V.vecs[i * V.ld + j] != 0.0f;
    }
    for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xFFFFFFFFu, m, off));
    if ((threadIdx.x & 31) == 0) atomicMax(out, __float_as_uint(m));   // non-negative floats order like their bit patterns
    if (__any_sync(0xFFFFFFFFu, bad) && (threadIdx.x & 31) == 0) atomicOr(out + 1, 1u);
}

// The HNSW walk's fp16 screening copy (hs_screened_out in hnsw_search.cuh derives the bound), one warp per row:
//   h = fp16(v * 2^e) with e = min(15 - exponent(max |v_i|), 126): max |v_i| * 2^e lies in [2^14, 2^15), so no element overflows
//   fp16, and 2^-e is a normal f32 (tiny rows then use fp16 subnormals, which only widens rho);
//   rec = {norms[i], 2^-e, err_q, err_abs}, err_q >= rho + g_m (2 |v| + rho), rho = |h * 2^-e - v|, err_abs >= 2^-149 (ld (1 + 2^-e) + 1).
//   rho^2 and |v|^2 are f64 sums of squares of exact (or, for rho, correctly rounded f64) terms: each is within ld * 2^-52 of its
//   value, which the factor 1 + 2^-20 covers along with the roundings of what follows; the f32 results are rounded up.  A row with
//   a non-finite element gets err_q = +inf, so the walk always reads its f32 row.
__global__ void hs_half_kernel(VecDev V, uint64_t n, int ldh, __half* __restrict__ hv, float4* __restrict__ rec) {
    const int lane = threadIdx.x & 31;
    const double slack = 1.0 + 0x1p-20, mu = dot_depth(V.ld) * 0x1p-24, gm = mu / (1.0 - mu);
    for (uint64_t i = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; i < n; i += ((uint64_t)gridDim.x * blockDim.x) >> 5) {
        const float* v = V.vecs + i * V.ld;
        float m = 0.0f;
        bool finite = true;
        for (int k = lane; k < V.ld; k += 32) { float x = v[k]; finite = finite && isfinite(x); m = fmaxf(m, fabsf(x)); }
        for (int off = 16; off >= 1; off >>= 1) m = fmaxf(m, __shfl_xor_sync(0xFFFFFFFFu, m, off));
        finite = __all_sync(0xFFFFFFFFu, finite);
        int e = 0;
        if (finite && m > 0.0f) { int ex; frexpf(m, &ex); e = min(15 - ex, 126); }
        const float up = ldexpf(1.0f, e), down = ldexpf(1.0f, -e);
        double r2 = 0.0, v2 = 0.0;
        for (int k = lane; k < ldh; k += 32) {
            float x = k < V.ld ? v[k] : 0.0f;
            __half h = __float2half_rn(__fmul_rn(x, up));
            hv[i * ldh + k] = h;
            double dd = (double)__half2float(h) * (double)down - (double)x;
            r2 = fma(dd, dd, r2);
            v2 = fma((double)x, (double)x, v2);
        }
        for (int off = 16; off >= 1; off >>= 1) { r2 += __shfl_xor_sync(0xFFFFFFFFu, r2, off); v2 += __shfl_xor_sync(0xFFFFFFFFu, v2, off); }
        if (lane == 0) {
            double rho = sqrt(r2 * slack), vn = sqrt(v2 * slack);
            double eq = (rho + gm * (2.0 * vn + rho)) * slack;
            double ea = 0x1p-149 * ((double)V.ld * (1.0 + (double)down) + 1.0) * slack;
            rec[i] = make_float4(V.norms[i], down, finite ? __double2float_ru(eq) : INFINITY, __double2float_ru(ea));
        }
    }
}

// Attach the screening copy to V for an HNSW walk, making it on the segment's first walk (build, extend or search) under the
// segment's lock; the conversion has finished before any caller gets the pointers.  When the copy (ldh * 2 + 16 bytes per
// vector) does not fit next to what HBM already holds with HS_HALF_MARGIN to spare, the segment keeps the f32-only walk.
// NIDX_B200_HS_F16=0 forces the f32-only walk (the tests compare the two walks).
constexpr size_t HS_HALF_MARGIN = (size_t)4 << 30;
static int attach_half_copy(nidx_vec_segment* s, VecDev* V) {
    const char* e = getenv("NIDX_B200_HS_F16");
    if (e && !strcmp(e, "0")) return 0;
    std::lock_guard<std::mutex> g(s->half_mu);
    if (!s->half_decided && s->n) {
        s->half_decided = true;
        const int ldh = (s->ld + 7) / 8 * 8;
        const size_t hbytes = (size_t)s->n * ldh * 2, rbytes = (size_t)s->n * 16;
        size_t free_b = 0, total_b = 0;
        CU(cudaMemGetInfo(&free_b, &total_b));
        if (free_b < hbytes + rbytes + HS_HALF_MARGIN) return 0;
        if (s->d_hvecs.try_alloc(hbytes) != cudaSuccess || s->d_hrec.try_alloc(rbytes) != cudaSuccess) {
            s->d_hvecs.release();   // out of memory is not an error here: the f32-only walk runs
            return 0;
        }
        hs_half_kernel<<<s->sm_count * 8, 256>>>(s->vdev(), s->n, ldh, s->d_hvecs, s->d_hrec);
        LAUNCHED();
        CU(cudaGetLastError());
        CU(cudaDeviceSynchronize());
        s->ldh = ldh;
    }
    if (s->ldh) { V->hvecs = s->d_hvecs; V->hrec = s->d_hrec; V->ldh = s->ldh; }
    return 0;
}

// cuTensorMapEncodeTiled through the runtime's driver entry point (no link-time dependency on libcuda)
typedef CUresult (*tmap_encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                   CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static int make_row_tensor_map(CUtensorMap* map, const float* base, uint64_t rows, int ld, int box_rows) {
    static tmap_encode_fn encode = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess)
            encode = reinterpret_cast<tmap_encode_fn>(fn);
    });
    if (!encode) return fail(NIDX_ECUDA, "cuTensorMapEncodeTiled is not available from this driver");
    cuuint64_t dims[2] = {(cuuint64_t)ld, (cuuint64_t)rows};
    cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
    cuuint32_t box[2] = {(cuuint32_t)TC2_KB, (cuuint32_t)box_rows};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = encode(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(NIDX_ECUDA, "cuTensorMapEncodeTiled failed (%d)", (int)r);
    return 0;
}

// A per-row array the caller sets (n values from the host, into *dev, allocated on first use) or clears (host == NULL)
template <class T>
static int set_rows(int device, DevArray<T>& dev, const T* host, size_t n) {
    CU(cudaSetDevice(device));
    if (!host) { dev.release(); return 0; }
    if (!dev) ALLOC(dev, std::max<size_t>(n, 1) * sizeof(T));
    CU(cudaMemcpy(dev, host, n * sizeof(T), cudaMemcpyHostToDevice));
    return 0;
}

extern "C" {

const char* nidx_last_error(void) { return g_err.c_str(); }
int nidx_device_count(void) {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}
uint64_t nidx_launch_count(void) { return g_launches.load(); }

static int check_device(int device) {
    int n = nidx_device_count();
    if (n <= 0) return fail(NIDX_ENODEVICE, "no CUDA device available (nidx_b200 has no CPU fallback)");
    if (device < 0 || device >= n) return fail(NIDX_EINVAL, "device %d out of range (have %d)", device, n);
    CU(cudaSetDevice(device));
    return 0;
}

static int fill_defaults(nidx_vec_config* c) {
    if (c->dimension <= 0) return fail(NIDX_EINVAL, "dimension must be positive");
    if (c->similarity != NIDX_SIM_DOT && c->similarity != NIDX_SIM_COSINE && c->similarity != NIDX_SIM_L2) return fail(NIDX_EINVAL, "unknown similarity %d", c->similarity);
    if (c->m <= 0) c->m = 30;                              // params.rs:40
    if (c->m0 <= 0) c->m0 = 60;                            // params.rs:34
    if (c->ef_construction <= 0) c->ef_construction = 100; // params.rs:43
    if (c->ef_search <= 0) c->ef_search = 30;              // params.rs:46
    if (c->m0 > HS_MAX_ROW || c->m > HS_MAX_ROW) return fail(NIDX_EINVAL, "M / M0 above %d not supported", HS_MAX_ROW);
    if (c->ef_construction > HB_MAX_CAND) return fail(NIDX_EINVAL, "ef_construction above %d not supported", HB_MAX_CAND);
    return 0;
}

// Common tail of create/open: vectors are in d_vecs; compute norms, paragraph CSR.
static int finish_create(nidx_vec_segment* s, const uint32_t* paragraph_of_host) {
    uint64_t n = s->n;
    ALLOC(s->d_norms, std::max<uint64_t>(n, 1) * 4);
    if (n) {
        int blocks = (int)std::min<uint64_t>((n + 7) / 8, (uint64_t)s->sm_count * 16);
        row_norms_kernel<<<blocks, 256>>>(s->d_vecs, s->ld, n, s->d_norms);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    s->n_par = (uint32_t)n;
    if (paragraph_of_host) {
        // paragraphs own contiguous vector ranges (data_store/v2: first_vector / num_vectors)
        std::vector<uint32_t> first;
        uint32_t prev = NIDX_NIL;
        for (uint64_t i = 0; i < n; ++i) {
            uint32_t p = paragraph_of_host[i];
            if (i == 0 || p != prev) {
                if (p != (uint32_t)first.size()) return fail(NIDX_EINVAL, "paragraph_of must be contiguous and ascending from 0 (vector %llu -> %u)", (unsigned long long)i, p);
                first.push_back((uint32_t)i);
                prev = p;
            }
        }
        first.push_back((uint32_t)n);
        s->n_par = (uint32_t)first.size() - 1;
        if (s->n_par != n) {  // only materialise when some paragraph has several vectors
            ALLOC(s->d_par_of, n * 4);
            CU(cudaMemcpy(s->d_par_of, paragraph_of_host, n * 4, cudaMemcpyHostToDevice));
            ALLOC(s->d_par_first, first.size() * 4);
            CU(cudaMemcpy(s->d_par_first, first.data(), first.size() * 4, cudaMemcpyHostToDevice));
        }
    }
    if (n) {   // max |v| for the Dot error bound of the tensor-core filter, and whether every row meets the bound
        DevArray<unsigned int> d_bits;
        ALLOC(d_bits, 8);
        CU(cudaMemset(d_bits, 0, 8));
        max_norm_kernel<<<std::min<uint64_t>((n + 255) / 256, (uint64_t)s->sm_count * 8), 256>>>(s->vdev(), n, d_bits);
        LAUNCHED();
        unsigned int hb[2] = {0, 0};
        CU(cudaMemcpy(hb, d_bits, 8, cudaMemcpyDeviceToHost));
        memcpy(&s->max_norm, &hb[0], 4);
        s->tc_rows_ok = hb[1] == 0;
    }
    ALLOC(s->d_counters, 8 * sizeof(unsigned long long));
    CU(cudaMemset(s->d_counters, 0, 8 * sizeof(unsigned long long)));
    ALLOC(s->d_work_counter, 64);
    CU(cudaEventCreate(&s->ev_k0));
    CU(cudaEventCreate(&s->ev_k1));
    CU(cudaDeviceSynchronize());
    return 0;
}

// A new segment, freed with everything it holds unless the call that creates it succeeds and releases it to the caller
static int new_segment(const nidx_vec_config* cfg, std::unique_ptr<nidx_vec_segment>& out) {
    if (!cfg) return fail(NIDX_EINVAL, "null argument");
    nidx_vec_config c = *cfg;
    int r = fill_defaults(&c);
    if (r) return r;
    r = check_device(c.device);
    if (r) return r;
    out.reset(new nidx_vec_segment());
    nidx_vec_segment* s = out.get();
    s->cfg = c;
    s->d = c.dimension;
    s->ld = (c.dimension + 3) / 4 * 4;
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, c.device);
    s->sm_count = prop.multiProcessorCount;
    return 0;
}

// The segment's n rows into d_vecs ([n][ld], zero padded).  Source rows are row_bytes apart and start with the d floats; `whole`:
// they are [ld] floats already, copied as they are.
static int upload_rows(nidx_vec_segment* s, const void* rows, size_t row_bytes, bool host, bool whole) {
    const uint64_t n = s->n;
    ALLOC(s->d_vecs, std::max<size_t>((size_t)n * s->ld * 4, 16));
    if (n == 0) return 0;
    if (whole) {
        CU(cudaMemcpy(s->d_vecs, rows, (size_t)n * row_bytes, host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice));
        return 0;
    }
    const unsigned char* src = static_cast<const unsigned char*>(rows);
    DevBuf staged;
    if (host) {
        ALLOC(staged, (size_t)n * row_bytes);
        CU(cudaMemcpy(staged, rows, (size_t)n * row_bytes, cudaMemcpyHostToDevice));
        src = staged;
    }
    pad_rows_kernel<<<s->sm_count * 8, 256>>>(src, row_bytes, s->d, s->d_vecs, s->ld, n);
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaDeviceSynchronize());
    return 0;
}

int nidx_vec_create(const nidx_vec_config* cfg, const float* vectors, uint64_t n, int32_t ld, int mem, const uint32_t* paragraph_of,
                    nidx_vec_segment** out) {
    if (!out) return fail(NIDX_EINVAL, "null argument");
    std::unique_ptr<nidx_vec_segment> s;
    int r = new_segment(cfg, s);
    if (r) return r;
    if (n >= (1ull << 31)) return fail(NIDX_EINVAL, "at most 2^31-1 vectors per segment");
    if (ld < s->d) return fail(NIDX_EINVAL, "ld %d < dimension %d (VectorErr::InconsistentDimensions)", ld, s->d);
    s->n = n;
    r = upload_rows(s.get(), vectors, (size_t)ld * 4, mem == NIDX_MEM_HOST, ld == s->ld);
    if (!r) r = finish_create(s.get(), paragraph_of);
    if (r) return r;
    *out = s.release();
    return 0;
}

// ---- utils::normalize_vector (nidx_vector/src/utils.rs:20-23) ----------------------------------------------
// magnitude = sqrt(fold(0.0, |acc, x| acc + x.powi(2))) -- a SEQUENTIAL f32 fold (powi(2) = one rounded multiply, no FMA) --
// then x / magnitude per element.  One warp per vector: the row is staged in shared memory with coalesced loads, lane 0 replays
// the fold in the reference's order (bit-identical to it), all lanes divide.  A zero vector divides by zero like the reference
// (NaN components).  Called at index time (indexer.rs:94-146) and per query (searcher.rs:246-252): negligible next to a search.
constexpr int NRM_WARPS = 4;
__global__ void __launch_bounds__(NRM_WARPS * 32) normalize_rows_kernel(float* __restrict__ v, uint64_t n, int d, int ld) {
    extern __shared__ float nrm_row[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float* row = nrm_row + (size_t)warp * d;
    for (uint64_t i = (uint64_t)blockIdx.x * NRM_WARPS + warp; i < n; i += (uint64_t)gridDim.x * NRM_WARPS) {
        float* src = v + i * (uint64_t)ld;
        for (int j = lane; j < d; j += 32) row[j] = src[j];
        __syncwarp();
        float acc = 0.0f;
        if (lane == 0)
            for (int j = 0; j < d; ++j) acc = __fadd_rn(acc, __fmul_rn(row[j], row[j]));
        float mag = __fsqrt_rn(__shfl_sync(0xFFFFFFFFu, acc, 0));
        for (int j = lane; j < d; j += 32) src[j] = __fdiv_rn(row[j], mag);
        __syncwarp();
    }
}

int nidx_normalize_vectors(int32_t device, float* vectors, uint64_t n, int32_t d, int32_t ld, int mem, void* stream_) {
    int r = check_device(device);
    if (r) return r;
    if (d <= 0 || ld < d || !vectors) return fail(NIDX_EINVAL, "normalize: d %d, ld %d", d, ld);
    if ((size_t)d * 4 * NRM_WARPS > 200 * 1024) return fail(NIDX_EINVAL, "normalize: dimension %d too large", d);
    if (n == 0) return 0;
    cudaStream_t st = static_cast<cudaStream_t>(stream_);
    float* dv = vectors;
    DevArray<float> staged;
    size_t bytes = (size_t)n * ld * 4;
    if (mem == NIDX_MEM_HOST) {
        ALLOC(staged, bytes);
        dv = staged;
        cudaError_t e = cudaMemcpyAsync(dv, vectors, bytes, cudaMemcpyHostToDevice, st);
        if (e != cudaSuccess) return fail(NIDX_ECUDA, "normalize: H2D failed: %s", cudaGetErrorString(e));
    }
    int sm = 0;
    cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, device);
    size_t smem = (size_t)d * 4 * NRM_WARPS;
    cudaFuncSetAttribute(normalize_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    uint64_t want = (n + NRM_WARPS - 1) / NRM_WARPS;
    int grid = (int)std::min<uint64_t>(want, (uint64_t)sm * 16);
    normalize_rows_kernel<<<grid, NRM_WARPS * 32, smem, st>>>(dv, n, d, ld);
    LAUNCHED();
    cudaError_t e = cudaGetLastError();
    if (e == cudaSuccess && staged) e = cudaMemcpyAsync(vectors, dv, bytes, cudaMemcpyDeviceToHost, st);
    if (e == cudaSuccess && staged) e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(NIDX_ECUDA, "normalize failed: %s", cudaGetErrorString(e));
    return 0;
}

void nidx_vec_close(nidx_vec_segment* s) {
    if (!s) return;
    cudaSetDevice(s->cfg.device);
    cudaDeviceSynchronize();
    delete s;
}

uint64_t nidx_vec_len(const nidx_vec_segment* s) { return s ? s->n : 0; }
const float* nidx_vec_device_vectors(const nidx_vec_segment* s, int32_t* ld_out) {
    if (!s) return nullptr;
    if (ld_out) *ld_out = s->ld;
    return s->d_vecs;
}

int nidx_vec_set_alive(nidx_vec_segment* s, const uint64_t* alive_bits, int mem) {
    if (!s) return fail(NIDX_EINVAL, "null segment");
    CU(cudaSetDevice(s->cfg.device));
    if (!alive_bits) { s->d_alive.release(); return 0; }
    size_t words = ((size_t)s->n_par + 63) / 64;
    if (!s->d_alive) ALLOC(s->d_alive, std::max<size_t>(words, 1) * 8 + 8);
    CU(cudaMemcpy(s->d_alive, alive_bits, words * 8, mem == NIDX_MEM_DEVICE ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice));
    // the number of alive paragraphs: what the reference counts per request (segment.rs:531) when there is no filter
    std::vector<uint64_t> h(words);
    if (words) CU(cudaMemcpy(h.data(), s->d_alive, words * 8, cudaMemcpyDeviceToHost));
    uint64_t cnt = 0;
    for (size_t i = 0; i < words; ++i) {
        uint64_t v = h[i];
        if ((i + 1) * 64 > s->n_par) v &= s->n_par > i * 64 ? (~0ull >> (64 - (s->n_par - i * 64))) : 0ull;
        cnt += (uint64_t)__builtin_popcountll(v);
    }
    s->alive_count = cnt;
    return 0;
}

static bool use_hnsw_cost(size_t total_nodes, size_t matching_nodes, size_t top_k, size_t M, bool has_rabitq);
int nidx_use_hnsw(uint64_t total_nodes, uint64_t matching_nodes, uint64_t top_k, int has_rabitq, int m) {
    if (matching_nodes == 0 || top_k == 0 || m <= 0) return 0;
    return use_hnsw_cost((size_t)total_nodes, (size_t)matching_nodes, (size_t)top_k, (size_t)m, has_rabitq != 0) ? 1 : 0;
}

int nidx_vec_graph_dims(const nidx_vec_segment* s, int32_t* s0, int32_t* su, uint64_t* upper_rows, uint32_t* entry_node, uint32_t* entry_layer) {
    if (!s) return fail(NIDX_EINVAL, "null segment");
    if (!s->has_graph) return fail(NIDX_ESTATE, "segment has no HNSW graph");
    if (s0) *s0 = s->s0;
    if (su) *su = s->su;
    if (upper_rows) *upper_rows = s->upper_rows;
    if (entry_node) *entry_node = s->entry_node;
    if (entry_layer) *entry_layer = s->entry_layer;
    return 0;
}

int nidx_vec_set_graph(nidx_vec_segment* s, const uint8_t* level, const uint32_t* adj0, const float* w0, const uint32_t* adjU, const float* wU) {
    if (!s || !level || !adj0) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(s->cfg.device));
    for (uint64_t i = 0; i < s->n; ++i)
        if (level[i] >= HS_MAX_LAYERS) return fail(NIDX_EINVAL, "node %llu has level %d >= %d", (unsigned long long)i, level[i], HS_MAX_LAYERS);
    int r = alloc_graph(s, level);
    if (r) return r;
    size_t n0 = (size_t)s->n * s->s0, nu = (size_t)s->upper_rows * s->su;
    CU(cudaMemcpy(s->d_adj0, adj0, n0 * 4, cudaMemcpyHostToDevice));
    if (w0) CU(cudaMemcpy(s->d_w0, w0, n0 * 4, cudaMemcpyHostToDevice));
    if (nu && adjU) CU(cudaMemcpy(s->d_adjU, adjU, nu * 4, cudaMemcpyHostToDevice));
    if (nu && wU) CU(cudaMemcpy(s->d_wU, wU, nu * 4, cudaMemcpyHostToDevice));
    s->has_graph = true;
    return 0;
}

int nidx_vec_get_graph(const nidx_vec_segment* s, uint8_t* level, uint32_t* adj0, float* w0, uint32_t* adjU, float* wU) {
    if (!s) return fail(NIDX_EINVAL, "null segment");
    if (!s->has_graph) return fail(NIDX_ESTATE, "segment has no HNSW graph");
    CU(cudaSetDevice(s->cfg.device));
    CU(cudaDeviceSynchronize());
    size_t n0 = (size_t)s->n * s->s0, nu = (size_t)s->upper_rows * s->su;
    if (level) memcpy(level, s->h_level.data(), s->n);
    if (adj0) CU(cudaMemcpy(adj0, s->d_adj0, n0 * 4, cudaMemcpyDeviceToHost));
    if (w0) CU(cudaMemcpy(w0, s->d_w0, n0 * 4, cudaMemcpyDeviceToHost));
    if (adjU && nu) CU(cudaMemcpy(adjU, s->d_adjU, nu * 4, cudaMemcpyDeviceToHost));
    if (wU && nu) CU(cudaMemcpy(wU, s->d_wU, nu * 4, cudaMemcpyDeviceToHost));
    return 0;
}

// The counters of the last search call (of the last build before any search) into out: out[i] = h[pick[i]] of the eight, the
// visited-set and closest_up overflows (h[2] + h[3]) where pick[i] is -1
static int read_counters(nidx_vec_segment* s, uint64_t* out, std::initializer_list<int> pick) {
    if (!s || !out) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(s->cfg.device));
    unsigned long long h[8];
    unsigned long long* src = s->last_counters.load();
    CU(cudaMemcpy(h, src ? src : s->d_counters, sizeof(h), cudaMemcpyDeviceToHost));
    for (int i : pick) *out++ = i < 0 ? h[2] + h[3] : h[i];
    return 0;
}
int nidx_vec_counters_ex(nidx_vec_segment* s, uint64_t out[6]) { return read_counters(s, out, {0, 1, 2, 3, 4, 5}); }
int nidx_vec_counters(nidx_vec_segment* s, uint64_t out[3]) { return read_counters(s, out, {0, 1, -1}); }
int nidx_vec_exact_rows(nidx_vec_segment* s, uint64_t* out) { return read_counters(s, out, {6}); }
int nidx_vec_scan_counters(nidx_vec_segment* s, uint64_t out[2]) { return read_counters(s, out, {6, 7}); }
// The dense walk keeps its flagged-query count in the 64 bytes before the counters (w.sched: [0] the work counter, [2] this count,
// [3] the re-run's work counter, as unsigned ints), zeroed with them
int nidx_vec_walk_reruns(nidx_vec_segment* s, uint64_t* out) {
    if (!s || !out) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(s->cfg.device));
    unsigned int h = 0;
    unsigned long long* src = s->last_counters.load();
    if (src) CU(cudaMemcpy(&h, reinterpret_cast<unsigned int*>(src - 8) + 2, sizeof(h), cudaMemcpyDeviceToHost));
    *out = h;
    return 0;
}

// ---- RaBitQ --------------------------------------------------------------------------------------
static int rabitq_check(const nidx_vec_segment* s) {
    if (s->cfg.similarity != NIDX_SIM_DOT || s->d % 64 != 0) return fail(NIDX_EINVAL, "RaBitQ needs Dot similarity and dimension %% 64 == 0 (config.rs:170-173)");
    if (s->d / 32 > RQ_MAX_WORDS32) return fail(NIDX_EINVAL, "RaBitQ: dimension above %d not supported", RQ_MAX_WORDS32 * 32);
    return 0;
}

int nidx_vec_rabitq_encode(nidx_vec_segment* s, void* stream_) {
    if (!s) return fail(NIDX_EINVAL, "null segment");
    int r = rabitq_check(s);
    if (r) return r;
    CU(cudaSetDevice(s->cfg.device));
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    s->quant_stride = rabitq_stride(s->d);
    if (!s->d_quant) ALLOC(s->d_quant, std::max<size_t>((size_t)s->n * s->quant_stride, 16));
    if (s->n) {
        rabitq_encode_kernel<<<(unsigned)((s->n + 7) / 8), 256, 0, stream>>>(s->vdev(), s->d_quant, s->quant_stride);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    CU(cudaStreamSynchronize(stream));
    return 0;
}

int nidx_vec_rabitq_codes(const nidx_vec_segment* s, uint8_t* out) {
    if (!s || !out) return fail(NIDX_EINVAL, "null argument");
    if (!s->d_quant) return fail(NIDX_ESTATE, "segment has no RaBitQ codes (call nidx_vec_rabitq_encode)");
    CU(cudaSetDevice(s->cfg.device));
    size_t rec = (size_t)s->d / 8 + 8;
    CU(cudaMemcpy2D(out, rec, s->d_quant, (size_t)s->quant_stride, rec, (size_t)s->n, cudaMemcpyDeviceToHost));
    return 0;
}

// What the RaBitQ scan and the quantised walk need of the segment
static int rabitq_ready(const nidx_vec_segment* s) {
    int r = rabitq_check(s);
    if (r) return r;
    if (!s->d_quant) return fail(NIDX_ESTATE, "segment has no RaBitQ codes (call nidx_vec_rabitq_encode)");
    return 0;
}

// The queries as [nq][ld] zero-padded rows on the device.  `queries` is device memory: the caller's, or (staged) the call's own
// copy of host rows, which is used as it is when it needs no padding.
static int upload_queries(nidx_vec_segment* s, Workspace& w, const float* queries, int nq, int ldq, bool staged, cudaStream_t stream, const float** dq) {
    *dq = queries;
    if (ldq == s->ld && staged) return 0;
    ENSURE(w.queries, (size_t)nq * s->ld * 4);
    *dq = w.queries.as<float>();
    if (ldq == s->ld) {
        CU(cudaMemcpyAsync(w.queries.p, queries, (size_t)nq * ldq * 4, cudaMemcpyDeviceToDevice, stream));
    } else {
        pad_rows_kernel<<<std::min(nq, 1024), 256, 0, stream>>>(reinterpret_cast<const unsigned char*>(queries), (size_t)ldq * 4, s->d, w.queries.as<float>(),
                                                               s->ld, (uint64_t)nq);
        LAUNCHED();
    }
    return 0;
}

// The RaBitQ query planes and parameters of the padded queries, in w.misc
static int rabitq_query_planes(nidx_vec_segment* s, Workspace& w, const float* dq, int nq, cudaStream_t stream, uint32_t** planes, RabitqQueryParams** params) {
    size_t plane_bytes = ((size_t)nq * 4 * (s->d / 32) * 4 + 15) / 16 * 16;
    ENSURE(w.misc, plane_bytes + (size_t)nq * sizeof(RabitqQueryParams) + 64);
    *planes = w.misc.as<uint32_t>();
    *params = reinterpret_cast<RabitqQueryParams*>(w.misc.as<unsigned char>() + plane_bytes);
    rabitq_query_kernel<<<(nq + 7) / 8, 256, 0, stream>>>(dq, s->ld, s->d, nq, *planes, *params);
    LAUNCHED();
    return 0;
}

int nidx_vec_rabitq_estimate(nidx_vec_segment* s, const float* queries, int32_t nq, int32_t ldq, int mem, float* out_est, float* out_err, void* stream_) {
    if (!s || !queries || !out_est || !out_err || nq <= 0) return fail(NIDX_EINVAL, "bad argument");
    if (!s->d_quant) return fail(NIDX_ESTATE, "segment has no RaBitQ codes (call nidx_vec_rabitq_encode)");
    if (ldq < s->d) return fail(NIDX_EINVAL, "query dimension %d != index dimension %d", ldq, s->d);
    CU(cudaSetDevice(s->cfg.device));
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    WsGuard g(s->pool, stream);
    Workspace& w = *g.w;
    const bool host = mem == NIDX_MEM_HOST;
    Stage st(stream, host, host);
    const float* d_q;
    float *d_est, *d_err;
    st.in(queries, (size_t)nq * ldq, &d_q);
    st.out(out_est, (size_t)nq * s->n, &d_est);
    st.out(out_err, (size_t)nq * s->n, &d_err);
    int r = st.place(w.stage);
    const float* dq;
    if (!r) r = upload_queries(s, w, d_q, nq, ldq, host, stream, &dq);
    uint32_t* planes; RabitqQueryParams* params;
    if (!r) r = rabitq_query_planes(s, w, dq, nq, stream, &planes, &params);
    if (r) return r;
    if (s->n) {
        rabitq_estimate_kernel<<<dim3((unsigned)((s->n + 255) / 256), nq), 256, 0, stream>>>(s->d_quant, s->quant_stride, (uint32_t)s->n, s->d, planes, params, d_est, d_err);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    return st.finish();
}

int nidx_vec_last_kernel_ms(nidx_vec_segment* s, float* ms) {
    if (!s || !ms) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(s->cfg.device));
    CU(cudaEventSynchronize(s->ev_k1));
    CU(cudaEventElapsedTime(ms, s->ev_k0, s->ev_k1));
    return 0;
}

// ---- search -----------------------------------------------------------------------------------
// segment.rs:626-660: estimated vector evaluations of the HNSW walk vs the exhaustive scan; with RaBitQ codes a raw
// vector costs 16 quantised ones, layer 0 is searched for RERANKING_FACTOR * 3/4 times more nodes and
// RERANKING_FACTOR / 2 candidates per result are reranked (rabitq.rs:34).
static bool use_hnsw_cost(size_t total_nodes, size_t matching_nodes, size_t top_k, size_t M, bool has_rabitq) {
    const size_t RERANKING_FACTOR = 100;
    size_t full_cost = has_rabitq ? 16 : 1, search_mult = has_rabitq ? RERANKING_FACTOR * 3 / 4 : 1, rerank_mult = has_rabitq ? RERANKING_FACTOR / 2 : 0;
    float l = logf((float)total_nodes) - 2.0f;
    float hnsw_rq = l * l * logf((float)top_k) * (float)search_mult;
    size_t hnsw_full = top_k * rerank_mult + top_k * M * total_nodes / std::max<size_t>(matching_nodes, 1);
    size_t hnsw_cost = (size_t)(hnsw_rq < 0 ? 0 : hnsw_rq) + hnsw_full * full_cost;   // `as usize` saturates a negative estimate to 0
    size_t bf_cost = matching_nodes + top_k * rerank_mult * full_cost;
    return hnsw_cost < bf_cost;
}

__global__ void and_bits_kernel(const uint64_t* a, const uint64_t* b, uint64_t* out, size_t words, unsigned long long* count) {
    unsigned long long local = 0;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < words; i += (size_t)gridDim.x * blockDim.x) {
        uint64_t v = a[i] & (b ? b[i] : ~0ull);
        out[i] = v;
        local += __popcll(v);
    }
    for (int off = 16; off >= 1; off >>= 1) local += __shfl_xor_sync(0xFFFFFFFFu, local, off);
    if (count && (threadIdx.x & 31) == 0 && local) atomicAdd(count, local);
}

// Shared-memory plans of the two walks, used by AUTO's choice and by the launch alike.  Each returns false when the plan does not
// fit one CTA (the list and the visited set grow with ef and k).
static bool hnsw_search_smem(const nidx_vec_segment* s, int ef0, int k, int* list_cap, int* cu_cap, int* hash_bits, size_t* bytes) {
    // closest_up_nodes pops at most k-1 candidates before it has k results when nothing is filtered
    // (search.rs:205-216), each adding at most one adjacency row of pending candidates.
    int cu = std::min(std::max(ef0 + k * s->s0, 2 * ef0), 4096);
    int lc = std::max(ef0, cu);
    // visited-set slots: a walk visits about ef0 * s0 * 0.6 nodes on easy data and up to ~1.3x that on clustered data at small ef
    // (10 M x 768, 4096 centres, ef = 30: 13 of 1024 queries overflowed 2048 slots): at least 4096, 1.5 x ef0 x s0 above that
    int slots = next_pow2(std::max(4096, (ef0 * s->s0 * 3) / 2));
    slots = std::max(slots, next_pow2(4 * lc));
    *list_cap = lc; *cu_cap = cu; *hash_bits = ilog2(slots);
    *bytes = hs_smem_bytes(s->ld, lc, *hash_bits);
    return *bytes <= 200 * 1024;
}

// log2 of the smallest visited table whose insert limit (VisitedSet::init) stays above n nodes: a walk on it never overflows.
// At most 28: VisitedSet::init computes the limit in 32 bits (a 2^28-slot table already holds 251 M nodes, 1 GiB per CTA).
static int rq_table_bits(uint64_t n) {
    int b = 1;
    while (b < 28 && ((15ull << b) >> 4) < n + 1 + HS_MAX_ROW) ++b;
    return b;
}

static bool rq_walk_smem(const nidx_vec_segment* s, int k, int* last_k, int* cu_cap, int* list_cap, int* hash_bits, size_t* bytes) {
    *last_k = (int)std::min<size_t>((size_t)k * 100, 2000);              // rabitq.rs:34-36 RERANKING_FACTOR / RERANKING_LIMIT
    *cu_cap = std::min(std::max(k + k * s->s0, 2 * k), 4096);
    *list_cap = std::max(*last_k, *cu_cap);
    *hash_bits = ilog2(next_pow2(std::max(2048, 4 * *cu_cap)));
    *bytes = rq_smem_bytes(s->ld, s->d, *list_cap, *hash_bits, k);
    return *bytes <= 200 * 1024;
}

}  // extern "C"

// The vector kernels are instantiated for the common row lengths, ld = NG * 128 floats with NG among NGs; other dimensions use the
// run-time loop (NG = 0).  `inst(std::integral_constant<int, NG>())` names the instance.
template <int... NGs, typename F>
static auto pick_ng(int ld, F inst) {
    auto k = inst(std::integral_constant<int, 0>());
    auto match = [&](auto ng) { if (ld == ng * 128) k = inst(ng); };
    (match(std::integral_constant<int, NGs>()), ...);
    return k;
}

typedef void (*hs_kernel_t)(VecDev, GraphDev, SearchArgs);
// defer: closest_up_nodes may settle neighbours on the kept layer-0 set (hnsw_search_kernel's DEFER)
static hs_kernel_t pick_search_kernel(int ld, bool defer = false) {
    return pick_ng<1, 2, 3, 4, 6, 8>(ld, [defer](auto ng) -> hs_kernel_t { return defer ? hnsw_search_kernel<ng, true> : hnsw_search_kernel<ng>; });
}
// the dense walk's re-run of its flagged queries (hnsw_search_kernel's RERUN)
static hs_kernel_t pick_rerun_kernel(int ld) {
    return pick_ng<1, 2, 3, 4, 6, 8>(ld, [](auto ng) -> hs_kernel_t { return hnsw_search_kernel<ng, false, true>; });
}

// w4: the 4-warp CTA shape (quantised_walk)
static hs_kernel_t pick_rabitq_walk_kernel(int ld, bool w4) {
    return pick_ng<2, 3, 4, 6, 8>(ld, [w4](auto ng) -> hs_kernel_t { return w4 ? hnsw_rabitq_kernel<ng, 4> : hnsw_rabitq_kernel<ng>; });
}

// four vectors in flight per warp for rows of up to 384 floats, two for longer ones
typedef void (*scan_kernel_t)(VecDev, const float*, const float*, int, int, float*);
static scan_kernel_t pick_scan_kernel(int ld) {
    return pick_ng<1, 2, 3, 4, 6, 8>(ld, [](auto ng) -> scan_kernel_t {
        if constexpr (ng == 0) return scan_scores_kernel;
        else return scan_scores_kernel_t<ng, ng <= 3 ? 4 : 2>;
    });
}

// ---- filters on the device: running a program of prefilter.cuh ----------------------------------------------------------
// One run of a compiled program over n_docs documents (A: the document columns the program reads and the alive set; paragraphs have
// no columns).  w.prefilter holds [n_slots][words] leaf bitsets | the match count | the program | extra_bytes of the caller's leaf
// data; scatter(slot bits, extra) sets the slots once they are zeroed.  The result goes to out ([words], padding bits zero) and the
// number of its set bits to *h_count; the caller synchronises before either is read and before the program's storage goes.  A
// program that is one bitset leaf is ANDed with alive by and_bits_kernel instead of the pass.  ev0 / ev1 (optional) time that kernel or the pass.
template <class Scatter>
static int run_program(Workspace& w, cudaStream_t stream, int sm_count, const std::vector<PfOp>& prog, size_t n_slots, PrefilterArgs A,
                       size_t extra_bytes, Scatter scatter, uint64_t* out, unsigned long long* h_count, cudaEvent_t ev0 = nullptr,
                       cudaEvent_t ev1 = nullptr) {
    if (prog.size() > (size_t)PF_MAX_PROGRAM) return fail(NIDX_EINVAL, "the filter program has more than %d instructions", PF_MAX_PROGRAM);
    const size_t words = A.words;
    const size_t o_count = (n_slots * words * 8 + 15) & ~(size_t)15, o_prog = o_count + 16, o_extra = o_prog + prog.size() * sizeof(PfOp);
    ENSURE(w.prefilter, o_extra + extra_bytes);
    uint64_t* bits = w.prefilter.as<uint64_t>();
    unsigned long long* d_count = reinterpret_cast<unsigned long long*>(w.prefilter.p + o_count);
    PfOp* d_prog = reinterpret_cast<PfOp*>(w.prefilter.p + o_prog);
    CU(cudaMemsetAsync(d_count, 0, 8, stream));
    if (n_slots && words) {
        CU(cudaMemsetAsync(bits, 0, n_slots * words * 8, stream));
        int r = scatter(bits, w.prefilter.p + o_extra);
        if (r) return r;
    }
    if (prog.size() == 1 && prog[0].op == PF_BITS) {
        if (ev0) CU(cudaEventRecord(ev0, stream));
        and_bits_kernel<<<(unsigned)std::max<size_t>(1, std::min<size_t>((words + 255) / 256, 1024)), 256, 0, stream>>>(
            bits + (size_t)prog[0].arg * words, A.alive, out, words, d_count);
    } else {
        CU(cudaMemcpyAsync(d_prog, prog.data(), prog.size() * sizeof(PfOp), cudaMemcpyHostToDevice, stream));
        A.kw_bits = bits; A.prog = d_prog; A.n_prog = (uint32_t)prog.size(); A.out = reinterpret_cast<uint32_t*>(out); A.count = d_count;
        const size_t smem = prog.size() * sizeof(PfOp);
        CU(cudaFuncSetAttribute(prefilter_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        if (ev0) CU(cudaEventRecord(ev0, stream));
        const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)sm_count * 8, (2 * words * 32 + PF_THREADS - 1) / PF_THREADS));
        prefilter_eval_kernel<<<blocks, PF_THREADS, smem, stream>>>(A);
    }
    LAUNCHED();
    if (ev1) CU(cudaEventRecord(ev1, stream));
    CU(cudaGetLastError());
    CU(cudaMemcpyAsync(h_count, d_count, 8, cudaMemcpyDeviceToHost, stream));
    return 0;
}

static int cmp_key(const unsigned char* a, size_t la, const unsigned char* b, size_t lb) {
    int c = memcmp(a, b, std::min(la, lb));
    return c ? c : (la < lb ? -1 : (la > lb ? 1 : 0));
}
// The postings [*b, *e) of key q: get_prefix (every key that starts with q) for the label index, get (the exact key) for the fields
static void key_postings(const nidx_vec_segment::InvIndex& ix, bool prefix, const unsigned char* q, size_t lq, uint64_t* b, uint64_t* e) {
    uint32_t lo = 0, hi = ix.n_keys;
    while (lo < hi) {   // the first key >= q
        uint32_t mid = (lo + hi) / 2;
        if (cmp_key(ix.key_bytes.data() + ix.key_off[mid], ix.key_off[mid + 1] - ix.key_off[mid], q, lq) < 0) lo = mid + 1; else hi = mid;
    }
    if (prefix) {
        for (uint32_t c = ix.n_keys; hi < c;) {
            uint32_t mid = (hi + c) / 2;
            size_t lk = ix.key_off[mid + 1] - ix.key_off[mid];
            if (lk >= lq && memcmp(ix.key_bytes.data() + ix.key_off[mid], q, lq) == 0) hi = mid + 1; else c = mid;
        }
    } else if (lo < ix.n_keys && cmp_key(ix.key_bytes.data() + ix.key_off[lo], ix.key_off[lo + 1] - ix.key_off[lo], q, lq) == 0) {
        hi = lo + 1;
    }
    *b = ix.post_off[lo]; *e = ix.post_off[hi];
}

// ParagraphInvertedIndexes::filter (inverted_index/paragraph.rs:124-186) as a program over the segment's paragraphs.  The key lookups
// (the fst's job in the reference) run here; every atom that finds postings is a bitset leaf whose ranges set its slot, and the
// atoms that are operands of one OR share a slot (the union of their ranges is the OR).  An atom without postings is the constant 0.
// AND / OR of n operands are n - 1 binary ops, NOT the complement of its operands' intersection (paragraph.rs:160-178).  Operands
// are emitted heaviest first (Sethi-Ullman), so the bit stack never holds more than log2(leaves) + 1 entries.
struct FormulaPlan {
    const nidx_vec_segment* s = nullptr;
    const nidx_filter_node* nodes = nullptr;
    int n_nodes = 0;
    uint32_t slots = 0;                                  // slots below the first one the formula takes belong to the caller
    std::vector<uint64_t> ranges[2];                     // per inverted index (NIDX_INV_*): [2 r] posting ranges
    std::vector<uint32_t> range_slot[2];                 // and the slot each one sets
    std::vector<PfOp> prog;

    static bool atom(const nidx_filter_node& nd) { return nd.kind == NIDX_F_LABEL || nd.kind == NIDX_F_KEYS; }
    static PfOp leaf(int slot) {   // slot < 0: no postings
        PfOp o{};
        o.op = slot >= 0 ? PF_BITS : PF_CONST;
        o.arg = slot >= 0 ? (uint32_t)slot : 0;
        return o;
    }
    // the atom's ranges into `slot`; false when it has no postings
    bool lookup(const nidx_filter_node& nd, uint32_t slot) {
        const int which = nd.kind == NIDX_F_LABEL ? NIDX_INV_LABELS : NIDX_INV_FIELDS;
        bool any = false;
        for (int j = 0; j < nd.n; ++j) {
            uint64_t b, e;
            key_postings(s->inv[which], nd.kind == NIDX_F_LABEL, nd.keys[j], nd.key_len[j], &b, &e);
            if (e > b) { ranges[which].push_back(b); ranges[which].push_back(e); range_slot[which].push_back(slot); any = true; }
        }
        return any;
    }
    // the subtree at node i -> its program (code) and the bit stack entries it needs; returns the node after it, or -1 when the
    // operand counts do not add up
    int plan(int i, std::vector<PfOp>& code, int& need) {
        const nidx_filter_node& nd = nodes[i];
        need = 1;
        if (atom(nd)) { code.assign(1, leaf(lookup(nd, slots) ? (int)slots++ : -1)); return i + 1; }
        std::vector<std::pair<int, std::vector<PfOp>>> v;   // the operands: need, code
        int or_slot = -1, j = i + 1;                        // or_slot: the slot of this OR's atoms
        bool or_atoms = false;
        for (int c = 0; c < nd.n; ++c) {
            if (j >= n_nodes) return -1;
            if (nd.kind == NIDX_F_OR && atom(nodes[j])) {
                or_atoms = true;
                if (lookup(nodes[j++], or_slot >= 0 ? (uint32_t)or_slot : slots) && or_slot < 0) or_slot = (int)slots++;
                continue;
            }
            v.emplace_back();
            j = plan(j, v.back().second, v.back().first);
            if (j < 0) return -1;
        }
        if (or_atoms) v.push_back({1, {leaf(or_slot)}});
        std::stable_sort(v.begin(), v.end(), [](const auto& a, const auto& b) { return a.first > b.first; });
        need = v.size() > 1 ? std::max(v[0].first, v[1].first + 1) : v[0].first;
        code = std::move(v[0].second);
        PfOp op{};
        op.op = nd.kind == NIDX_F_OR ? PF_OR : PF_AND;   // Not | And => intersect (paragraph.rs:160-164)
        for (size_t c = 1; c < v.size(); ++c) {
            code.insert(code.end(), v[c].second.begin(), v[c].second.end());
            code.push_back(op);
        }
        if (nd.kind == NIDX_F_NOT) { op.op = PF_NOT; code.push_back(op); }
        return j;
    }
    int compile(const nidx_vec_segment* seg, const nidx_filter_node* nd, int n) {
        s = seg; nodes = nd; n_nodes = n;
        if (!nodes || n_nodes <= 0) return fail(NIDX_EINVAL, "empty filter formula");
        for (int i = 0; i < n_nodes; ++i) {
            int kd = nodes[i].kind;
            if (kd < NIDX_F_LABEL || kd > NIDX_F_NOT || nodes[i].n < 0) return fail(NIDX_EINVAL, "filter node %d: bad kind / count", i);
            if ((kd == NIDX_F_LABEL || kd == NIDX_F_KEYS) && nodes[i].n > 0 && (!nodes[i].keys || !nodes[i].key_len)) return fail(NIDX_EINVAL, "filter node %d: null keys", i);
            if ((kd == NIDX_F_AND || kd == NIDX_F_OR || kd == NIDX_F_NOT) && nodes[i].n < 1) return fail(NIDX_EINVAL, "filter node %d: a compound clause needs operands", i);
        }
        int need;
        if (plan(0, prog, need) != n_nodes) return fail(NIDX_EINVAL, "malformed filter formula (operand counts do not add up to %d nodes)", n_nodes);
        // at most log2(leaves) + 1 <= 13 within the program limit; one entry stays free for nidx_vec_prefilter_bits' combination
        if (need >= PF_MAX_DEPTH) return fail(NIDX_EINVAL, "the filter formula needs more than %d bit stack entries", PF_MAX_DEPTH - 1);
        return 0;
    }
    // leaf data in w.prefilter after the program: the ranges of both indexes, then their slots
    size_t extra_bytes() const { return (range_slot[0].size() + range_slot[1].size()) * 20; }
    int scatter(uint64_t* bits, unsigned char* extra, size_t words, cudaStream_t stream) const {
        const size_t n0 = range_slot[0].size(), n = n0 + range_slot[1].size();
        if (!n) return 0;
        uint64_t* d_ranges = reinterpret_cast<uint64_t*>(extra);
        uint32_t* d_slot = reinterpret_cast<uint32_t*>(extra + n * 16);
        for (int which = 0, at = 0; which < 2; at += (int)range_slot[which++].size()) {
            if (range_slot[which].empty()) continue;
            CU(cudaMemcpyAsync(d_ranges + 2 * at, ranges[which].data(), range_slot[which].size() * 16, cudaMemcpyHostToDevice, stream));
            CU(cudaMemcpyAsync(d_slot + at, range_slot[which].data(), range_slot[which].size() * 4, cudaMemcpyHostToDevice, stream));
        }
        prefilter_scatter_kernel<<<(unsigned)n, 256, 0, stream>>>(s->inv[NIDX_INV_LABELS].d_post.p, s->inv[NIDX_INV_FIELDS].d_post.p, (uint32_t)n0, nullptr,
                                                                   0, nullptr, d_ranges, d_slot, 0, bits, words);
        LAUNCHED();
        return 0;
    }
};

static PrefilterArgs paragraph_args(const nidx_vec_segment* s) {
    PrefilterArgs A{};
    A.n_docs = (uint32_t)s->n_par; A.words = ((size_t)s->n_par + 63) / 64; A.alive = s->d_alive;
    return A;
}

// filter ∧ alive (segment.rs:516-534) into w.filter ([words] bits | its match count), returned in *bits.  With h_count, the number of
// set bits is copied back to it (the caller synchronises).
static int filter_and_alive(nidx_vec_segment* s, Workspace& w, const uint64_t* filter, unsigned long long* h_count, cudaStream_t stream,
                            const uint64_t** bits) {
    const size_t words = ((size_t)s->n_par + 63) / 64;
    ENSURE(w.filter, (words + 8) * 8);
    uint64_t* out = w.filter.as<uint64_t>();
    unsigned long long* count = reinterpret_cast<unsigned long long*>(out + words);
    CU(cudaMemsetAsync(count, 0, 8, stream));
    and_bits_kernel<<<std::min<size_t>((words + 255) / 256, 1024), 256, 0, stream>>>(filter, s->d_alive, out, words, count);
    LAUNCHED();
    if (h_count) CU(cudaMemcpyAsync(h_count, count, 8, cudaMemcpyDeviceToHost, stream));
    *bits = out;
    return 0;
}

// ParagraphInvertedIndexes::filter ∧ alive on the device (segment.rs:516-531): nodes (pre-order; several top-level nodes are not
// allowed: wrap them in an AND / OR node) -> out, the number of matches -> *h_count.  Returns with the stream synchronised.
static int filter_formula(nidx_vec_segment* s, Workspace& w, const nidx_filter_node* nodes, int n_nodes, cudaStream_t stream, uint64_t* out,
                          unsigned long long* h_count) {
    FormulaPlan P;
    int r = P.compile(s, nodes, n_nodes);
    if (r) return r;
    const PrefilterArgs A = paragraph_args(s);
    r = run_program(w, stream, s->sm_count, P.prog, P.slots, A, P.extra_bytes(),
                    [&](uint64_t* bits, unsigned char* extra) { return P.scatter(bits, extra, A.words, stream); }, out, h_count);
    if (r) return r;
    CU(cudaStreamSynchronize(stream));   // the program and the ranges are host temporaries
    return 0;
}

// The tensor-core filter + refine path serves large batches of small-k queries on single-vector segments whose rows are whole
// 128-byte swizzle rows.  NIDX_B200_SCAN=exact forces the CUDA-core kernels (same results, bit for bit), =tensor forces the filter.
// Rows outside the filter's error bound (a non-finite norm, a tiny cosine row) keep the whole segment on the CUDA-core kernels.
static bool use_tc_filter(const nidx_vec_segment* s, int nq, int k) {
    if (k > TC2_KMAX || s->ld % TC2_KB != 0 || s->d_par_first || s->n < (uint64_t)TC2_N || s->cfg.similarity == NIDX_SIM_L2 || !s->tc_rows_ok) return false;
    const char* e = getenv("NIDX_B200_SCAN");
    if (e && !strcmp(e, "exact")) return false;
    if (e && !strcmp(e, "tensor")) return true;
    return nq >= 64;
}

// One vector search call as its method sees it: the padded queries and their norms, filter ∧ alive (NULL: every paragraph), the
// outputs (device pointers) and this call's counters.
struct VecCall {
    nidx_vec_segment* s;
    Workspace& w;
    cudaStream_t stream;
    const nidx_vec_search_params* p;
    VecDev V;
    int nq, k;
    const float* dq;
    float* qnorms;
    const uint64_t* bits;
    uint32_t* ids;
    float* scores;
    int* counts;
    unsigned long long* counters;   // [8], zeroed for this call; the 64 bytes before them (w.sched) hold the kernels' work counter

    // Every id NIDX_NIL, every score and count 0
    int write_empty() const {
        CU(cudaMemsetAsync(ids, 0xFF, (size_t)nq * k * 4, stream));
        CU(cudaMemsetAsync(scores, 0, (size_t)nq * k * 4, stream));
        CU(cudaMemsetAsync(counts, 0, (size_t)nq * 4, stream));
        return 0;
    }

    // segment.rs:581-608 with SearchVector::RabitQ: estimate every vector from its 1-bit code, keep upper_bound >= min_score,
    // rerank_top with the raw vectors (sequential semantics preserved, see rabitq_rerank_kernel)
    int rabitq_scan() {
        int r = rabitq_ready(s);
        if (r) return r;
        if (s->d_par_first) return fail(NIDX_EINVAL, "RaBitQ scan of multi-vector paragraphs is not implemented");
        if (k > 1024) return fail(NIDX_EINVAL, "k above 1024 not supported");
        uint32_t* planes; RabitqQueryParams* params;
        r = rabitq_query_planes(s, w, dq, nq, stream, &planes, &params);
        if (r) return r;
        int qgroup = (int)std::max<size_t>(1, std::min<size_t>((size_t)nq, ((size_t)4 << 30) / ((size_t)s->n * 8)));
        ENSURE(w.scores, (size_t)qgroup * s->n * 8);
        size_t smem_rr = rr_smem_bytes(s->ld, k);
        CU(cudaFuncSetAttribute(rabitq_rerank_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rr));
        for (int q0 = 0; q0 < nq; q0 += qgroup) {
            int nqg = std::min(qgroup, nq - q0);
            float* d_est = w.scores.as<float>();
            float* d_err = d_est + (size_t)nqg * s->n;
            if (q0 == 0) CU(cudaEventRecord(s->ev_k0, stream));
            const uint32_t* qplanes = planes + (size_t)q0 * 4 * (s->d / 32);
            rabitq_estimate_kernel<<<dim3((unsigned)((s->n + 255) / 256), nqg), 256, 0, stream>>>(s->d_quant, s->quant_stride, (uint32_t)s->n, s->d, qplanes,
                                                                                                     params + q0, d_est, d_err);
            if (q0 == 0) CU(cudaEventRecord(s->ev_k1, stream));
            LAUNCHED();
            rabitq_rerank_kernel<<<nqg, RR_THREADS, smem_rr, stream>>>(V, dq + (size_t)q0 * s->ld, d_est, d_err, bits, p->min_score, k,
                                                                         ids + (size_t)q0 * k, scores + (size_t)q0 * k, counts + q0, nullptr);
            LAUNCHED();
        }
        CU(cudaGetLastError());
        return 0;
    }

    // Large batches: TF32 tensor-core filter + bit-exact refine (scan_tc2.cuh); nothing of size [Q x N] touches HBM
    int tc_filter_scan() {
        int n_chunks = (int)((s->n + TC2_CHUNK - 1) / TC2_CHUNK), n_qblocks = (nq + TC2_M - 1) / TC2_M;
        {
            std::lock_guard<std::mutex> lk(s->map_mu);
            if (!s->map_v_ready) {
                int mr = make_row_tensor_map(&s->map_v, s->d_vecs, s->n, s->ld, TC2_N);
                if (mr) return mr;
                s->map_v_ready = true;
            }
        }
        CUtensorMap map_q;
        int mr = make_row_tensor_map(&map_q, dq, (uint64_t)nq, s->ld, TC2_M);
        if (mr) return mr;
        int grid = std::min(n_chunks * n_qblocks, s->sm_count);
        int slots = std::max(1, std::min(grid / n_qblocks, n_chunks));   // CTAs per query block; 1 when there are more blocks than CTAs
        size_t cand_n = (size_t)nq * slots * TC2_LISTS * TC2_L;
        ENSURE(w.scores, cand_n * 8 + 64);
        Tc2Args ta;
        ta.nq = nq; ta.n_qblocks = n_qblocks; ta.n_chunks = n_chunks; ta.slots = slots; ta.qnorms = qnorms; ta.bits = bits;
        ta.cand_score = w.scores.as<float>(); ta.cand_id = reinterpret_cast<uint32_t*>(w.scores.as<float>() + cand_n);
        ta.work_counter = w.sched.as<unsigned int>();
        CU(cudaFuncSetAttribute(scan_tc_filter_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)TC2_SMEM_BYTES));
        grid = n_qblocks <= grid ? n_qblocks * slots : grid;
        CU(cudaEventRecord(s->ev_k0, stream));
        scan_tc_filter_kernel<<<grid, TC2_THREADS, TC2_SMEM_BYTES, stream>>>(map_q, s->map_v, V, ta);
        CU(cudaEventRecord(s->ev_k1, stream));
        LAUNCHED();
        int cap = topk_cap(k, 256);
        size_t smem_rf = tc2_refine_smem(s->ld, cap);
        if (smem_rf > 48 * 1024) CU(cudaFuncSetAttribute(scan_tc_refine_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rf));
        scan_tc_refine_kernel<<<nq, 256, smem_rf, stream>>>(V, dq, qnorms, slots * TC2_LISTS, ta.cand_score, ta.cand_id, bits, s->max_norm,
                                                              p->min_score, k, cap, ids, scores, counts, counters + 6);
        LAUNCHED();
        CU(cudaGetLastError());
        return 0;
    }

    // The exhaustive scan on the CUDA cores: score matrix per query group, per-chunk top-k, merge
    int exact_scan() {
        if (k > 1024) return fail(NIDX_EINVAL, "brute-force k above 1024 not supported");
        int cap = topk_cap(k, 256);
        int n_chunks = (int)std::min<uint64_t>(std::max<uint64_t>(1, ((uint64_t)s->sm_count * 4 + nq - 1) / nq), (s->n_par + 4095) / 4096);
        n_chunks = std::max(n_chunks, 1);
        // bound the score matrix: process queries in groups
        size_t max_score_bytes = (size_t)4 << 30;
        int qgroup = (int)std::max<size_t>(1, std::min<size_t>((size_t)nq, max_score_bytes / ((size_t)s->n * 4)));
        qgroup = std::max(SCAN_QT, qgroup / SCAN_QT * SCAN_QT);
        qgroup = std::min(qgroup, (nq + SCAN_QT - 1) / SCAN_QT * SCAN_QT);
        ENSURE(w.scores, (size_t)qgroup * s->n * 4);
        ENSURE(w.partial, (size_t)qgroup * n_chunks * k * 8);
        size_t smem_scan = (size_t)SCAN_QT * s->ld * 4;
        scan_kernel_t scan_kern = pick_scan_kernel(s->ld);
        if (smem_scan > 48 * 1024) CU(cudaFuncSetAttribute(scan_kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_scan));
        if ((size_t)cap * 8 > 48 * 1024) {
            CU(cudaFuncSetAttribute(scan_select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap * 8));
            CU(cudaFuncSetAttribute(topk_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap * 8));
        }
        for (int q0 = 0; q0 < nq; q0 += qgroup) {
            int nqg = std::min(qgroup, nq - q0);
            int n_qtiles = (nqg + SCAN_QT - 1) / SCAN_QT;
            uint64_t n_vchunks = (s->n + SCAN_WARPS * SCAN_VPW - 1) / (SCAN_WARPS * SCAN_VPW);
            uint64_t grid = n_vchunks * n_qtiles;
            if (grid > 0x7FFFFFFFull) return fail(NIDX_EINVAL, "scan grid too large");
            if (q0 == 0) CU(cudaEventRecord(s->ev_k0, stream));
            scan_kern<<<(unsigned)grid, SCAN_WARPS * 32, smem_scan, stream>>>(V, dq + (size_t)q0 * s->ld, qnorms + q0, nqg, n_qtiles, w.scores.as<float>());
            if (q0 == 0) CU(cudaEventRecord(s->ev_k1, stream));
            LAUNCHED();
            scan_select_kernel<<<dim3(n_chunks, nqg), 256, (size_t)cap * 8, stream>>>(w.scores.as<float>(), (uint32_t)s->n, s->n_par, s->d_par_first, nullptr,
                                                                                        bits, p->min_score, k, cap, n_chunks, w.partial.as<uint64_t>());
            LAUNCHED();
            topk_merge_kernel<<<nqg, 256, (size_t)cap * 8, stream>>>(w.partial.as<uint64_t>(), n_chunks * k, k, cap, ids + (size_t)q0 * k,
                                                                       scores + (size_t)q0 * k, counts + q0);
            LAUNCHED();
        }
        CU(cudaGetLastError());
        return 0;
    }

    // SearchArgs of a walk (mode 0) of this call
    SearchArgs walk_args(int ef0, int list_cap, int cu_cap, int hash_bits) const {
        SearchArgs a;
        memset(&a, 0, sizeof(a));
        a.mode = 0; a.nq = nq; a.queries = dq; a.qnorms = qnorms; a.k = k; a.ef0 = ef0; a.min_score = p->min_score;
        a.with_duplicates = p->with_duplicates; a.multi_vector = s->cfg.multi_vector; a.filter = bits;
        a.out_ids = ids; a.out_scores = scores; a.out_counts = counts;
        a.hash_bits = hash_bits; a.list_cap = list_cap; a.cu_cap = cu_cap;
        a.work_counter = w.sched.as<unsigned int>();   // the scheduler counter lives in the workspace: concurrent calls must not share it
        a.counters = counters;
        return a;
    }

    // The grid of a walk: as many CTAs as are resident at once, at most one per query
    int walk_grid(hs_kernel_t kern, int threads, size_t smem, int* grid) const {
        CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        int occ = 0;
        CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, threads, smem));
        *grid = std::min(nq, std::max(1, occ) * s->sm_count);
        return 0;
    }

    int launch_walk(hs_kernel_t kern, int grid, int threads, size_t smem, const VecDev& Vw, const SearchArgs& a) const {
        CU(cudaEventRecord(s->ev_k0, stream));
        kern<<<grid, threads, smem, stream>>>(Vw, s->gdev(), a);
        CU(cudaEventRecord(s->ev_k1, stream));
        LAUNCHED();
        CU(cudaGetLastError());
        return 0;
    }

    // hnsw/search.rs:306-383 with SearchVector::RabitQ: estimate-ranked walk, k * 100 layer-0 results, exact rerank + closest_up
    int quantised_walk() {
        int r = rabitq_ready(s);
        if (r) return r;
        uint32_t* planes; RabitqQueryParams* params;
        r = rabitq_query_planes(s, w, dq, nq, stream, &planes, &params);
        if (r) return r;
        int last_k, cu_cap, list_cap, hash_bits;
        size_t smem;
        if (!rq_walk_smem(s, k, &last_k, &cu_cap, &list_cap, &hash_bits, &smem))
            return fail(NIDX_EINVAL, "quantised HNSW search needs %zu bytes of shared memory (k=%d, dim=%d): too large", smem, k, s->d);
        // Layer 0's visited set is a table in global memory, one slice per resident CTA.  A walk estimates about 0.5 x last_k x s0
        // nodes, up to 0.6 x on hard data (500 000 x 64 Dot rows, M0 = 60, k = 20: 74 391 of last_k x s0 = 128 000), so the table has
        // 1.5 x last_k x s0 slots and at least 2^16, as the dense walk sizes its shared one -- and no more than the smallest table whose
        // insert limit holds every node of the segment, which cannot overflow.
        const int all_bits = rq_table_bits(s->n);
        int gv_bits = std::min(ilog2(next_pow2(std::max(1 << 16, last_k * s->s0 * 3 / 2))), all_bits);
        if (const char* eg = getenv("NIDX_B200_RQ_GV_BITS")) gv_bits = std::min(all_bits, std::max(8, atoi(eg)));   // tests: a smaller table
        // CTA shape: the walk is bound by the ~1 000 dependent hops of a query, so what counts is how many queries are resident.
        // 8 warps per query: 4 CTAs per SM; 4 warps: 7 per SM.  The 4-warp shape is taken when the batch does not fit one wave of the
        // 8-warp shape (NIDX_B200_RQ_W = 4 / 8 forces one).
        hs_kernel_t kern = pick_rabitq_walk_kernel(s->ld, false);
        int threads = HS_THREADS, grid = 0;
        r = walk_grid(kern, threads, smem, &grid);
        const char* ew = getenv("NIDX_B200_RQ_W");
        const int force = ew ? atoi(ew) : 0;
        if (!r && (force == 4 || (force != 8 && nq > grid))) {
            kern = pick_rabitq_walk_kernel(s->ld, true);
            threads = 128;
            r = walk_grid(kern, threads, smem, &grid);
        }
        if (r) return r;
        ENSURE(w.scores, ((size_t)grid << gv_bits) * 4);
        SearchArgs a = walk_args(last_k, list_cap, cu_cap, hash_bits);
        a.codes = s->d_quant; a.code_stride = s->quant_stride; a.planes = planes; a.qparams = params;
        a.gvisited = w.scores.as<uint32_t>(); a.gv_bits = gv_bits; a.last_k = last_k;
        r = launch_walk(kern, grid, threads, smem, V, a);
        if (r || gv_bits == all_bits) return r;
        // A full table reports its new nodes as visited, and the walk would skip neighbours the reference scores.  When a query
        // overflowed the layer-0 table (counters[7]; the shared-memory sets count in [2] only), the batch runs again with the table
        // that holds every node, on as many CTAs as fit the workspace the first run used (at least 1 GiB).
        unsigned long long overflows = 0;
        CU(cudaMemcpyAsync(&overflows, counters + 7, sizeof(overflows), cudaMemcpyDeviceToHost, stream));
        CU(cudaStreamSynchronize(stream));
        if (!overflows) return 0;
        const size_t budget = std::max(((size_t)grid << gv_bits) * 4, (size_t)1 << 30);
        grid = (int)std::max<size_t>(1, std::min<size_t>((size_t)grid, budget / (((size_t)4) << all_bits)));
        ENSURE(w.scores, ((size_t)grid << all_bits) * 4);
        CU(cudaMemsetAsync(w.sched.p, 0, 128, stream));              // the work counter and this call's counters
        a.gvisited = w.scores.as<uint32_t>(); a.gv_bits = all_bits;
        return launch_walk(kern, grid, threads, smem, V, a);
    }

    // hnsw/search.rs:306-383 on the f32 vectors, screened on the fp16 copy when the segment has one
    int dense_walk() {
        int ef = p->ef > 0 ? p->ef : s->cfg.ef_search;
        int ef0 = std::max(k, ef);  // search.rs:338-345
        int list_cap, cu_cap, hash_bits;
        size_t smem;
        if (!hnsw_search_smem(s, ef0, k, &list_cap, &cu_cap, &hash_bits, &smem))
            return fail(NIDX_EINVAL, "HNSW search needs %zu bytes of shared memory (ef=%d, k=%d, dim=%d): too large", smem, ef0, k, s->d);
        if (const char* eb = getenv("NIDX_B200_HS_BITS")) {   // tests: a smaller visited table (one that still holds a reseeded list)
            hash_bits = std::min(hash_bits, std::max(ilog2(next_pow2(4 * ef0)), atoi(eb)));
            smem = hs_smem_bytes(s->ld, list_cap, hash_bits);
        }
        VecDev Vh = V;   // with the screening copy attached
        int r = attach_half_copy(s, &Vh);
        // deferral needs the fp16 copy's walk and pops that are never rejected (hs_can_defer)
        const bool defer = Vh.hvecs != nullptr && !bits && p->with_duplicates && !s->cfg.multi_vector;
        hs_kernel_t kern = pick_search_kernel(s->ld, defer);
        int grid = 0;
        if (!r) r = walk_grid(kern, HS_THREADS, smem, &grid);
        if (r) return r;
        // The shared-memory capacities can overflow (a filter that rejects most pops makes closest_up_nodes score thousands of
        // nodes, where the reference's BitSet and heap are unbounded).  The walk flags the queries that lost something to them, and
        // a second launch walks those again with lists of n + ef0 entries and a visited table that holds every node, which cannot
        // overflow.  The second launch is enqueued whatever happened -- no host synchronisation -- and its CTAs exit at once when no
        // query was flagged.  Its scratch: one slice per CTA, as many CTAs as 1 GiB holds (at least one, at most one per SM).
        const size_t cap = (size_t)s->n + ef0;
        const int all_bits = rq_table_bits(s->n);
        const size_t slice = cap * 16 + ((size_t)4 << all_bits);
        const int rgrid = (int)std::max<size_t>(1, std::min<size_t>(((size_t)1 << 30) / slice, (size_t)std::min(nq, s->sm_count)));
        const size_t o_list = ((size_t)nq * 4 + 255) & ~(size_t)255, o_vis = o_list + (size_t)rgrid * cap * 16;
        ENSURE(w.rerun, o_vis + ((size_t)rgrid << all_bits) * 4);
        SearchArgs a = walk_args(ef0, list_cap, cu_cap, hash_bits);
        a.flagged = w.rerun.as<uint32_t>();
        a.n_flagged = w.sched.as<unsigned int>() + 2;   // zeroed with the counters (nidx_vec_walk_reruns reads it)
        CU(cudaEventRecord(s->ev_k0, stream));
        kern<<<grid, HS_THREADS, smem, stream>>>(Vh, s->gdev(), a);
        LAUNCHED();
        SearchArgs b = a;
        b.work_counter = w.sched.as<unsigned int>() + 3;
        b.list_cap = b.cu_cap = (int)cap;
        b.hash_bits = 0;
        b.glist = reinterpret_cast<uint64_t*>(w.rerun.p + o_list);
        b.gvisited = reinterpret_cast<uint32_t*>(w.rerun.p + o_vis); b.gv_bits = all_bits;
        pick_rerun_kernel(s->ld)<<<rgrid, HS_THREADS, hs_smem_bytes(s->ld, 0, 0), stream>>>(Vh, s->gdev(), b);
        LAUNCHED();
        CU(cudaEventRecord(s->ev_k1, stream));
        CU(cudaGetLastError());
        return 0;
    }
};

// NIDX_METHOD_AUTO: the walk or the exhaustive scan by the reference's cost model.  A segment that carries codes is searched with a
// RaBitQ query on either path (segment.rs:506-513: `rabitq` = has_quantized): the quantised walk (hnsw/search.rs:332-366) or the
// quantised scan (segment.rs:581-608).
static int choose_method(const nidx_vec_segment* s, uint64_t matching, int k, int ef) {
    if (!s->has_graph) return NIDX_METHOD_BRUTE;
    bool walk_ok = s->d_quant && s->cfg.similarity == NIDX_SIM_DOT;
    bool scan_ok = walk_ok && !s->d_par_first && k <= 1024;
    if (!use_hnsw_cost(s->n_par, matching, (size_t)k, (size_t)s->cfg.m, walk_ok)) return scan_ok ? NIDX_METHOD_BRUTE_RABITQ : NIDX_METHOD_BRUTE;
    // A walk keeps its list and visited set in shared memory: a very large top_k (the reference has no limit on it) does not fit one
    // CTA.  AUTO then takes the exhaustive scan -- exact results -- instead of failing the request.
    int last_k, list_cap, cu_cap, hash_bits;
    size_t bytes;
    bool fits = walk_ok ? rq_walk_smem(s, k, &last_k, &cu_cap, &list_cap, &hash_bits, &bytes)
                        : hnsw_search_smem(s, std::max(k, ef > 0 ? ef : s->cfg.ef_search), k, &list_cap, &cu_cap, &hash_bits, &bytes);
    if (!fits && k <= 1024) return NIDX_METHOD_BRUTE;
    return walk_ok ? NIDX_METHOD_HNSW_RABITQ : NIDX_METHOD_HNSW;
}

// The body of nidx_vec_search.  qhost: the queries (and filter bits) are host pointers; ohost: the outputs are host pointers
// (copied back and the stream synchronised before returning).  The sharded entry point (shard.cuh) passes host queries with
// device outputs: the partial results go straight into the exchange buffer.
static int vec_search_impl(nidx_vec_segment* s, const float* queries, int32_t nq, int32_t ldq, bool qhost, bool ohost, const nidx_vec_search_params* p,
                           uint32_t* out_ids, float* out_scores, int32_t* out_counts, cudaStream_t stream, const nidx_filter_node* formula = nullptr,
                           int32_t n_formula = 0) {
    if (!s || !p || (!queries && nq > 0) || !out_ids || !out_scores) return fail(NIDX_EINVAL, "null argument");
    if (nq <= 0) return 0;
    if (ldq < s->d) return fail(NIDX_EINVAL, "query dimension %d != index dimension %d (VectorErr::InconsistentDimensions)", ldq, s->d);
    const int k = p->k;
    if (k <= 0) return fail(NIDX_EINVAL, "k must be positive");
    CU(cudaSetDevice(s->cfg.device));
    WsGuard g(s->pool, stream);
    Workspace& w = *g.w;
    VecCall c{s, w, stream, p, s->vdev(), nq, k};
    Stage st(stream, qhost, ohost);
    const float* d_q;
    const uint64_t* d_filter;
    st.in(queries, (size_t)nq * ldq, &d_q);
    st.in(formula ? nullptr : p->filter_bits, ((size_t)s->n_par + 63) / 64, &d_filter);
    st.out(out_ids, (size_t)nq * k, &c.ids);
    st.out(out_scores, (size_t)nq * k, &c.scores);
    st.out(out_counts, (size_t)nq, &c.counts);
    int r = st.place(w.stage);
    if (r) return r;
    // this call's counters, zero whatever the method: the getters report them until the next search
    ENSURE(w.sched, 128);
    CU(cudaMemsetAsync(w.sched.p, 0, 128, stream));
    c.counters = reinterpret_cast<unsigned long long*>(w.sched.as<unsigned char>() + 64);
    s->last_counters.store(c.counters);

    // queries -> [nq][ld] zero padded on device, norms
    r = upload_queries(s, w, d_q, nq, ldq, qhost, stream, &c.dq);
    if (r) return r;
    ENSURE(w.qnorms, (size_t)nq * 4);
    c.qnorms = w.qnorms.as<float>();
    if (s->cfg.similarity != NIDX_SIM_DOT) {
        row_norms_kernel<<<(nq + 7) / 8, 256, 0, stream>>>(c.dq, s->ld, (uint64_t)nq, c.qnorms);
        LAUNCHED();
    }

    // filter ∧ alive (segment.rs:516-534)
    c.bits = s->d_alive;
    uint64_t matching = s->d_alive ? s->alive_count : s->n_par;
    if (formula) {   // the formula is evaluated on the device (inverted_index/paragraph.rs:124-186): no host bitset, no copy
        ENSURE(w.filter, ((size_t)s->n_par + 63) / 64 * 8);
        unsigned long long h = 0;   // segment.rs:531: the reference counts the matches of every filtered request (8 bytes back, one sync)
        r = filter_formula(s, w, formula, n_formula, stream, w.filter.as<uint64_t>(), &h);
        if (r) return r;
        c.bits = w.filter.as<uint64_t>();
        matching = h;
    } else if (d_filter) {
        matching = p->filter_matching;
        unsigned long long h = 0;
        r = filter_and_alive(s, w, d_filter, matching ? nullptr : &h, stream, &c.bits);
        if (r) return r;
        if (matching == 0) {
            CU(cudaStreamSynchronize(stream));
            matching = h;
        }
    }

    const int method = p->method == NIDX_METHOD_AUTO ? choose_method(s, matching, k, p->ef) : p->method;
    const bool walk = method == NIDX_METHOD_HNSW || method == NIDX_METHOD_HNSW_RABITQ;
    if (matching == 0) r = c.write_empty();   // segment.rs:532-534: nothing can match (everything deleted / filtered out), whatever the method
    else if (walk && !s->has_graph) return fail(NIDX_ESTATE, "HNSW search requested but the segment has no graph");
    else if (s->n == 0) r = c.write_empty();
    else if (method == NIDX_METHOD_BRUTE_RABITQ) r = c.rabitq_scan();
    else if (method == NIDX_METHOD_BRUTE && use_tc_filter(s, nq, k)) r = c.tc_filter_scan();
    else if (method == NIDX_METHOD_BRUTE) r = c.exact_scan();
    else if (method == NIDX_METHOD_HNSW_RABITQ) r = c.quantised_walk();
    else r = c.dense_walk();
    if (r) return r;
    return st.finish();
}

extern "C" {

int nidx_vec_search(nidx_vec_segment* s, const float* queries, int32_t nq, int32_t ldq, int mem, const nidx_vec_search_params* p, uint32_t* out_ids,
                    float* out_scores, int32_t* out_counts, void* stream_) {
    bool host = mem == NIDX_MEM_HOST;
    return vec_search_impl(s, queries, nq, ldq, host, host, p, out_ids, out_scores, out_counts, reinterpret_cast<cudaStream_t>(stream_));
}

int nidx_vec_search_formula(nidx_vec_segment* s, const float* queries, int32_t nq, int32_t ldq, int mem, const nidx_vec_search_params* p,
                            const nidx_filter_node* nodes, int32_t n_nodes, uint32_t* out_ids, float* out_scores, int32_t* out_counts, void* stream_) {
    bool host = mem == NIDX_MEM_HOST;
    if (p && p->filter_bits) return fail(NIDX_EINVAL, "give either filter_bits or a formula");
    return vec_search_impl(s, queries, nq, ldq, host, host, p, out_ids, out_scores, out_counts, reinterpret_cast<cudaStream_t>(stream_), nodes, n_nodes);
}

int nidx_vec_set_inverted_index(nidx_vec_segment* s, int32_t which, uint32_t n_keys, const uint8_t* key_bytes, const uint64_t* key_off, const uint64_t* post_off,
                                const uint32_t* postings) {
    if (!s || (which != NIDX_INV_LABELS && which != NIDX_INV_FIELDS)) return fail(NIDX_EINVAL, "bad argument");
    if (n_keys && (!key_off || !post_off || (!key_bytes && key_off[n_keys]) || (!postings && post_off[n_keys]))) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(s->cfg.device));
    nidx_vec_segment::InvIndex ix;
    if (!n_keys) { ix.key_off.assign(1, 0); ix.post_off.assign(1, 0); s->inv[which] = std::move(ix); return 0; }
    for (uint32_t i = 0; i + 1 < n_keys; ++i)
        if (cmp_key(key_bytes + key_off[i], key_off[i + 1] - key_off[i], key_bytes + key_off[i + 1], key_off[i + 2] - key_off[i + 1]) >= 0)
            return fail(NIDX_EINVAL, "inverted index keys must be strictly ascending (key %u)", i + 1);
    uint64_t np = post_off[n_keys];
    for (uint64_t i = 0; i < np; ++i) if (postings[i] >= s->n_par) return fail(NIDX_EINVAL, "posting %llu: paragraph %u out of range", (unsigned long long)i, postings[i]);
    ix.key_bytes.assign(key_bytes, key_bytes + key_off[n_keys]);
    ix.key_off.assign(key_off, key_off + n_keys + 1);
    ix.post_off.assign(post_off, post_off + n_keys + 1);
    ALLOC(ix.d_post, std::max<uint64_t>(np, 1) * 4);
    if (np) CU(cudaMemcpy(ix.d_post, postings, np * 4, cudaMemcpyHostToDevice));
    ALLOC(ix.d_post_off, ((size_t)n_keys + 1) * 8);
    CU(cudaMemcpy(ix.d_post_off, post_off, ((size_t)n_keys + 1) * 8, cudaMemcpyHostToDevice));
    ix.n_keys = n_keys;
    s->inv[which] = std::move(ix);   // only now: a rejected or failed call leaves the previous index in place
    return 0;
}

int nidx_vec_filter(nidx_vec_segment* s, const nidx_filter_node* nodes, int32_t n_nodes, uint64_t* out_bits, int mem, uint64_t* out_matching, void* stream_) {
    if (!s) return fail(NIDX_EINVAL, "null segment");
    CU(cudaSetDevice(s->cfg.device));
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    WsGuard g(s->pool, stream);
    Workspace& w = *g.w;
    const bool host = mem == NIDX_MEM_HOST;
    Stage st(stream, host, host);
    uint64_t* d_bits;
    st.out(out_bits, ((size_t)s->n_par + 63) / 64, &d_bits);
    int r = st.place(w.stage);
    unsigned long long h = 0;
    if (!r) r = filter_formula(s, w, nodes, n_nodes, stream, d_bits, &h);   // segment.rs:523-526: intersect with the alive set
    if (!r) r = st.finish(true);
    if (r) return r;
    if (out_matching) *out_matching = h;
    return 0;
}

// The text merge of n_parts top-k lists: (score desc, part asc, position asc)
static int launch_parts_merge(const uint32_t* ids, const float* scores, int n_parts, size_t part_stride, int nq, int k, uint32_t* out_ids, float* out_scores,
                              int* out_part, cudaStream_t stream) {
    if (k > 1024 || (long long)n_parts * k >= (1ll << 31)) return fail(NIDX_EINVAL, "k above 1024 not supported");
    int cap = topk_cap(k, 256);
    if ((size_t)cap * 8 > 48 * 1024) CU(cudaFuncSetAttribute(parts_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap * 8));
    parts_merge_kernel<<<nq, 256, (size_t)cap * 8, stream>>>(ids, scores, n_parts, part_stride, nq, k, cap, out_ids, out_scores, out_part);
    LAUNCHED();
    return 0;
}

int nidx_merge_topk(int32_t device, const uint32_t* ids, const float* scores, int32_t n_parts, int64_t part_stride, int32_t nq, int32_t k,
                    uint32_t* out_ids, float* out_scores, int32_t* out_part, void* stream_) {
    int r = check_device(device);
    if (r) return r;
    if (!ids || !scores || !out_ids || !out_scores || n_parts <= 0 || nq <= 0 || k <= 0) return fail(NIDX_EINVAL, "bad argument");
    r = launch_parts_merge(ids, scores, n_parts, part_stride > 0 ? (size_t)part_stride : (size_t)nq * k, nq, k, out_ids, out_scores, out_part,
                           reinterpret_cast<cudaStream_t>(stream_));
    if (r) return r;
    CU(cudaGetLastError());
    return 0;
}

// kmerge_parts_kernel: one thread per query, n_parts heap entries (u32) per thread in shared memory
static int launch_kmerge(const uint32_t* ids, const float* scores, int n_parts, size_t part_stride, int nq, int k, uint32_t* out_ids, float* out_scores,
                         int* out_part, int* out_counts, cudaStream_t stream) {
    if ((long long)n_parts * k >= (1ll << 31)) return fail(NIDX_EINVAL, "n_parts * k must stay below 2^31");
    size_t per = (size_t)n_parts * 4;
    if (per > 96 * 1024) return fail(NIDX_EINVAL, "%d parts are too many for the vector merge", n_parts);
    int threads = (int)std::max<size_t>(1, std::min<size_t>(128, (size_t)(48 * 1024) / per));
    threads = std::min(threads, nq);
    size_t smem = per * threads;
    if (smem > 48 * 1024) CU(cudaFuncSetAttribute(kmerge_parts_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kmerge_parts_kernel<<<(nq + threads - 1) / threads, threads, smem, stream>>>(ids, scores, n_parts, part_stride, nq, k, out_ids, out_scores, out_part,
                                                                                 out_counts);
    LAUNCHED();
    return 0;
}

int nidx_merge_vector_parts(int32_t device, const uint32_t* ids, const float* scores, int32_t n_parts, int64_t part_stride, int32_t nq, int32_t k,
                            uint32_t* out_ids, float* out_scores, int32_t* out_part, void* stream_) {
    int r = check_device(device);
    if (r) return r;
    if (!ids || !scores || !out_ids || !out_scores || n_parts <= 0 || nq <= 0 || k <= 0) return fail(NIDX_EINVAL, "bad argument");
    r = launch_kmerge(ids, scores, n_parts, part_stride > 0 ? (size_t)part_stride : (size_t)nq * k, nq, k, out_ids, out_scores, out_part, nullptr,
                      reinterpret_cast<cudaStream_t>(stream_));
    if (r) return r;
    CU(cudaGetLastError());
    return 0;
}

// ---- build ------------------------------------------------------------------------------------
// Level RNG: build.rs:40,97-101.  rand 0.10 SmallRng = xoshiro256++ seeded by SplitMix64 [recalled].
static void host_assign_levels(uint64_t n, int M, uint64_t seed, uint8_t* level) {
    uint64_t st[4], state = seed;
    for (int i = 0; i < 4; ++i) {
        state += 0x9e3779b97f4a7c15ull;
        uint64_t z = state;
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        st[i] = z ^ (z >> 31);
    }
    auto rotl = [](uint64_t x, int k) { return (x << k) | (x >> (64 - k)); };
    double level_factor = 1.0 / std::log((double)M);
    for (uint64_t i = 0; i < n; ++i) {
        uint64_t r = rotl(st[0] + st[3], 23) + st[0];
        uint64_t t = st[1] << 17;
        st[2] ^= st[0]; st[3] ^= st[1]; st[1] ^= st[2]; st[0] ^= st[3];
        st[2] ^= t;
        st[3] = rotl(st[3], 45);
        double u = (double)(r >> 12) * (1.0 / 4503599627370496.0);
        double lv = std::round(-std::log(u) * level_factor);
        if (!(lv < (double)(HS_MAX_LAYERS - 1))) lv = (double)(HS_MAX_LAYERS - 1);
        level[i] = (uint8_t)lv;
    }
}

}  // extern "C"

// Batch-synchronous insertion of order[0 .. n) into the segment's graph (which may already hold other nodes):
// the loop of build.rs:123-166 as search / select / sort / reverse-link kernels per batch (hnsw_build.cuh).
// entry_after_first (node, layer), if given, becomes the entry point once the first batch has been inserted.
static int insert_batches(nidx_vec_segment* s, const std::vector<uint8_t>& level, const std::vector<uint32_t>& order, const std::vector<uint32_t>& ends,
                          cudaStream_t stream, const uint32_t* entry_after_first) {
    uint64_t n = order.size();
    // work items (node position, layer), insertion order, layer ascending
    std::vector<uint64_t> wstart(n + 1);
    uint64_t W = 0;
    for (uint64_t i = 0; i < n; ++i) { wstart[i] = W; W += (uint64_t)level[order[i]] + 1; }
    wstart[n] = W;
    std::vector<uint32_t> w_pos(W);
    std::vector<unsigned char> w_layer(W);
    for (uint64_t i = 0; i < n; ++i)
        for (int l = 0; l <= level[order[i]]; ++l) { w_pos[wstart[i] + l] = (uint32_t)i; w_layer[wstart[i] + l] = (unsigned char)l; }
    uint64_t max_b = 0, max_w = 0;
    for (size_t b = 0, begin = 0; b < ends.size(); begin = ends[b], ++b) {
        max_b = std::max<uint64_t>(max_b, ends[b] - begin);
        max_w = std::max<uint64_t>(max_w, wstart[ends[b]] - wstart[begin]);
    }
    int efC = s->cfg.ef_construction, M = s->cfg.m;
    DevArray<uint32_t> d_order, d_wpos, d_rev_x, d_idx, d_idx_sorted, d_heads;
    DevArray<unsigned int> d_head_ctr;  // [0] number of heads, [1] work counter
    DevArray<unsigned char> d_wlayer;
    DevArray<uint64_t> d_found, d_rev_key, d_key_sorted;
    DevArray<int> d_found_count;
    DevArray<float> d_rev_sim;
    DevBuf d_cub;
    size_t cub_bytes = 0;
    size_t max_rev = (size_t)max_w * M;
    ALLOC(d_order, n * 4);
    ALLOC(d_wpos, W * 4);
    ALLOC(d_wlayer, W);
    ALLOC(d_found, (size_t)max_b * HS_MAX_LAYERS * efC * 8);
    ALLOC(d_found_count, (size_t)max_b * HS_MAX_LAYERS * 4);
    ALLOC(d_rev_key, max_rev * 8);
    ALLOC(d_key_sorted, max_rev * 8);
    ALLOC(d_rev_x, max_rev * 4);
    ALLOC(d_rev_sim, max_rev * 4);
    ALLOC(d_idx, max_rev * 4);
    ALLOC(d_idx_sorted, max_rev * 4);
    ALLOC(d_heads, max_rev * 4);
    ALLOC(d_head_ctr, 64);
    CU(cudaMemcpyAsync(d_order, order.data(), n * 4, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_wpos, w_pos.data(), W * 4, cudaMemcpyHostToDevice, stream));
    CU(cudaMemcpyAsync(d_wlayer, w_layer.data(), W, cudaMemcpyHostToDevice, stream));
    {
        std::vector<uint32_t> iota(max_rev);
        for (size_t i = 0; i < max_rev; ++i) iota[i] = (uint32_t)i;
        CU(cudaMemcpyAsync(d_idx, iota.data(), max_rev * 4, cudaMemcpyHostToDevice, stream));
        CU(cudaStreamSynchronize(stream));
    }
    CU(cub::DeviceRadixSort::SortPairs(nullptr, cub_bytes, d_rev_key.p, d_key_sorted.p, d_idx.p, d_idx_sorted.p, (int)max_rev, 0, 40, stream));
    ALLOC(d_cub, cub_bytes);

    // shared-memory plans

    int list_cap = efC, hash_bits;
    int slots = next_pow2(std::max(2048, (efC * s->s0 * 3) / 2));
    slots = std::max(slots, next_pow2(4 * list_cap));
    hash_bits = ilog2(slots);
    size_t smem_search = hs_smem_bytes(s->ld, list_cap, hash_bits);
    if (smem_search > 200 * 1024) return fail(NIDX_EINVAL, "HNSW build search needs %zu bytes of shared memory", smem_search);
    hs_kernel_t kern = pick_search_kernel(s->ld);
    CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_search));
    int occ = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kern, HS_THREADS, smem_search));
    size_t row_bytes = (size_t)s->ld * 4;
    size_t budget = 96 * 1024;
    int cache_sel = (int)std::min<size_t>(M, budget / row_bytes);
    int prune_max = std::max(s->cfg.m0, M) * 95 / 100;
    int cache_rev = (int)std::min<size_t>(prune_max, budget / row_bytes);
    size_t smem_sel = hb_smem_bytes(s->ld, cache_sel), smem_rev = hb_smem_bytes(s->ld, cache_rev);
    CU(cudaFuncSetAttribute(select_link_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_sel));
    CU(cudaFuncSetAttribute(reverse_link_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_rev));
    int occ_rev = 0;
    CU(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ_rev, reverse_link_kernel, HB_THREADS, smem_rev));
    int rev_grid = std::max(1, occ_rev) * s->sm_count;
    CU(cudaMemsetAsync(s->d_counters, 0, 8 * sizeof(unsigned long long), stream));
    s->last_counters.store(nullptr);   // the getters report the build's counters until the next search


    VecDev V = s->vdev();
    int hr = attach_half_copy(s, &V);
    if (hr) return hr;
    GraphDev G = s->gdev();
    uint32_t begin = 0;
    for (size_t b = 0; b < ends.size(); ++b) {
        uint32_t end = ends[b];
        int nb = (int)(end - begin);
        int nw = (int)(wstart[end] - wstart[begin]);
        SearchArgs a;
        memset(&a, 0, sizeof(a));
        a.mode = 1; a.nq = nb; a.nodes = d_order + begin; a.efC = efC; a.found = d_found; a.found_count = d_found_count;
        a.hash_bits = hash_bits; a.list_cap = list_cap; a.cu_cap = 0; a.work_counter = s->d_work_counter; a.counters = s->d_counters;
        CU(cudaMemsetAsync(s->d_work_counter, 0, 4, stream));
        int grid = std::min(nb, std::max(1, occ) * s->sm_count);
        kern<<<grid, HS_THREADS, smem_search, stream>>>(V, G, a);
        LAUNCHED();
        BuildArgs ba;
        ba.n_work = nw; ba.w_pos = d_wpos + wstart[begin]; ba.w_layer = d_wlayer + wstart[begin]; ba.order = d_order; ba.batch_begin = begin;
        ba.efC = efC; ba.M = M; ba.found = d_found; ba.found_count = d_found_count; ba.rev_key = d_rev_key; ba.rev_x = d_rev_x; ba.rev_sim = d_rev_sim;
        ba.cache_cap = cache_sel;
        select_link_kernel<<<nw, HB_THREADS, smem_sel, stream>>>(V, G, ba);
        LAUNCHED();
        int n_rev = nw * M;
        size_t tmp = cub_bytes;
        CU(cub::DeviceRadixSort::SortPairs(d_cub.p, tmp, d_rev_key.p, d_key_sorted.p, d_idx.p, d_idx_sorted.p, n_rev, 0, 40, stream));
        LAUNCHED();
        ReverseArgs ra;
        ra.n_rev = n_rev; ra.key_sorted = d_key_sorted; ra.idx_sorted = d_idx_sorted; ra.rev_x = d_rev_x; ra.rev_sim = d_rev_sim; ra.cache_cap = cache_rev;
        ra.heads = d_heads; ra.n_heads = d_head_ctr; ra.work_counter = d_head_ctr + 1;
        CU(cudaMemsetAsync(d_head_ctr, 0, 8, stream));
        collect_heads_kernel<<<(n_rev + 255) / 256, 256, 0, stream>>>(d_key_sorted, n_rev, d_heads, d_head_ctr);
        LAUNCHED();
        reverse_link_kernel<<<std::min(n_rev, rev_grid), HB_THREADS, smem_rev, stream>>>(V, G, ra);
        LAUNCHED();
        begin = end;
        if (b == 0 && entry_after_first) {   // kernel arguments travel by value: later batches start from the new entry point
            s->entry_node = entry_after_first[0];
            s->entry_layer = entry_after_first[1];
            G = s->gdev();
        }
    }
    CU(cudaGetLastError());
    CU(cudaStreamSynchronize(stream));
    return 0;
}

// insert_batches; on failure the segment loses its graph
static int run_insertions(nidx_vec_segment* s, const std::vector<uint8_t>& level, const std::vector<uint32_t>& order, const std::vector<uint32_t>& ends,
                          cudaStream_t stream, const uint32_t* entry_after_first = nullptr) {
    int r = insert_batches(s, level, order, ends, stream, entry_after_first);
    if (r) free_graph(s);
    return r;
}

// Appends the insertion batches from `done` inserted nodes to n (ends counted from `base`): batch b = min(max_batch, max(1, done/16))
static void batch_ends(uint64_t done, uint64_t n, uint64_t base, int max_batch, std::vector<uint32_t>& ends) {
    if (max_batch <= 0) max_batch = 4096;
    while (done < n) {
        done += std::min<uint64_t>({(uint64_t)max_batch, std::max<uint64_t>(1, done / 16), n - done});
        ends.push_back((uint32_t)(done - base));
    }
}

extern "C" {

int nidx_hnsw_levels(uint64_t n, int32_t m, uint64_t seed, uint8_t* out_level) {
    if (!out_level && n) return fail(NIDX_EINVAL, "null argument");
    if (m < 2) return fail(NIDX_EINVAL, "M must be at least 2");
    host_assign_levels(n, m, seed, out_level);
    return 0;
}

int nidx_vec_build_hnsw(nidx_vec_segment* s, uint64_t seed, int32_t max_batch, void* stream_) {
    if (!s) return fail(NIDX_EINVAL, "null segment");
    CU(cudaSetDevice(s->cfg.device));
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    uint64_t n = s->n;
    std::vector<uint8_t> level(n ? n : 1);
    host_assign_levels(n, s->cfg.m, seed, level.data());
    int r = alloc_graph(s, level.data());
    if (r) return r;
    s->has_graph = true;
    if (n == 0) return 0;

    // insertion order: entry point first, then ascending id
    std::vector<uint32_t> order(n);
    order[0] = s->entry_node;
    for (uint64_t i = 0, j = 1; i < n; ++i) if (i != s->entry_node) order[j++] = (uint32_t)i;
    std::vector<uint32_t> ends;
    batch_ends(0, n, 0, max_batch, ends);
    return run_insertions(s, level, order, ends, stream);
}

// merge_indexes' fast path (segment.rs:143-167): the first n_existing vectors of this (merged) segment are the largest
// input segment, which had no deletions, so its graph is reused and only the remaining vectors are inserted.
// HnswBuilder::new seeds a fresh level RNG and initialize_graph(skip_nodes = n_existing, total) draws the new nodes'
// levels (build.rs:36-55); the entry point moves only if a higher layer appears (ram_hnsw.rs:99-107).
int nidx_vec_extend_hnsw(nidx_vec_segment* s, uint64_t n_existing, const uint8_t* level_existing, const uint32_t* adj0, const float* w0,
                         const uint32_t* adjU, const float* wU, uint32_t entry_node, uint32_t entry_layer, uint64_t seed, int32_t max_batch, void* stream_) {
    if (!s || !level_existing || !adj0) return fail(NIDX_EINVAL, "null argument");
    if (!w0 || (adjU && !wU)) return fail(NIDX_EINVAL, "the existing edges' similarities are required (hnsw.edges): the reverse-link prune ranks by them");
    if (n_existing == 0 || n_existing > s->n) return fail(NIDX_EINVAL, "n_existing must be in 1..len");
    if (entry_node >= n_existing || level_existing[entry_node] < entry_layer) return fail(NIDX_EINVAL, "bad entry point");
    CU(cudaSetDevice(s->cfg.device));
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    uint64_t n = s->n;
    std::vector<uint8_t> level(n);
    memcpy(level.data(), level_existing, n_existing);
    for (uint64_t i = 0; i < n_existing; ++i)
        if (level[i] >= HS_MAX_LAYERS) return fail(NIDX_EINVAL, "node %llu has level %d >= %d", (unsigned long long)i, level[i], HS_MAX_LAYERS);
    uint64_t rows_existing = 0;
    for (uint64_t i = 0; i < n_existing; ++i) rows_existing += level[i];
    if (rows_existing && !adjU) return fail(NIDX_EINVAL, "existing nodes have upper layers but adjU is null");
    host_assign_levels(n - n_existing, s->cfg.m, seed, level.data() + n_existing);
    int r = alloc_graph(s, level.data());
    if (r) return r;
    // alloc_graph left the entry point on the lowest id of the global top layer.  If that is a NEW node (the merge raises the
    // top layer) the reference moves the entry point there before the node has a single link (update_entry_point in
    // initialize_graph, build.rs:49-55), so every later search starts on an island and the reused graph becomes unreachable.
    // Deliberate deviation: that node is inserted first, from the old entry point, and the entry point moves afterwards.
    uint32_t raised[2] = {s->entry_node, s->entry_layer};
    bool raises = raised[1] > entry_layer && raised[0] >= n_existing;
    if (raised[1] > entry_layer && !raises) { entry_node = raised[0]; entry_layer = raised[1]; }   // the caller's entry point was below its own top layer
    s->entry_layer = entry_layer;
    s->entry_node = entry_node;
    // the existing nodes' rows: layer 0 rows are a prefix, and so are their upper-pool rows (offsets depend on earlier nodes only)
    CU(cudaMemcpy(s->d_adj0, adj0, (size_t)n_existing * s->s0 * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(s->d_w0, w0, (size_t)n_existing * s->s0 * 4, cudaMemcpyHostToDevice));
    if (rows_existing) {
        // fix_broken_graph (ram_hnsw.rs:52-64,118-123): a link in layer L > 0 to a node that is not in layer L is dropped
        // (graphs written by an old version can hold them); the patched copy is made only if one is found
        std::vector<uint32_t> fixed_adj;
        std::vector<float> fixed_w;
        uint64_t row = 0;
        for (uint64_t i = 0; i < n_existing; ++i)
            for (int layer = 1; layer <= level[i]; ++layer, ++row) {
                const uint32_t* r0 = adjU + row * s->su;
                bool broken = false;
                for (int j = 0; j < s->su && r0[j] != NIL; ++j)
                    if (r0[j] >= n_existing || level[r0[j]] < layer) { broken = true; break; }
                if (!broken) continue;
                if (fixed_adj.empty()) {
                    fixed_adj.assign(adjU, adjU + rows_existing * s->su);
                    if (wU) fixed_w.assign(wU, wU + rows_existing * s->su);
                }
                uint32_t* dst = fixed_adj.data() + row * s->su;
                float* dw = wU ? fixed_w.data() + row * s->su : nullptr;
                int kept = 0;
                for (int j = 0; j < s->su && r0[j] != NIL; ++j)
                    if (r0[j] < n_existing && level[r0[j]] >= layer) {
                        dst[kept] = r0[j];
                        if (dw) dw[kept] = wU[row * s->su + j];
                        ++kept;
                    }
                for (int j = kept; j < s->su; ++j) { dst[j] = NIL; if (dw) dw[j] = 0.0f; }
            }
        const uint32_t* srcA = fixed_adj.empty() ? adjU : fixed_adj.data();
        const float* srcW = fixed_adj.empty() ? wU : fixed_w.data();
        CU(cudaMemcpy(s->d_adjU, srcA, (size_t)rows_existing * s->su * 4, cudaMemcpyHostToDevice));
        if (wU) CU(cudaMemcpy(s->d_wU, srcW, (size_t)rows_existing * s->su * 4, cudaMemcpyHostToDevice));
    }
    s->has_graph = true;
    if (n == n_existing) return 0;
    std::vector<uint32_t> order;
    order.reserve(n - n_existing);
    if (raises) order.push_back(raised[0]);
    for (uint64_t i = n_existing; i < n; ++i)
        if (!raises || i != raised[0]) order.push_back((uint32_t)i);
    std::vector<uint32_t> ends;
    if (raises) ends.push_back(1);
    batch_ends(n_existing + (raises ? 1 : 0), n, n_existing, max_batch, ends);
    return run_insertions(s, level, order, ends, stream, raises ? raised : nullptr);
}

// ---- segment files ----------------------------------------------------------------------------
int nidx_vec_open(const nidx_vec_config* cfg, const char* dir, nidx_vec_segment** out) {
    if (!dir) return fail(NIDX_EINVAL, "null dir");
    if (!out) return fail(NIDX_EINVAL, "null argument");
    std::unique_ptr<nidx_vec_segment> s;
    int r = new_segment(cfg, s);
    if (r) return r;
    std::string err;
    std::vector<unsigned char> raw;
    if (!segio::read_file(std::string(dir) + "/vectors.bin", raw, err)) return fail(NIDX_EIO, "%s", err.c_str());
    size_t rec = (size_t)s->d * 4 + 4;  // vector_store.rs:33-68: [dim x f32 LE][paragraph_addr u32]
    if (raw.size() % rec) return fail(NIDX_EIO, "vectors.bin size %zu is not a multiple of the record length %zu", raw.size(), rec);
    uint64_t n = raw.size() / rec;
    s->n = n;
    std::vector<uint32_t> par(n);
    for (uint64_t i = 0; i < n; ++i) memcpy(&par[i], raw.data() + i * rec + (size_t)s->d * 4, 4);
    r = upload_rows(s.get(), raw.data(), rec, true, false);
    if (!r) r = finish_create(s.get(), n ? par.data() : nullptr);
    if (r) return r;
    // hnsw.graph (+ hnsw.edges) if present
    std::vector<unsigned char> graph, edges;
    if (segio::read_file(std::string(dir) + "/hnsw.graph", graph, err) && !graph.empty()) {
        segio::read_file(std::string(dir) + "/hnsw.edges", edges, err);
        segio::FlatGraph fg;
        if (!segio::parse_graph_v2(graph, edges, n, stride0_for(s->cfg.m0), strideU_for(s->cfg.m), HS_MAX_LAYERS, fg, err))
            return fail(NIDX_EIO, "hnsw.graph: %s", err.c_str());
        r = nidx_vec_set_graph(s.get(), fg.level.data(), fg.adj0.data(), fg.w0.empty() ? nullptr : fg.w0.data(), fg.adjU.data(), fg.wU.empty() ? nullptr : fg.wU.data());
        if (r) return r;
        s->entry_node = fg.entry_node;   // the file's entry point (ram_hnsw.rs: hash-order dependent in the reference)
        s->entry_layer = fg.entry_layer;
    }
    // vectors.quant (data_store/v2/quant_vector_store.rs:29-62): the RaBitQ codes, one record of dim / 8 + 8 bytes per vector, loaded as they
    // are (re-laid out to the 16-byte stride in HBM) instead of re-encoding
    std::vector<unsigned char> quant;
    if (s->cfg.similarity == NIDX_SIM_DOT && s->d % 64 == 0 && s->d / 32 <= RQ_MAX_WORDS32 && segio::read_file(std::string(dir) + "/vectors.quant", quant, err) && !quant.empty()) {
        size_t rec_q = (size_t)s->d / 8 + 8;
        if (quant.size() != rec_q * n) return fail(NIDX_EIO, "vectors.quant holds %zu bytes, expected %zu records of %zu", quant.size(), (size_t)n, rec_q);
        s->quant_stride = rabitq_stride(s->d);
        ALLOC(s->d_quant, std::max<size_t>((size_t)n * s->quant_stride, 16));
        CU(cudaMemset(s->d_quant, 0, std::max<size_t>((size_t)n * s->quant_stride, 16)));
        CU(cudaMemcpy2D(s->d_quant, (size_t)s->quant_stride, quant.data(), rec_q, rec_q, (size_t)n, cudaMemcpyHostToDevice));
    }
    *out = s.release();
    return 0;
}

int nidx_vec_save(nidx_vec_segment* s, const char* dir) {
    if (!s || !dir) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(s->cfg.device));
    CU(cudaDeviceSynchronize());
    uint64_t n = s->n;
    std::vector<float> vecs((size_t)n * s->ld);
    CU(cudaMemcpy(vecs.data(), s->d_vecs, vecs.size() * 4, cudaMemcpyDeviceToHost));
    std::vector<uint32_t> par(n);
    if (s->d_par_of) CU(cudaMemcpy(par.data(), s->d_par_of, n * 4, cudaMemcpyDeviceToHost));
    else for (uint64_t i = 0; i < n; ++i) par[i] = (uint32_t)i;
    std::string err;
    if (!segio::write_vectors_bin(std::string(dir) + "/vectors.bin", vecs.data(), n, s->d, s->ld, par.data(), err)) return fail(NIDX_EIO, "%s", err.c_str());
    if (s->has_graph) {
        segio::FlatGraph fg;
        fg.n = n; fg.s0 = s->s0; fg.su = s->su; fg.entry_node = s->entry_node; fg.entry_layer = s->entry_layer;
        fg.level = s->h_level;
        fg.upper_rows = s->upper_rows;
        fg.adj0.resize((size_t)n * s->s0); fg.w0.resize((size_t)n * s->s0);
        fg.adjU.resize((size_t)s->upper_rows * s->su); fg.wU.resize((size_t)s->upper_rows * s->su);
        int r = nidx_vec_get_graph(s, nullptr, fg.adj0.data(), fg.w0.data(), fg.adjU.data(), fg.wU.data());
        if (r) return r;
        if (!segio::write_graph_v2(std::string(dir) + "/hnsw.graph", std::string(dir) + "/hnsw.edges", fg, err)) return fail(NIDX_EIO, "%s", err.c_str());
    }
    if (s->d_quant) {   // vectors.quant: QuantVectorStoreWriter (quant_vector_store.rs), records back to back
        size_t rec_q = (size_t)s->d / 8 + 8;
        std::vector<unsigned char> quant(rec_q * n);
        if (n) CU(cudaMemcpy2D(quant.data(), rec_q, s->d_quant, (size_t)s->quant_stride, rec_q, (size_t)n, cudaMemcpyDeviceToHost));
        FILE* f = fopen((std::string(dir) + "/vectors.quant").c_str(), "wb");
        if (!f) return fail(NIDX_EIO, "cannot write %s/vectors.quant", dir);
        size_t wr = quant.empty() ? 0 : fwrite(quant.data(), 1, quant.size(), f);
        fclose(f);
        if (wr != quant.size()) return fail(NIDX_EIO, "short write to %s/vectors.quant", dir);
    }
    return 0;
}

// ---- text ---------------------------------------------------------------------------------------
// A dictionary of path keys on the host (in facet order) and every document's ords of it as CSR in HBM: the facets
// (nidx_txt_set_facets) and the access groups (nidx_txt_set_doc_groups).
struct OrdColumn {
    std::vector<std::string> keys;
    DevArray<uint32_t> d_off;         // [n_docs + 1]
    DevArray<uint32_t> d_ord;         // [n_ords]
    uint64_t n_ords = 0;
};

// What a text segment and its views share: everything but the alive bits.
struct TxtIndex {
    int device = 0, sm_count = 0;
    uint32_t n_docs = 0, n_terms = 0;
    uint64_t n_post = 0;
    DevArray<uint64_t> d_term_off;
    DevArray<uint2> d_post;           // (doc, tf << 8 | fieldnorm id)
    DevArray<uint32_t> d_skip_row;    // [n_terms]
    DevArray<uint32_t> d_skip;        // [rows][n_fine + 1]
    uint32_t n_fine = 0;
    DevArray<float> d_weight;         // [n_terms]
    DevArray<float> d_norm_cache;     // [256]
    DevArray<uint64_t> d_doc_keys;    // [n_docs] caller keys of the documents (paragraph ids) for rank fusion (nidx_txt_set_doc_keys)
    std::vector<uint64_t> own_df;
    uint64_t own_tokens = 0;
    cudaEvent_t ev_k0 = nullptr, ev_k1 = nullptr;  // around bm25_kernel of the last search (bench roofline)
    OrdColumn facets;                 // nidx_txt_set_facets
    OrdColumn groups;                 // nidx_txt_set_doc_groups: a document without ords is public
    // dates (nidx_txt_set_dates), per field (NIDX_ORDER_CREATED, NIDX_ORDER_MODIFIED): the seconds and every document's dense rank
    DevArray<int64_t> d_secs[2];      // [n_docs]
    DevArray<uint32_t> d_rank[2];     // [n_docs rounded up to 8], 0 = no date
    uint32_t n_ranks[2] = {0, 0};
    // positions (nidx_txt_set_positions): every posting's token positions, in posting order, and where each posting's start
    DevArray<uint64_t> d_pos_off;     // [n_post + 1]
    DevArray<uint32_t> d_pos;
    std::vector<float> idf;           // [n_terms] of the statistics set last: a phrase's weight sums its terms'
    // prefilter columns (nidx_txt_set_doc_columns): every document's resource and field ord
    DevArray<uint32_t> d_res_ord, d_field_ord;
    DevArray<uint64_t> d_repeated;    // nidx_txt_set_repeated: paragraphs repeated in their field (NULL: none)
    cudaEvent_t ev_sg[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};   // the last fuzzy suggest pass (created on its first call)
    WorkspacePool pool;

    ~TxtIndex() {
        if (ev_k0) cudaEventDestroy(ev_k0);
        if (ev_k1) cudaEventDestroy(ev_k1);
        for (cudaEvent_t e : ev_sg) if (e) cudaEventDestroy(e);
    }
};

// A segment owns its index; a view (nidx_txt_view) shares its parent's and owns only its alive bits.
struct nidx_txt_segment {
    std::unique_ptr<TxtIndex> own;    // NULL for a view
    TxtIndex* ix = nullptr;
    DevArray<uint64_t> d_alive;
};

// tantivy fieldnorm code -> token count (Lucene SmallFloat.byte4ToInt) [recalled]
static uint32_t fieldnorm_id_to_value(uint32_t id) {
    if (id < 24) return id;
    uint32_t j = id - 24, bits = j & 7, shift = j >> 3;
    return 24 + (shift == 0 ? bits : ((bits | 8u) << (shift - 1)));
}

static int txt_upload_stats(nidx_txt_segment* t, uint64_t total_docs, uint64_t total_tokens, const uint64_t* df) {
    const float K1 = 1.2f, B = 0.75f;
    float avg = (float)total_tokens / (float)total_docs;
    float cache[256];
    for (int i = 0; i < 256; ++i) cache[i] = K1 * (1.0f - B + B * (float)fieldnorm_id_to_value(i) / avg);
    std::vector<float> weight(t->ix->n_terms), idf(t->ix->n_terms);
    for (uint32_t i = 0; i < t->ix->n_terms; ++i) {
        float x = ((float)(total_docs - df[i]) + 0.5f) / ((float)df[i] + 0.5f);
        idf[i] = logf(1.0f + x);
        weight[i] = idf[i] * (1.0f + K1);
    }
    CU(cudaMemcpy(t->ix->d_norm_cache, cache, sizeof(cache), cudaMemcpyHostToDevice));
    if (t->ix->n_terms) CU(cudaMemcpy(t->ix->d_weight, weight.data(), (size_t)t->ix->n_terms * 4, cudaMemcpyHostToDevice));
    t->ix->idf = std::move(idf);
    return 0;
}

int nidx_txt_create(int32_t device, uint32_t n_docs, uint32_t n_terms, const uint64_t* term_off, const uint32_t* post_doc, const uint32_t* post_tf,
                    const uint8_t* fieldnorm_id, nidx_txt_segment** out) {
    if (!term_off || !fieldnorm_id || !out) return fail(NIDX_EINVAL, "null argument");
    int r = check_device(device);
    if (r) return r;
    if (n_docs >= (1u << 31)) return fail(NIDX_EINVAL, "at most 2^31-1 documents per segment");
    std::unique_ptr<nidx_txt_segment> t(new nidx_txt_segment());   // freed with everything it holds unless the call succeeds
    t->own.reset(new TxtIndex());
    t->ix = t->own.get();
    t->ix->device = device; t->ix->n_docs = n_docs; t->ix->n_terms = n_terms; t->ix->n_post = term_off[n_terms];
    cudaDeviceProp prop;
    cudaGetDeviceProperties(&prop, device);
    t->ix->sm_count = prop.multiProcessorCount;
    t->ix->n_fine = (n_docs + BM_FINE - 1) / BM_FINE;
    ALLOC(t->ix->d_term_off, ((size_t)n_terms + 1) * 8);
    ALLOC(t->ix->d_post, std::max<uint64_t>(t->ix->n_post, 1) * 8);
    ALLOC(t->ix->d_weight, std::max<uint32_t>(n_terms, 1) * 4);
    ALLOC(t->ix->d_norm_cache, 1024);
    ALLOC(t->ix->d_skip_row, std::max<uint32_t>(n_terms, 1) * 4);
    CU(cudaEventCreate(&t->ix->ev_k0));
    CU(cudaEventCreate(&t->ix->ev_k1));
    CU(cudaMemcpy(t->ix->d_term_off, term_off, ((size_t)n_terms + 1) * 8, cudaMemcpyHostToDevice));
    if (t->ix->n_post) {
        // staged only to be packed into the 8-byte posting records
        DevArray<uint32_t> d_doc, d_tf;
        DevArray<unsigned char> d_fn;
        ALLOC(d_doc, t->ix->n_post * 4);
        ALLOC(d_fn, std::max<uint32_t>(n_docs, 1));
        CU(cudaMemcpy(d_doc, post_doc, t->ix->n_post * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(d_fn, fieldnorm_id, n_docs, cudaMemcpyHostToDevice));
        if (post_tf) {
            ALLOC(d_tf, t->ix->n_post * 4);
            CU(cudaMemcpy(d_tf, post_tf, t->ix->n_post * 4, cudaMemcpyHostToDevice));
        }
        bm25_pack_kernel<<<t->ix->sm_count * 8, 256>>>(d_doc, d_tf, d_fn, t->ix->n_post, t->ix->d_post);
        LAUNCHED();
        CU(cudaGetLastError());
        CU(cudaDeviceSynchronize());
    }
    // skip rows for the terms with enough postings
    std::vector<uint32_t> skip_row(n_terms, NIDX_NIL), row_term;
    for (uint32_t i = 0; i < n_terms; ++i)
        if (term_off[i + 1] - term_off[i] >= (uint64_t)BM_SKIP_DF) { skip_row[i] = (uint32_t)row_term.size(); row_term.push_back(i); }
    if (n_terms) CU(cudaMemcpy(t->ix->d_skip_row, skip_row.data(), (size_t)n_terms * 4, cudaMemcpyHostToDevice));
    size_t skip_words = std::max<size_t>(row_term.size(), 1) * ((size_t)t->ix->n_fine + 1);
    ALLOC(t->ix->d_skip, skip_words * 4);
    if (!row_term.empty()) {
        DevArray<uint32_t> d_row_term;
        ALLOC(d_row_term, row_term.size() * 4);
        CU(cudaMemcpy(d_row_term, row_term.data(), row_term.size() * 4, cudaMemcpyHostToDevice));
        bm25_build_skip_kernel<<<t->ix->sm_count * 8, 256>>>(t->ix->d_term_off, t->ix->d_post, d_row_term, (uint32_t)row_term.size(), t->ix->n_fine, t->ix->d_skip);
        LAUNCHED();
        CU(cudaGetLastError());
        CU(cudaDeviceSynchronize());
    }
    t->ix->own_df.resize(n_terms);
    for (uint32_t i = 0; i < n_terms; ++i) t->ix->own_df[i] = term_off[i + 1] - term_off[i];
    // a segment alone only knows the quantised lengths; the exact token total comes with set_stats
    uint64_t tokens = 0;
    for (uint32_t i = 0; i < n_docs; ++i) tokens += fieldnorm_id_to_value(fieldnorm_id[i]);
    t->ix->own_tokens = tokens;
    r = txt_upload_stats(t.get(), std::max<uint32_t>(n_docs, 1), std::max<uint64_t>(tokens, 1), t->ix->own_df.data());
    if (r) return r;
    *out = t.release();
    return 0;
}

// The setters change what a segment's views share: a view has none.
static int require_owner(const nidx_txt_segment* t) {
    if (!t) return fail(NIDX_EINVAL, "null segment");
    return t->own ? 0 : fail(NIDX_EINVAL, "a view (nidx_txt_view) cannot be changed");
}

int nidx_txt_set_stats(nidx_txt_segment* t, uint64_t total_docs, uint64_t total_tokens, const uint64_t* doc_freq) {
    int r = require_owner(t);
    if (r) return r;
    if (!total_docs) return fail(NIDX_EINVAL, "bad argument");
    CU(cudaSetDevice(t->ix->device));
    return txt_upload_stats(t, total_docs, total_tokens, doc_freq ? doc_freq : t->ix->own_df.data());
}

int nidx_txt_set_alive(nidx_txt_segment* t, const uint64_t* alive_bits) {
    int r = require_owner(t);
    if (r) return r;
    return set_rows(t->ix->device, t->d_alive, alive_bits, ((size_t)t->ix->n_docs + 63) / 64);
}

void nidx_txt_close(nidx_txt_segment* t) {
    if (!t) return;
    cudaSetDevice(t->ix->device);
    cudaDeviceSynchronize();
    delete t;
}

int nidx_txt_view(nidx_txt_segment* t, const uint64_t* mask_bits, int mem, nidx_txt_segment** out, void* stream_) {
    if (!t || !mask_bits || !out) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(t->ix->device));
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const size_t words = ((size_t)t->ix->n_docs + 63) / 64;
    std::unique_ptr<nidx_txt_segment> v(new nidx_txt_segment());
    v->ix = t->ix;
    ALLOC(v->d_alive, std::max<size_t>(words, 1) * 8);
    const uint64_t* d_mask = mask_bits;
    if (mem == NIDX_MEM_HOST && words) {
        CU(cudaMemcpyAsync(v->d_alive, mask_bits, words * 8, cudaMemcpyHostToDevice, stream));
        d_mask = v->d_alive;
    }
    if (words) {   // the parent's alive set AND the mask: one pass over the words, on the caller's stream
        and_bits_kernel<<<(unsigned)std::min<size_t>((words + 255) / 256, 1024), 256, 0, stream>>>(d_mask, t->d_alive, v->d_alive, words, nullptr);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    *out = v.release();
    return 0;
}

int nidx_txt_last_kernel_ms(nidx_txt_segment* t, float* ms) {
    if (!t || !ms) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(t->ix->device));
    CU(cudaEventSynchronize(t->ix->ev_k1));
    CU(cudaEventElapsedTime(ms, t->ix->ev_k0, t->ix->ev_k1));
    return 0;
}

}  // extern "C"

// nidx_txt_set_facets / nidx_txt_set_doc_groups: checks the dictionary and the CSR, uploads them and only then replaces `col`, so a
// rejected or failed call leaves the previous column in place.  `what` names the column in errors.
static int set_ord_column(nidx_txt_segment* t, OrdColumn TxtIndex::*column, const char* what, uint32_t n_keys, const uint8_t* key_bytes, const uint64_t* key_off,
                          const uint64_t* doc_off, const uint32_t* doc_ords) {
    int r = require_owner(t);
    if (r) return r;
    if (!doc_off || (n_keys && (!key_bytes || !key_off))) return fail(NIDX_EINVAL, "null argument");
    std::vector<std::string> keys(n_keys);
    for (uint32_t i = 0; i < n_keys; ++i) {
        keys[i].assign(reinterpret_cast<const char*>(key_bytes) + key_off[i], key_off[i + 1] - key_off[i]);
        if (i && !(keys[i - 1] < keys[i])) return fail(NIDX_EINVAL, "%s keys must be strictly ascending (facet order)", what);
    }
    const uint32_t n_docs = t->ix->n_docs;
    const uint64_t nnz = doc_off[n_docs];
    if (nnz >= (1ull << 32)) return fail(NIDX_EINVAL, "at most 2^32-1 %s ords per segment", what);
    if (nnz && !doc_ords) return fail(NIDX_EINVAL, "null argument");
    std::vector<uint32_t> off(n_docs + 1);
    for (uint32_t d = 0; d <= n_docs; ++d) {
        if (d && doc_off[d] < doc_off[d - 1]) return fail(NIDX_EINVAL, "doc_off must be non-decreasing");
        off[d] = (uint32_t)doc_off[d];
    }
    for (uint32_t d = 0; d < n_docs; ++d)
        for (uint64_t i = doc_off[d]; i < doc_off[d + 1]; ++i)
            if (doc_ords[i] >= n_keys || (i > doc_off[d] && doc_ords[i] <= doc_ords[i - 1]))
                return fail(NIDX_EINVAL, "document %u: %s ords must be < n_%ss and strictly ascending", d, what, what);
    CU(cudaSetDevice(t->ix->device));
    DevArray<uint32_t> d_off, d_ord;
    ALLOC(d_off, ((size_t)n_docs + 1) * 4);
    ALLOC(d_ord, std::max<uint64_t>(nnz, 1) * 4);
    CU(cudaMemcpy(d_off, off.data(), off.size() * 4, cudaMemcpyHostToDevice));
    if (nnz) CU(cudaMemcpy(d_ord, doc_ords, nnz * 4, cudaMemcpyHostToDevice));
    OrdColumn& col = t->ix->*column;
    col.d_off = std::move(d_off);
    col.d_ord = std::move(d_ord);
    col.keys = std::move(keys);
    col.n_ords = nnz;
    return 0;
}

extern "C" {

int nidx_txt_set_facets(nidx_txt_segment* t, uint32_t n_facets, const uint8_t* key_bytes, const uint64_t* key_off, const uint64_t* doc_off,
                        const uint32_t* doc_ords) {
    return set_ord_column(t, &TxtIndex::facets, "facet", n_facets, key_bytes, key_off, doc_off, doc_ords);
}

int nidx_txt_set_doc_groups(nidx_txt_segment* t, uint32_t n_groups, const uint8_t* key_bytes, const uint64_t* key_off, const uint64_t* doc_off,
                            const uint32_t* doc_ords) {
    return set_ord_column(t, &TxtIndex::groups, "group", n_groups, key_bytes, key_off, doc_off, doc_ords);
}

int nidx_txt_set_dates(nidx_txt_segment* t, const int64_t* created, const int64_t* modified) {
    if (!t || !created || !modified) return fail(NIDX_EINVAL, "null argument");
    int r = require_owner(t);
    if (r) return r;
    CU(cudaSetDevice(t->ix->device));
    const uint32_t n = t->ix->n_docs;
    const size_t padded = std::max<size_t>(((size_t)n + 7) & ~(size_t)7, 8);
    // ranks: sort (seconds, doc) on the device, flag the first document of every distinct date, inclusive prefix sum, scatter
    DevArray<int64_t> d_sorted, secs[2];
    DevArray<uint32_t> d_doc, d_doc_sorted, d_flag, d_incl, rank[2];
    DevBuf d_cub;
    uint32_t n_ranks[2] = {0, 0};
    size_t sort_bytes = 0, scan_bytes = 0;
    if (n) {
        ALLOC(d_sorted, (size_t)n * 8);
        ALLOC(d_doc, (size_t)n * 4);
        ALLOC(d_doc_sorted, (size_t)n * 4);
        ALLOC(d_flag, (size_t)n * 4);
        ALLOC(d_incl, (size_t)n * 4);
        std::vector<uint32_t> iota(n);
        for (uint32_t i = 0; i < n; ++i) iota[i] = i;
        CU(cudaMemcpy(d_doc, iota.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
        CU(cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, (const int64_t*)nullptr, d_sorted.p, d_doc.p, d_doc_sorted.p, (int)n));
        CU(cub::DeviceScan::InclusiveSum(nullptr, scan_bytes, d_flag.p, d_incl.p, (int)n));
        ALLOC(d_cub, std::max(sort_bytes, scan_bytes));
    }
    const int blocks = std::max(1, std::min<int>(t->ix->sm_count * 8, (int)((n + 255) / 256)));
    for (int f = 0; f < 2; ++f) {
        ALLOC(secs[f], std::max<size_t>(n, 1) * 8);
        ALLOC(rank[f], padded * 4);
        CU(cudaMemset(rank[f], 0, padded * 4));
        if (!n) continue;
        CU(cudaMemcpy(secs[f], f == 0 ? created : modified, (size_t)n * 8, cudaMemcpyHostToDevice));
        size_t tmp = sort_bytes;
        CU(cub::DeviceRadixSort::SortPairs(d_cub.p, tmp, (const int64_t*)secs[f].p, d_sorted.p, d_doc.p, d_doc_sorted.p, (int)n));
        LAUNCHED();
        date_flag_kernel<<<blocks, 256>>>(d_sorted, n, d_flag);
        LAUNCHED();
        tmp = scan_bytes;
        CU(cub::DeviceScan::InclusiveSum(d_cub.p, tmp, d_flag.p, d_incl.p, (int)n));
        LAUNCHED();
        date_scatter_kernel<<<blocks, 256>>>(d_incl, d_doc_sorted, n, rank[f]);
        LAUNCHED();
        CU(cudaGetLastError());
        CU(cudaMemcpy(&n_ranks[f], d_incl + n - 1, 4, cudaMemcpyDeviceToHost));
    }
    CU(cudaDeviceSynchronize());
    for (int f = 0; f < 2; ++f) {   // only now: a failed call leaves the previous dates in place
        t->ix->d_secs[f] = std::move(secs[f]);
        t->ix->d_rank[f] = std::move(rank[f]);
        t->ix->n_ranks[f] = n_ranks[f];
    }
    return 0;
}

int nidx_txt_set_positions(nidx_txt_segment* t, const uint32_t* positions, uint64_t n_positions) {
    if (!t || (n_positions && !positions)) return fail(NIDX_EINVAL, "null argument");
    int r = require_owner(t);
    if (r) return r;
    CU(cudaSetDevice(t->ix->device));
    const uint64_t n = t->ix->n_post;
    DevArray<uint64_t> tf, pos_off;
    DevArray<uint32_t> pos;
    DevArray<unsigned int> flags;   // [0] a tf was clamped when packed, [1] positions not strictly ascending
    DevBuf d_cub;
    ALLOC(tf, (n + 1) * 8);
    ALLOC(pos_off, (n + 1) * 8);
    ALLOC(pos, std::max<uint64_t>(n_positions, 1) * 4);
    ALLOC(flags, 8);
    CU(cudaMemset(flags, 0, 8));
    const int blocks = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)t->ix->sm_count * 8, (n + 256) / 256));
    pos_tf_kernel<<<blocks, 256>>>(t->ix->d_post, n, tf, flags);
    LAUNCHED();
    size_t scan_bytes = 0;
    CU(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, tf.p, pos_off.p, n + 1));
    ALLOC(d_cub, std::max<size_t>(scan_bytes, 1));
    CU(cub::DeviceScan::ExclusiveSum(d_cub.p, scan_bytes, tf.p, pos_off.p, n + 1));
    LAUNCHED();
    unsigned int h_flags[2];
    uint64_t total = 0;
    CU(cudaMemcpy(h_flags, flags, 8, cudaMemcpyDeviceToHost));
    CU(cudaMemcpy(&total, pos_off + n, 8, cudaMemcpyDeviceToHost));
    if (h_flags[0]) return fail(NIDX_EINVAL, "a term frequency of the segment does not fit 24 bits: its positions cannot be located");
    if (total != n_positions) return fail(NIDX_EINVAL, "%llu positions given, the postings' term frequencies sum to %llu",
                                          (unsigned long long)n_positions, (unsigned long long)total);
    if (n_positions) CU(cudaMemcpy(pos, positions, n_positions * 4, cudaMemcpyHostToDevice));
    pos_check_kernel<<<blocks, 256>>>(pos_off, pos, n, flags + 1);
    LAUNCHED();
    CU(cudaGetLastError());
    CU(cudaMemcpy(h_flags, flags, 8, cudaMemcpyDeviceToHost));
    if (h_flags[1]) return fail(NIDX_EINVAL, "the positions of every posting must be strictly ascending");
    t->ix->d_pos_off = std::move(pos_off);   // only now: a rejected or failed call leaves the previous positions in place
    t->ix->d_pos = std::move(pos);
    return 0;
}

}  // extern "C"

// The phrases of a batch (nidx_txt_phrases) laid out for phrase.cuh and bm25_body: grouped by query (stable), each phrase's driver
// (its rarest term in the segment) and slots (the driver's df), weight and skip row.  One host buffer, uploaded in one copy.
struct PhrasePlan {
    std::vector<unsigned char> buf;
    size_t o_qoff, o_terms, o_off, o_driver, o_skip_row, o_row_term, o_cap_off, o_weight, o_range, o_post, o_skip;
    uint32_t nv = 0, n_rows = 0;
    uint64_t slots = 0;
    size_t bytes = 0;
};

static int phrase_plan(const nidx_txt_segment* t, const nidx_txt_phrases* ph, int32_t nq, const std::vector<uint32_t>& h_off, PhrasePlan& P) {
    if (ph->n < 0 || (ph->n && (!ph->terms || !ph->off || !ph->query))) return fail(NIDX_EINVAL, "bad phrases");
    if (!t->ix->d_pos) return fail(NIDX_EINVAL, "the segment has no positions (nidx_txt_set_positions)");
    const uint32_t nv = (uint32_t)ph->n;
    std::vector<uint32_t> per_q(nq + 1, 0);
    for (uint32_t i = 0; i < nv; ++i) {
        const uint32_t m = ph->off[i + 1] - ph->off[i];
        if (ph->off[i + 1] < ph->off[i] || m < 2 || m > PHRASE_MAX_TERMS) return fail(NIDX_EINVAL, "a phrase has 2 to %d terms", PHRASE_MAX_TERMS);
        if (ph->query[i] >= (uint32_t)nq) return fail(NIDX_EINVAL, "phrase %u belongs to no query of the batch", i);
        ++per_q[ph->query[i] + 1];
    }
    for (int32_t q = 0; q < nq; ++q) {
        if (h_off[q + 1] - h_off[q] + per_q[q + 1] > (uint32_t)BM_MAX_TERMS)
            return fail(NIDX_EINVAL, "queries with more than %d clauses (terms and phrases) are not supported", BM_MAX_TERMS);
        per_q[q + 1] += per_q[q];
    }
    std::vector<uint32_t> order(nv), terms, off(nv + 1, 0), driver(nv), skip_row(nv, NIDX_NIL), row_term;
    std::vector<uint64_t> cap_off(nv + 1, 0);
    std::vector<float> weight(nv);
    {
        std::vector<uint32_t> at(per_q.begin(), per_q.end() - 1);
        for (uint32_t i = 0; i < nv; ++i) order[at[ph->query[i]]++] = i;
    }
    const float K1 = 1.2f;
    for (uint32_t v = 0; v < nv; ++v) {
        const uint32_t i = order[v];
        bool known = true;
        uint32_t dv = 0;
        uint64_t cap = ~0ull;
        float idf = 0.0f;   // f32 sum in phrase order, repeats counted (Bm25Weight::for_terms) [recalled]
        for (uint32_t j = ph->off[i]; j < ph->off[i + 1]; ++j) {
            const uint32_t term = ph->terms[j];
            terms.push_back(term);
            if (term >= t->ix->n_terms) { known = false; continue; }
            idf += t->ix->idf[term];
            if (t->ix->own_df[term] < cap) { cap = t->ix->own_df[term]; dv = j - ph->off[i]; }
        }
        if (!known) cap = 0;   // a term the segment's dictionary lacks: the phrase matches nothing and weighs 0, like the term alone
        off[v + 1] = (uint32_t)terms.size();
        driver[v] = dv;
        cap_off[v + 1] = cap_off[v] + cap;
        weight[v] = known ? idf * (1.0f + K1) : 0.0f;
        if (cap >= (uint64_t)BM_SKIP_DF) { skip_row[v] = (uint32_t)row_term.size(); row_term.push_back(2 * v); }
    }
    // one buffer: inputs first (copied), then the outputs of the phrase pass
    auto take = [&](size_t& o, size_t bytes) { o = (P.bytes + 15) & ~(size_t)15; P.bytes = o + bytes; };
    take(P.o_qoff, per_q.size() * 4);
    take(P.o_terms, std::max<size_t>(terms.size(), 1) * 4);
    take(P.o_off, off.size() * 4);
    take(P.o_driver, std::max<size_t>(nv, 1) * 4);
    take(P.o_skip_row, std::max<size_t>(nv, 1) * 4);
    take(P.o_row_term, std::max<size_t>(row_term.size(), 1) * 4);
    take(P.o_cap_off, cap_off.size() * 8);
    take(P.o_weight, std::max<size_t>(nv, 1) * 4);
    const size_t in_bytes = P.bytes;
    take(P.o_range, std::max<size_t>(nv, 1) * 16);
    take(P.o_post, std::max<uint64_t>(cap_off[nv], 1) * 8);
    take(P.o_skip, std::max<size_t>(row_term.size(), 1) * ((size_t)t->ix->n_fine + 1) * 4);
    P.buf.assign(in_bytes, 0);
    auto put = [&](size_t o, const auto& v) { if (!v.empty()) memcpy(P.buf.data() + o, v.data(), v.size() * sizeof(v[0])); };
    put(P.o_qoff, per_q); put(P.o_terms, terms); put(P.o_off, off); put(P.o_driver, driver); put(P.o_skip_row, skip_row);
    put(P.o_row_term, row_term); put(P.o_cap_off, cap_off); put(P.o_weight, weight);
    P.nv = nv; P.n_rows = (uint32_t)row_term.size(); P.slots = cap_off[nv];
    return 0;
}

// Uploads the plan into w.phrases, runs the phrase pass on `stream` and points a's overlay at its lists.
static int phrase_pass(nidx_txt_segment* t, const PhrasePlan& P, const TxtDev& T, Workspace& w, cudaStream_t stream, Bm25Args& a) {
    ENSURE(w.phrases, P.bytes);
    unsigned char* d = w.phrases.p;
    CU(cudaMemcpyAsync(d, P.buf.data(), P.buf.size(), cudaMemcpyHostToDevice, stream));
    PhraseArgs A;
    A.pos_off = t->ix->d_pos_off; A.pos = t->ix->d_pos;
    A.terms = reinterpret_cast<const uint32_t*>(d + P.o_terms); A.off = reinterpret_cast<const uint32_t*>(d + P.o_off);
    A.driver = reinterpret_cast<const uint32_t*>(d + P.o_driver); A.cap_off = reinterpret_cast<const uint64_t*>(d + P.o_cap_off);
    A.nv = P.nv; A.out = reinterpret_cast<uint2*>(d + P.o_post); A.range = reinterpret_cast<uint64_t*>(d + P.o_range);
    if (P.slots) {
        const int blocks = (int)std::min<uint64_t>((uint64_t)t->ix->sm_count * 8, (P.slots + 255) / 256);
        phrase_match_kernel<<<blocks, 256, 0, stream>>>(T, A);
        LAUNCHED();
    }
    phrase_compact_kernel<<<P.nv, PHRASE_COMPACT_THREADS, 0, stream>>>(A);
    LAUNCHED();
    if (P.n_rows) {
        bm25_build_skip_kernel<<<t->ix->sm_count * 8, 256, 0, stream>>>(A.range, A.out, reinterpret_cast<const uint32_t*>(d + P.o_row_term), P.n_rows, t->ix->n_fine,
                                                                    reinterpret_cast<uint32_t*>(d + P.o_skip));
        LAUNCHED();
    }
    a.ph_qoff = reinterpret_cast<const uint32_t*>(d + P.o_qoff); a.ph_range = A.range; a.ph_post = A.out;
    a.ph_skip_row = reinterpret_cast<const uint32_t*>(d + P.o_skip_row); a.ph_skip = reinterpret_cast<const uint32_t*>(d + P.o_skip);
    a.ph_weight = reinterpret_cast<const float*>(d + P.o_weight);
    return 0;
}

// An order resolved against the segment: the field's rank column and seconds.
static int order_args(const nidx_txt_segment* t, const nidx_txt_order* order, OrderArgs& O) {
    if (!order || (order->field != NIDX_ORDER_CREATED && order->field != NIDX_ORDER_MODIFIED) || (order->type != NIDX_ORDER_DESC && order->type != NIDX_ORDER_ASC))
        return fail(NIDX_EINVAL, "bad order");
    if (!t->ix->d_rank[order->field]) return fail(NIDX_EINVAL, "the segment has no dates (nidx_txt_set_dates)");
    O.rank = t->ix->d_rank[order->field];
    O.secs = t->ix->d_secs[order->field];
    O.n_ranks = t->ix->n_ranks[order->field];
    O.asc = order->type == NIDX_ORDER_ASC;
    return 0;
}

// A facet request resolved against the segment's dictionary: bucket[ord] = the bucket of the requested facet's child the ord lies
// under (NIL: none), and per bucket the request it belongs to and the first ord under its child (what names it).  Requests are
// taken in facet order, so buckets ascend with the ord.
struct FacetPlan {
    std::vector<uint32_t> bucket, b_req, b_ord;
};

static int facet_plan(const nidx_txt_segment* t, const nidx_txt_facet_request* r, FacetPlan& P) {
    if (!r || r->n < 0 || (r->n && (!r->key_bytes || !r->key_off))) return fail(NIDX_EINVAL, "bad facet request");
    if (!t->ix->facets.d_off) return fail(NIDX_ESTATE, "the segment has no facets (nidx_txt_set_facets)");
    std::vector<std::pair<std::string, int>> req;
    for (int i = 0; i < r->n; ++i) req.emplace_back(std::string(reinterpret_cast<const char*>(r->key_bytes) + r->key_off[i], r->key_off[i + 1] - r->key_off[i]), i);
    std::sort(req.begin(), req.end());
    req.erase(std::unique(req.begin(), req.end(), [](const auto& x, const auto& y) { return x.first == y.first; }), req.end());   // duplicates collapse
    // tantivy's FacetCollector::add_facet asserts that no requested facet is an ancestor of another: here an error.  In facet
    // order an ancestor is immediately followed by one of its descendants (the root "" by anything).
    for (size_t i = 0; i + 1 < req.size(); ++i) {
        const std::string &a = req[i].first, &b = req[i + 1].first;
        if (a.empty() || (b.size() > a.size() && b.compare(0, a.size(), a) == 0 && b[a.size()] == '\0'))
            return fail(NIDX_EINVAL, "a requested facet is an ancestor of another requested facet");
    }
    const std::vector<std::string>& K = t->ix->facets.keys;
    P.bucket.assign(K.size(), NIDX_NIL);
    P.b_req.clear(); P.b_ord.clear();
    for (const auto& [f, idx] : req) {
        const std::string prefix = f.empty() ? f : f + '\0';   // the root's children are the top-level facets
        size_t o = std::lower_bound(K.begin(), K.end(), prefix) - K.begin();
        std::string child;
        for (; o < K.size() && K[o].compare(0, prefix.size(), prefix) == 0; ++o) {
            if (K[o].size() == prefix.size()) continue;   // the root key "": the requested facet itself counts nothing
            size_t end = K[o].find('\0', prefix.size());
            std::string c = K[o].substr(0, end);
            if (P.b_req.empty() || c != child) { child = c; P.b_req.push_back((uint32_t)idx); P.b_ord.push_back((uint32_t)o); }
            P.bucket[o] = (uint32_t)P.b_req.size() - 1;
        }
    }
    return 0;
}

// Uploads the plan's collapse table into the workspace and fills F (the counts go to d_out: [rows][n_buckets]).
static int facet_args(const nidx_txt_segment* t, const FacetPlan& P, Workspace& w, uint32_t* d_out, cudaStream_t stream, FacetArgs& F) {
    ENSURE(w.facets, std::max<size_t>(P.bucket.size(), 1) * 4);
    if (!P.bucket.empty()) CU(cudaMemcpyAsync(w.facets.p, P.bucket.data(), P.bucket.size() * 4, cudaMemcpyHostToDevice, stream));
    F.doc_off = t->ix->facets.d_off; F.ords = t->ix->facets.d_ord; F.bucket = w.facets.as<uint32_t>();
    F.n_buckets = (uint32_t)P.b_req.size();
    F.smem = F.n_buckets <= FACET_SMEM_BUCKETS;
    F.out = d_out;
    return 0;
}

// The body of nidx_txt_search (facets == nullptr), nidx_txt_search_faceted and nidx_txt_search_ordered (order != nullptr: dates to
// out_dates instead of scores to out_scores).  qhost / ohost as in vec_search_impl.
static int txt_search_impl(nidx_txt_segment* t, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, bool qhost, bool ohost,
                           const nidx_txt_search_params* p, uint32_t* out_docs, float* out_scores, int32_t* out_counts, uint64_t* out_total, cudaStream_t stream,
                           const nidx_txt_facet_request* facets = nullptr, uint32_t* out_facet_counts = nullptr, const nidx_txt_order* order = nullptr,
                           int64_t* out_dates = nullptr, const nidx_txt_phrases* phrases = nullptr) {
    if (!t || !p || !query_off || !out_docs || !(order ? (void*)out_dates : (void*)out_scores) || !out_counts) return fail(NIDX_EINVAL, "null argument");
    FacetPlan plan;
    if (facets) {
        if (!out_facet_counts) return fail(NIDX_EINVAL, "null argument");
        int r = facet_plan(t, facets, plan);
        if (r) return r;
    }
    OrderArgs O{};
    if (order) {
        int r = order_args(t, order, O);
        if (r) return r;
    }
    if (nq <= 0) return 0;
    int k = p->k;
    if (k <= 0 || k > 1024) return fail(NIDX_EINVAL, "k must be in 1..1024");
    CU(cudaSetDevice(t->ix->device));
    WsGuard g(t->ix->pool, stream);
    Workspace& w = *g.w;
    // query offsets are needed on the host to size things
    std::vector<uint32_t> h_off(nq + 1);
    if (qhost) memcpy(h_off.data(), query_off, ((size_t)nq + 1) * 4);
    else { CU(cudaMemcpyAsync(h_off.data(), query_off, ((size_t)nq + 1) * 4, cudaMemcpyDeviceToHost, stream)); CU(cudaStreamSynchronize(stream)); }
    uint32_t n_qt = h_off[nq];
    int max_terms = 0;
    for (int i = 0; i < nq; ++i) max_terms = std::max<int>(max_terms, h_off[i + 1] - h_off[i]);
    if (max_terms > BM_MAX_TERMS) return fail(NIDX_EINVAL, "queries with more than %d terms are not supported", BM_MAX_TERMS);
    PhrasePlan pp;
    if (phrases && phrases->n) {
        int r = phrase_plan(t, phrases, nq, h_off, pp);
        if (r) return r;
    }
    bool conj = p->mode == NIDX_BM25_AND;
    int cap = topk_cap(k, BM_THREADS);
    size_t smem = bm_smem_bytes(cap, conj);
    if (smem > 220 * 1024) return fail(NIDX_EINVAL, "BM25 needs %zu bytes of shared memory (k=%d): too large", smem, k);
    ENSURE(w.partial, (size_t)nq * k * 8);
    const size_t nb = plan.b_req.size();
    Stage st(stream, qhost, ohost);
    const uint32_t *d_qt, *d_qo;
    uint32_t *d_docs, *d_fc = nullptr;
    float* d_sc = nullptr;
    int64_t* d_dates = nullptr;
    int* d_cnt;
    uint64_t* d_total;
    st.in(query_off, (size_t)nq + 1, &d_qo);
    st.in(query_terms, n_qt, &d_qt);
    st.out(out_docs, (size_t)nq * k, &d_docs);
    if (order) st.out(out_dates, (size_t)nq * k, &d_dates);
    else st.out(out_scores, (size_t)nq * k, &d_sc);
    st.out(out_counts, (size_t)nq, &d_cnt);
    st.out(out_total, (size_t)nq, &d_total);
    if (facets) st.out(out_facet_counts, (size_t)nq * nb, &d_fc);
    int r = st.place(w.stage);
    if (r) return r;
    TxtDev T;
    T.n_docs = t->ix->n_docs; T.n_terms = t->ix->n_terms; T.n_fine = t->ix->n_fine; T.term_off = t->ix->d_term_off; T.post = t->ix->d_post;
    T.skip_row = t->ix->d_skip_row; T.skip = t->ix->d_skip; T.alive = t->d_alive;
    Bm25Args a;
    a.query_terms = d_qt; a.query_off = d_qo; a.nq = nq; a.k = k; a.cap = cap;
    a.term_weight = t->ix->d_weight; a.norm_cache = t->ix->d_norm_cache;
    a.after_mode = p->after_mode; a.after_score = p->after_score; a.after_docaddr = p->after_docaddr; a.docaddr_base = p->docaddr_base;
    a.out_keys = w.partial.as<uint64_t>(); a.out_total = reinterpret_cast<unsigned long long*>(d_total);
    if (order) a.after_mode = 0;   // TopDocs::order_by_fast_field: no search-after
    a.ph_qoff = nullptr; a.ph_range = nullptr; a.ph_post = nullptr; a.ph_skip_row = nullptr; a.ph_skip = nullptr; a.ph_weight = nullptr;
    // a phrase scores its frequency: beside Basic terms the TF kernel runs with the terms' tf taken as 1 (the same two roundings)
    const bool use_tf = p->use_tf || pp.nv;
    a.basic_terms = !p->use_tf && pp.nv;
    if (pp.nv) {
        r = phrase_pass(t, pp, T, w, stream, a);
        if (r) return r;
    }
    auto launch = [&](auto kern, size_t bytes, auto... extra) -> int {   // the BM25 pass, between the roofline events
        CU(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
        CU(cudaEventRecord(t->ix->ev_k0, stream));
        kern<<<nq, BM_THREADS, bytes, stream>>>(T, a, extra...);
        CU(cudaEventRecord(t->ix->ev_k1, stream));
        LAUNCHED();
        return 0;
    };
    FacetArgs F;
    size_t fsmem = smem;
    if (facets) {
        r = facet_args(t, plan, w, d_fc, stream, F);
        if (r) return r;
        if (F.smem && smem + nb * 4 > 220 * 1024) F.smem = 0;
        if (!F.smem && nb) CU(cudaMemsetAsync(d_fc, 0, (size_t)nq * nb * 4, stream));
        fsmem += F.smem ? nb * 4 : 0;
    }
    if (order && !facets) r = launch(conj ? bm25_order_kernel<true> : bm25_order_kernel<false>, smem, O);
    else if (!facets)
        r = launch(conj ? (use_tf ? bm25_kernel<true, true> : bm25_kernel<true, false>) : (use_tf ? bm25_kernel<false, true> : bm25_kernel<false, false>),
                   smem);
    else if (order) r = launch(conj ? bm25_order_facet_kernel<true> : bm25_order_facet_kernel<false>, fsmem, F, O);
    else
        r = launch(conj ? (use_tf ? bm25_facet_kernel<true, true> : bm25_facet_kernel<true, false>)
                        : (use_tf ? bm25_facet_kernel<false, true> : bm25_facet_kernel<false, false>), fsmem, F);
    if (r) return r;
    if (order) date_finish_kernel<<<nq, 128, 0, stream>>>(w.partial.as<uint64_t>(), nq, k, O.secs, d_docs, d_dates, d_cnt);
    else bm25_finish_kernel<<<nq, 128, 0, stream>>>(w.partial.as<uint64_t>(), nq, k, p->min_score, d_docs, d_sc, d_cnt);
    LAUNCHED();
    CU(cudaGetLastError());
    return st.finish();
}

extern "C" {

int nidx_txt_search(nidx_txt_segment* t, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem, const nidx_txt_search_params* p,
                    uint32_t* out_docs, float* out_scores, int32_t* out_counts, uint64_t* out_total, void* stream_) {
    bool host = mem == NIDX_MEM_HOST;
    return txt_search_impl(t, query_terms, query_off, nq, host, host, p, out_docs, out_scores, out_counts, out_total, reinterpret_cast<cudaStream_t>(stream_));
}

int nidx_txt_facet_buckets(nidx_txt_segment* t, const nidx_txt_facet_request* facets, uint32_t* out_bucket_req, uint32_t* out_bucket_ord, uint32_t cap,
                           uint32_t* out_n_buckets) {
    if (!t || !out_n_buckets) return fail(NIDX_EINVAL, "null argument");
    FacetPlan plan;
    int r = facet_plan(t, facets, plan);
    if (r) return r;
    const size_t n = std::min<size_t>(plan.b_req.size(), cap);
    if (n && (!out_bucket_req || !out_bucket_ord)) return fail(NIDX_EINVAL, "null argument");
    if (n) { memcpy(out_bucket_req, plan.b_req.data(), n * 4); memcpy(out_bucket_ord, plan.b_ord.data(), n * 4); }
    *out_n_buckets = (uint32_t)plan.b_req.size();
    return 0;
}

int nidx_txt_search_faceted(nidx_txt_segment* t, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem, const nidx_txt_search_params* p,
                            const nidx_txt_facet_request* facets, uint32_t* out_docs, float* out_scores, int32_t* out_counts, uint64_t* out_total,
                            uint32_t* out_facet_counts, void* stream_) {
    if (!facets) return fail(NIDX_EINVAL, "null argument");
    bool host = mem == NIDX_MEM_HOST;
    return txt_search_impl(t, query_terms, query_off, nq, host, host, p, out_docs, out_scores, out_counts, out_total, reinterpret_cast<cudaStream_t>(stream_),
                           facets, out_facet_counts);
}

int nidx_txt_facet_count_all(nidx_txt_segment* t, const nidx_txt_facet_request* facets, int mem, uint32_t* out_facet_counts, void* stream_) {
    if (!t || !out_facet_counts) return fail(NIDX_EINVAL, "null argument");
    FacetPlan plan;
    int r = facet_plan(t, facets, plan);
    if (r) return r;
    const size_t nb = plan.b_req.size();
    if (!nb) return 0;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    CU(cudaSetDevice(t->ix->device));
    WsGuard g(t->ix->pool, stream);
    Workspace& w = *g.w;
    Stage st(stream, host, host);
    uint32_t* d_fc;
    st.out(out_facet_counts, nb, &d_fc);
    r = st.place(w.stage);
    FacetArgs F;
    if (!r) r = facet_args(t, plan, w, d_fc, stream, F);
    if (r) return r;
    CU(cudaMemsetAsync(d_fc, 0, nb * 4, stream));
    const int threads = 256;
    const int blocks = std::max(1, std::min<int>(t->ix->sm_count * (2048 / threads), (int)((t->ix->n_docs + threads - 1) / threads)));
    CU(cudaEventRecord(t->ix->ev_k0, stream));
    facet_count_all_kernel<<<blocks, threads, F.smem ? nb * 4 : 0, stream>>>(t->ix->n_docs, t->d_alive, F);
    CU(cudaEventRecord(t->ix->ev_k1, stream));
    LAUNCHED();
    CU(cudaGetLastError());
    return st.finish();
}

int nidx_txt_search_ordered(nidx_txt_segment* t, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem, const nidx_txt_search_params* p,
                            const nidx_txt_order* order, const nidx_txt_facet_request* facets, uint32_t* out_docs, int64_t* out_dates, int32_t* out_counts,
                            uint64_t* out_total, uint32_t* out_facet_counts, void* stream_) {
    if (!order) return fail(NIDX_EINVAL, "null argument");
    bool host = mem == NIDX_MEM_HOST;
    return txt_search_impl(t, query_terms, query_off, nq, host, host, p, out_docs, nullptr, out_counts, out_total, reinterpret_cast<cudaStream_t>(stream_),
                           facets, out_facet_counts, order, out_dates);
}

int nidx_txt_search_phrases(nidx_txt_segment* t, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem, const nidx_txt_search_params* p,
                            const nidx_txt_phrases* phrases, const nidx_txt_order* order, const nidx_txt_facet_request* facets, uint32_t* out_docs,
                            float* out_scores, int64_t* out_dates, int32_t* out_counts, uint64_t* out_total, uint32_t* out_facet_counts, void* stream_) {
    if (!phrases) return fail(NIDX_EINVAL, "null argument");
    bool host = mem == NIDX_MEM_HOST;
    return txt_search_impl(t, query_terms, query_off, nq, host, host, p, out_docs, order ? nullptr : out_scores, out_counts, out_total,
                           reinterpret_cast<cudaStream_t>(stream_), facets, out_facet_counts, order, out_dates, phrases);
}

int nidx_txt_list_ordered(nidx_txt_segment* t, const nidx_txt_order* order, int32_t k, int mem, uint32_t* out_docs, int64_t* out_dates, int32_t* out_count,
                          uint64_t* out_total, void* stream_) {
    if (!t || !out_docs || !out_dates || !out_count) return fail(NIDX_EINVAL, "null argument");
    OrderArgs O;
    int r = order_args(t, order, O);
    if (r) return r;
    if (k <= 0 || k > 1024) return fail(NIDX_EINVAL, "k must be in 1..1024");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    CU(cudaSetDevice(t->ix->device));
    WsGuard g(t->ix->pool, stream);
    Workspace& w = *g.w;
    // per-CTA top-k over a grid-stride slice, then one merge (the scan_select / topk_merge pattern)
    const int threads = 512;
    const int blocks = std::max(1, std::min<int>(t->ix->sm_count * 2, (int)(((size_t)t->ix->n_docs + threads * DATE_PT - 1) / (threads * DATE_PT))));
    const int cap = topk_cap(k, threads);
    ENSURE(w.partial, (size_t)blocks * k * 8);
    Stage st(stream, host, host);
    uint32_t* d_docs;
    int64_t* d_dates;
    int* d_cnt;
    uint64_t* d_total;
    st.out(out_docs, (size_t)k, &d_docs);
    st.out(out_dates, (size_t)k, &d_dates);
    st.out(out_count, 1, &d_cnt);
    st.out(out_total, 1, &d_total);
    r = st.place(w.stage);
    if (r) return r;
    CU(cudaFuncSetAttribute(date_topk_all_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap * 8));
    CU(cudaFuncSetAttribute(date_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap * 8));
    CU(cudaMemsetAsync(d_total, 0, 8, stream));
    CU(cudaEventRecord(t->ix->ev_k0, stream));
    date_topk_all_kernel<<<blocks, threads, (size_t)cap * 8, stream>>>(t->ix->n_docs, t->d_alive, O, k, cap, w.partial.as<uint64_t>(),
                                                                      reinterpret_cast<unsigned long long*>(d_total));
    LAUNCHED();
    date_merge_kernel<<<1, threads, (size_t)cap * 8, stream>>>(w.partial.as<uint64_t>(), blocks * k, k, cap, O.secs, d_docs, d_dates, d_cnt);
    LAUNCHED();
    CU(cudaEventRecord(t->ix->ev_k1, stream));
    CU(cudaGetLastError());
    return st.finish();
}

// ---- prefilter (prefilter.cuh) --------------------------------------------------------------------
// A handle-taking entry point without a device: NIDX_ENODEVICE (no handle can exist), else a NULL handle is NIDX_EINVAL.
static int require_handle(const void* h) {
    if (nidx_device_count() <= 0) return fail(NIDX_ENODEVICE, "no CUDA device available (nidx_b200 has no CPU fallback)");
    return h ? 0 : fail(NIDX_EINVAL, "null segment");
}

int nidx_txt_set_doc_columns(nidx_txt_segment* t, const uint32_t* resource_ord, const uint32_t* field_ord) {
    int r = require_handle(t);
    if (!r) r = require_owner(t);
    if (r) return r;
    if (t->ix->n_docs && (!resource_ord || !field_ord)) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(t->ix->device));
    DevArray<uint32_t> res, fld;
    const size_t n = t->ix->n_docs;
    ALLOC(res, std::max<size_t>(n, 1) * 4);
    ALLOC(fld, std::max<size_t>(n, 1) * 4);
    if (n) {
        CU(cudaMemcpy(res, resource_ord, n * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(fld, field_ord, n * 4, cudaMemcpyHostToDevice));
    }
    t->ix->d_res_ord = std::move(res);   // only now: a failed call leaves the previous columns in place
    t->ix->d_field_ord = std::move(fld);
    return 0;
}

}  // extern "C"

// An expression (pre-order nidx_prefilter_node) as the pass runs it: leaves and binary AND / OR in post-order, so that the bit stack
// never holds more than the nesting depth.  Keyword leaves get a bitset slot each: terms first, then phrases.
struct PrefilterPlan {
    std::vector<PfOp> prog;
    std::vector<uint32_t> terms;                       // term leaves, slot = index
    std::vector<uint32_t> ph_terms, ph_off{0}, ph_query;   // phrase leaves, slot = terms.size() + index
    bool facets = false, columns = false, groups = false, dates[2] = {false, false};

    int compile(const nidx_prefilter_node* nodes, int n_nodes, int& i, int depth) {
        if (i >= n_nodes) return fail(NIDX_EINVAL, "malformed prefilter expression (operand counts do not add up to %d nodes)", n_nodes);
        if (depth > NIDX_PREFILTER_MAX_DEPTH) return fail(NIDX_EINVAL, "the prefilter expression nests deeper than %d levels", NIDX_PREFILTER_MAX_DEPTH);
        const nidx_prefilter_node& nd = nodes[i++];
        PfOp o{};
        o.lo = nd.lo; o.hi = nd.hi;
        switch (nd.kind) {
            case NIDX_P_FACET: o.op = PF_FACET; facets = true; break;
            case NIDX_P_GROUP: o.op = PF_FACET; o.arg = 1; groups = true; break;
            case NIDX_P_PUBLIC: o.op = PF_PUBLIC; o.arg = 1; groups = true; break;
            case NIDX_P_FIELD: o.op = PF_FIELD; columns = true; break;
            case NIDX_P_RESOURCE: o.op = PF_RESOURCE; columns = true; break;
            case NIDX_P_DATE:
                if (nd.n != NIDX_ORDER_CREATED && nd.n != NIDX_ORDER_MODIFIED) return fail(NIDX_EINVAL, "prefilter node %d: bad date field", i - 1);
                o.op = PF_DATE; o.arg = (uint32_t)nd.n; dates[nd.n] = true;
                break;
            case NIDX_P_KEYWORD:
                if (nd.n < 0 || nd.n > PHRASE_MAX_TERMS || (nd.n && !nd.terms)) return fail(NIDX_EINVAL, "prefilter node %d: a keyword has 0 to %d terms", i - 1, PHRASE_MAX_TERMS);
                if (nd.n == 0) { o.op = PF_CONST; o.arg = 0; break; }
                o.op = PF_BITS;
                if (nd.n == 1) { o.arg = (uint32_t)terms.size(); terms.push_back(nd.terms[0]); break; }
                o.arg = 0x80000000u | (uint32_t)ph_query.size();   // a phrase slot, resolved once the number of term leaves is known
                ph_query.push_back((uint32_t)ph_query.size() / BM_MAX_TERMS);   // at most BM_MAX_TERMS phrases per query of the phrase pass
                ph_terms.insert(ph_terms.end(), nd.terms, nd.terms + nd.n);
                ph_off.push_back((uint32_t)ph_terms.size());
                break;
            case NIDX_P_ALL: o.op = PF_CONST; o.arg = 1; break;
            case NIDX_P_AND: case NIDX_P_OR: {
                if (nd.n < 0) return fail(NIDX_EINVAL, "prefilter node %d: bad operand count", i - 1);
                if (nd.n == 0) { o.op = PF_CONST; o.arg = 0; break; }   // a BooleanQuery without clauses matches nothing
                for (int c = 0; c < nd.n; ++c) {
                    int r = compile(nodes, n_nodes, i, depth + 1);
                    if (r) return r;
                    if (c) { PfOp b{}; b.op = nd.kind == NIDX_P_AND ? PF_AND : PF_OR; prog.push_back(b); }
                }
                return 0;
            }
            case NIDX_P_NOT: {
                if (nd.n != 1) return fail(NIDX_EINVAL, "prefilter node %d: NOT takes one operand", i - 1);
                int r = compile(nodes, n_nodes, i, depth + 1);
                if (r) return r;
                o.op = PF_NOT;
                break;
            }
            default: return fail(NIDX_EINVAL, "prefilter node %d: bad kind %d", i - 1, nd.kind);
        }
        prog.push_back(o);
        return 0;
    }
};

extern "C" {

int nidx_txt_prefilter(nidx_txt_segment* t, const nidx_prefilter_node* nodes, int32_t n_nodes, uint64_t* out_bits, int mem, uint64_t* out_matching,
                       void* stream_) {
    int r = require_handle(t);
    if (r) return r;
    if (!nodes || n_nodes <= 0) return fail(NIDX_EINVAL, "empty prefilter expression");
    PrefilterPlan P;
    int at = 0;
    r = P.compile(nodes, n_nodes, at, 1);
    if (r) return r;
    if (at != n_nodes) return fail(NIDX_EINVAL, "malformed prefilter expression (operand counts do not add up to %d nodes)", n_nodes);
    if (P.facets && !t->ix->facets.d_off) return fail(NIDX_ESTATE, "the segment has no facets (nidx_txt_set_facets)");
    if (P.columns && !t->ix->d_res_ord) return fail(NIDX_ESTATE, "the segment has no document columns (nidx_txt_set_doc_columns)");
    if (P.groups && !t->ix->groups.d_off) return fail(NIDX_ESTATE, "the segment has no access groups (nidx_txt_set_doc_groups)");
    if ((P.dates[0] && !t->ix->d_secs[0]) || (P.dates[1] && !t->ix->d_secs[1])) return fail(NIDX_ESTATE, "the segment has no dates (nidx_txt_set_dates)");
    if (!P.ph_query.empty() && !t->ix->d_pos) return fail(NIDX_ESTATE, "the segment has no positions (nidx_txt_set_positions)");
    const uint32_t n_terms = (uint32_t)P.terms.size(), nv = (uint32_t)P.ph_query.size();
    for (PfOp& o : P.prog)
        if (o.op == PF_BITS && (o.arg & 0x80000000u)) o.arg = n_terms + (o.arg & 0x7FFFFFFFu);
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    CU(cudaSetDevice(t->ix->device));
    WsGuard g(t->ix->pool, stream);
    Workspace& w = *g.w;
    const size_t words = ((size_t)t->ix->n_docs + 63) / 64, slots = (size_t)n_terms + nv;
    Stage st(stream, host, host);
    uint64_t* d_out;
    st.out(out_bits, words, &d_out);
    r = st.place(w.stage);
    if (r) return r;
    PrefilterArgs A{};
    A.n_docs = t->ix->n_docs; A.res_ord = t->ix->d_res_ord; A.field_ord = t->ix->d_field_ord; A.fdoc_off = t->ix->facets.d_off; A.ford = t->ix->facets.d_ord;
    A.gdoc_off = t->ix->groups.d_off; A.gord = t->ix->groups.d_ord;
    A.secs0 = t->ix->d_secs[0]; A.secs1 = t->ix->d_secs[1]; A.words = words; A.alive = t->d_alive;
    PhrasePlan pp;
    auto scatter = [&](uint64_t* kw, unsigned char* extra) -> int {   // keyword leaves: terms first, then phrases
        if (n_terms) {
            uint32_t* d_terms = reinterpret_cast<uint32_t*>(extra);
            CU(cudaMemcpyAsync(d_terms, P.terms.data(), (size_t)n_terms * 4, cudaMemcpyHostToDevice, stream));
            prefilter_scatter_kernel<<<n_terms, 256, 0, stream>>>(t->ix->d_post.p, t->ix->d_post.p, n_terms, t->ix->d_term_off, t->ix->n_terms, d_terms, nullptr, nullptr, 0, kw, words);
            LAUNCHED();
        }
        if (nv) {   // the phrases' virtual lists (phrase.cuh), as the keyword search makes them, then scattered like terms
            const int32_t nq = (int32_t)((nv + BM_MAX_TERMS - 1) / BM_MAX_TERMS);
            const std::vector<uint32_t> no_terms(nq + 1, 0);
            const nidx_txt_phrases ph{P.ph_terms.data(), P.ph_off.data(), P.ph_query.data(), (int32_t)nv};
            int r = phrase_plan(t, &ph, nq, no_terms, pp);
            if (r) return r;
            TxtDev T;
            T.n_docs = t->ix->n_docs; T.n_terms = t->ix->n_terms; T.n_fine = t->ix->n_fine; T.term_off = t->ix->d_term_off; T.post = t->ix->d_post;
            T.skip_row = t->ix->d_skip_row; T.skip = t->ix->d_skip; T.alive = t->d_alive;
            Bm25Args a{};
            r = phrase_pass(t, pp, T, w, stream, a);
            if (r) return r;
            prefilter_scatter_kernel<<<nv, 256, 0, stream>>>(a.ph_post, a.ph_post, nv, nullptr, 0, nullptr, a.ph_range, nullptr, n_terms, kw, words);
            LAUNCHED();
        }
        return 0;
    };
    unsigned long long h = 0;
    r = run_program(w, stream, t->ix->sm_count, P.prog, slots, A, (size_t)n_terms * 4, scatter, d_out, &h, t->ix->ev_k0, t->ix->ev_k1);
    if (!r) r = st.finish(true);   // the program and the plans are host temporaries, and the count is read back
    if (r) return r;
    if (out_matching) *out_matching = h;
    return 0;
}

int nidx_vec_prefilter_bits(nidx_vec_segment* s, const uint64_t* doc_bits, uint64_t n_docs, const uint32_t* join, int32_t doc_op,
                            const uint64_t* res_bits, uint64_t n_res, const uint64_t* res_ranges, const nidx_filter_node* nodes, int32_t n_nodes,
                            int32_t op, uint64_t* out_bits, int mem, uint64_t* out_matching, void* stream_) {
    int r = require_handle(s);
    if (r) return r;
    const bool text = doc_bits != nullptr, res = res_bits != nullptr;
    if (!text && !res) return fail(NIDX_EINVAL, "neither a text part nor a resource part");
    if (!text) n_docs = 0;
    if (!res) n_res = 0;
    if ((n_docs && !join) || (n_res && !res_ranges)) return fail(NIDX_EINVAL, "null argument");
    if ((op != NIDX_F_AND && op != NIDX_F_OR) || (text && res && doc_op != NIDX_F_AND && doc_op != NIDX_F_OR))
        return fail(NIDX_EINVAL, "op must be NIDX_F_AND or NIDX_F_OR");
    if (n_nodes < 0 || (n_nodes > 0 && !nodes)) return fail(NIDX_EINVAL, "bad filter formula");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    CU(cudaSetDevice(s->cfg.device));
    WsGuard g(s->pool, stream);
    Workspace& w = *g.w;
    const size_t words = ((size_t)s->n_par + 63) / 64;
    Stage st(stream, host, host);
    const uint64_t *d_doc, *d_res, *d_ranges;
    const uint32_t* d_join;
    uint64_t* d_out;
    st.in(doc_bits, (size_t)((n_docs + 63) / 64), &d_doc);
    st.in(text ? join : nullptr, (size_t)n_docs, &d_join);
    st.in(res_bits, (size_t)((n_res + 63) / 64), &d_res);
    st.in(res ? res_ranges : nullptr, (size_t)(2 * n_res), &d_ranges);
    st.out(out_bits, words, &d_out);
    r = st.place(w.stage);
    if (r) return r;
    // the program: [slot 0: the text documents' paragraphs] [slot rs: the resources' paragraphs] [doc_op when both], combined with
    // the paragraph formula (segment.rs:516-534) under op, as the reference combines its clauses
    const uint32_t rs = text ? 1 : 0;
    FormulaPlan P;
    P.slots = rs + (res ? 1 : 0);
    if (n_nodes) {
        r = P.compile(s, nodes, n_nodes);
        if (r) return r;
    }
    std::vector<PfOp> head;
    if (text) head.push_back(FormulaPlan::leaf(0));
    if (res) head.push_back(FormulaPlan::leaf((int)rs));
    if (text && res) { PfOp b{}; b.op = doc_op == NIDX_F_OR ? PF_OR : PF_AND; head.push_back(b); }
    P.prog.insert(P.prog.begin(), head.begin(), head.end());
    if (n_nodes) { PfOp b{}; b.op = op == NIDX_F_OR ? PF_OR : PF_AND; P.prog.push_back(b); }
    const nidx_vec_segment::InvIndex& ix = s->inv[NIDX_INV_FIELDS];
    auto scatter = [&](uint64_t* bits, unsigned char* extra) -> int {
        if (n_docs && ix.n_keys) {
            const int blocks = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)s->sm_count * 8, (n_docs + 255) / 256));
            prefilter_join_kernel<<<blocks, 256, 0, stream>>>(d_doc, d_join, n_docs, ix.n_keys, ix.d_post_off, ix.d_post, bits);
            LAUNCHED();
        }
        if (n_res && ix.n_keys) {
            const int blocks = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)s->sm_count * 8, (n_res + 255) / 256));
            prefilter_res_join_kernel<<<blocks, 256, 0, stream>>>(d_res, n_res, d_ranges, ix.d_post, bits + (size_t)rs * words);
            LAUNCHED();
        }
        return P.scatter(bits, extra, words, stream);
    };
    unsigned long long h = 0;
    r = run_program(w, stream, s->sm_count, P.prog, P.slots, paragraph_args(s), P.extra_bytes(), scatter, d_out, &h);
    if (!r) r = st.finish(true);   // the program and the ranges are host temporaries, and the count is read back
    if (r) return r;
    if (out_matching) *out_matching = h;
    return 0;
}

// ---- JSON filters: resource bitsets (prefilter.cuh) ------------------------------------------------------------------------------
int nidx_txt_resource_bits(nidx_txt_segment* t, const uint64_t* doc_bits, uint64_t n_resources, uint64_t* out_res_bits, int mem, void* stream_) {
    int r = require_handle(t);
    if (r) return r;
    if (!doc_bits || !out_res_bits) return fail(NIDX_EINVAL, "null argument");
    if (!t->ix->d_res_ord) return fail(NIDX_ESTATE, "the segment has no document columns (nidx_txt_set_doc_columns)");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    CU(cudaSetDevice(t->ix->device));
    WsGuard g(t->ix->pool, stream);
    const size_t n_docs = t->ix->n_docs, rwords = (size_t)(n_resources + 63) / 64;
    Stage st(stream, host, host);
    const uint64_t* d_doc;
    uint64_t* d_out;
    st.in(doc_bits, (n_docs + 63) / 64, &d_doc);
    st.out(out_res_bits, rwords, &d_out);
    r = st.place(g.w->stage);
    if (r) return r;
    if (rwords) CU(cudaMemsetAsync(d_out, 0, rwords * 8, stream));
    if (n_docs && rwords) {
        const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)t->ix->sm_count * 8, (n_docs + 255) / 256));
        prefilter_resource_kernel<<<blocks, 256, 0, stream>>>(d_doc, t->ix->d_res_ord, n_docs, n_resources, d_out);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    return st.finish();
}

int nidx_txt_join_mask(nidx_txt_segment* t, const uint64_t* and_bits, const uint64_t* doc_bits, uint64_t n_doc_bits, const uint32_t* doc_join,
                       const uint64_t* res_bits, uint64_t n_res, const uint32_t* res_join, int32_t op, uint64_t* out_bits, int mem,
                       uint64_t* out_matching, void* stream_) {
    int r = require_handle(t);
    if (r) return r;
    const size_t n = t->ix->n_docs;
    if ((n && !res_join) || (n_res && !res_bits) || (doc_bits && n && !doc_join) || !out_bits) return fail(NIDX_EINVAL, "null argument");
    if (op != NIDX_F_AND && op != NIDX_F_OR) return fail(NIDX_EINVAL, "op must be NIDX_F_AND or NIDX_F_OR");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    CU(cudaSetDevice(t->ix->device));
    WsGuard g(t->ix->pool, stream);
    Workspace& w = *g.w;
    const size_t words = (n + 63) / 64;
    Stage st(stream, host, host);
    const uint64_t *d_and, *d_doc, *d_res;
    const uint32_t *d_djoin, *d_rjoin;
    uint64_t* d_out;
    st.in(and_bits, words, &d_and);
    st.in(doc_bits, (size_t)((n_doc_bits + 63) / 64), &d_doc);
    st.in(doc_bits ? doc_join : nullptr, n, &d_djoin);
    st.in(n_res ? res_bits : nullptr, (size_t)((n_res + 63) / 64), &d_res);
    st.in(res_join, n, &d_rjoin);
    st.out(out_bits, words, &d_out);
    r = st.place(w.stage);
    if (r) return r;
    ENSURE(w.misc, 16);
    unsigned long long* d_count = w.misc.as<unsigned long long>();
    CU(cudaMemsetAsync(d_count, 0, 8, stream));
    if (words) {
        const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)t->ix->sm_count * 8, (2 * words * 32 + PF_THREADS - 1) / PF_THREADS));
        join_mask_kernel<<<blocks, PF_THREADS, 0, stream>>>(n, d_and, d_doc, n_doc_bits, d_djoin, d_res, n_res, d_rjoin, op == NIDX_F_OR,
                                                            reinterpret_cast<uint32_t*>(d_out), 2 * words, d_count);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    unsigned long long h = 0;
    CU(cudaMemcpyAsync(&h, d_count, 8, cudaMemcpyDeviceToHost, stream));
    r = st.finish(true);
    if (r) return r;
    if (out_matching) *out_matching = h;
    return 0;
}

// ---- sharded search (shard.cuh) -------------------------------------------------------------------
struct nidx_shard_comm {
    int rank = 0, world = 1, device = 0;
    nccl_comm_t comm = nullptr;
    std::mutex mu;          // collectives on one communicator must be issued in the same order by every rank: one call at a time
    DevBuf local, gathered, stage;   // this rank's record, every rank's, staged outputs
};

#define NC(expr)                                                                                                   \
    do {                                                                                                           \
        int e__ = (expr);                                                                                          \
        if (e__ != NCCL_SUCCESS) return fail(NIDX_ECUDA, "%s failed: %s", #expr, nccl_api().GetErrorString(e__)); \
    } while (0)

int nidx_shard_unique_id(uint8_t out[128]) {
    if (!out) return fail(NIDX_EINVAL, "null argument");
    NcclApi& N = nccl_api();
    if (!N.ok) return fail(NIDX_ESTATE, "NCCL (libnccl.so.2) is not available in this process");
    nccl_unique_id id;
    NC(N.GetUniqueId(&id));
    memcpy(out, id.internal, 128);
    return 0;
}

int nidx_shard_init(const uint8_t unique_id[128], int32_t rank, int32_t world, int32_t device, nidx_shard_comm** out) {
    if (!unique_id || !out || world <= 0 || rank < 0 || rank >= world) return fail(NIDX_EINVAL, "bad argument");
    int r = check_device(device);
    if (r) return r;
    NcclApi& N = nccl_api();
    if (!N.ok) return fail(NIDX_ESTATE, "NCCL (libnccl.so.2) is not available in this process");
    nidx_shard_comm* c = new nidx_shard_comm();
    c->rank = rank; c->world = world; c->device = device;
    nccl_unique_id id;
    memcpy(id.internal, unique_id, 128);
    int e = N.CommInitRank(&c->comm, world, id, rank);
    if (e != NCCL_SUCCESS) { delete c; return fail(NIDX_ECUDA, "ncclCommInitRank failed: %s", N.GetErrorString(e)); }
    *out = c;
    return 0;
}

void nidx_shard_destroy(nidx_shard_comm* c) {
    if (!c) return;
    cudaSetDevice(c->device);
    cudaDeviceSynchronize();
    if (c->comm) nccl_api().CommDestroy(c->comm);
    delete c;
}

int nidx_vec_set_paragraph_keys(nidx_vec_segment* s, const uint64_t* keys) {
    if (!s) return fail(NIDX_EINVAL, "null segment");
    return set_rows(s->cfg.device, s->d_par_keys, keys, s->n_par);
}

// How the parts of a sharded search are merged (step 3)
enum class PartsRule {
    text,     // documents of one index: (score desc, part asc, position asc), parts_merge_kernel + shard_count_kernel
    kmerge,   // vector shards: merge_vector_responses, kmerge_by(score >=) (kmerge_parts_kernel)
    fssc,     // vector segments of one index: Fssc with the paragraph / vector keys of the records (shard_fssc_kernel)
};

// The device outputs of a merge of parts (the caller's, or staged)
struct MergeOut {
    uint32_t* ids;
    float* scores;
    int* part;
    int* counts;
};
static void stage_merge_outputs(Stage& st, MergeOut& o, int nq, int k, uint32_t* ids, float* scores, int32_t* part, int32_t* counts) {
    st.out(ids, (size_t)nq * k, &o.ids);
    st.out(scores, (size_t)nq * k, &o.scores);
    st.out(part, (size_t)nq * k, &o.part);
    st.out(counts, (size_t)nq, &o.counts);
}

// Step 3: merge n_parts records laid end to end (shard_part_words each) into [nq][k] ids / scores / part + counts
static int shard_merge_impl(const uint32_t* gathered, int n_parts, int nq, int k, PartsRule rule, int with_duplicates, const MergeOut& o,
                            cudaStream_t stream) {
    size_t words = shard_part_words(nq, k, rule == PartsRule::fssc);
    const float* gathered_scores = reinterpret_cast<const float*>(gathered + (size_t)nq * k);
    if (rule == PartsRule::fssc) {
        size_t per = (size_t)k * 16 + (size_t)n_parts * k * 8;
        int threads = (int)std::max<size_t>(1, std::min<size_t>(64, (size_t)(96 * 1024) / per));
        if (per > 96 * 1024) return fail(NIDX_EINVAL, "k = %d is too large for the de-duplicating merge over %d parts", k, n_parts);
        threads = std::min(threads, nq);
        size_t smem = per * threads;
        if (smem > 48 * 1024) CU(cudaFuncSetAttribute(shard_fssc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        shard_fssc_kernel<<<(nq + threads - 1) / threads, threads, smem, stream>>>(gathered, n_parts, words, nq, k, with_duplicates, o.ids, o.scores, o.part,
                                                                                  o.counts);
        LAUNCHED();
    } else if (rule == PartsRule::kmerge) {
        int r = launch_kmerge(gathered, gathered_scores, n_parts, words, nq, k, o.ids, o.scores, o.part, o.counts, stream);
        if (r) return r;
    } else {
        int r = launch_parts_merge(gathered, gathered_scores, n_parts, words, nq, k, o.ids, o.scores, o.part, stream);
        if (r) return r;
        shard_count_kernel<<<(nq + 255) / 256, 256, 0, stream>>>(o.ids, nq, k, o.counts);
        LAUNCHED();
    }
    CU(cudaGetLastError());
    return 0;
}

// The exchange buffers of a sharded search: this rank's record (words long) + nq counts, and every rank's record
static int shard_buffers(nidx_shard_comm* c, int nq, int k, bool fssc, size_t* words) {
    *words = shard_part_words(nq, k, fssc);
    ENSURE(c->local, *words * 4 + (size_t)nq * 4);
    ENSURE(c->gathered, (size_t)c->world * *words * 4 + 64);
    return 0;
}

// Steps 2 and 3: all-gather the local records in rank order, merge them
static int shard_exchange_and_merge(nidx_shard_comm* c, int nq, int k, PartsRule rule, int with_duplicates, const MergeOut& o, cudaStream_t stream) {
    NcclApi& N = nccl_api();
    size_t words = shard_part_words(nq, k, rule == PartsRule::fssc);
    NC(N.AllGather(c->local.p, c->gathered.p, words * 4, NCCL_INT8, c->comm, stream));
    LAUNCHED();
    return shard_merge_impl(c->gathered.as<uint32_t>(), c->world, nq, k, rule, with_duplicates, o, stream);
}

// Step 1: this part's segment searched into its exchange record (queries from the caller's memory, results straight into the
// record), plus the de-duplication keys.  `counts` = nq ints of device scratch, or NULL.
static int shard_record_impl(nidx_vec_segment* seg, const float* queries, int32_t nq, int32_t ldq, bool qhost, const nidx_vec_search_params* p, int32_t rank,
                             bool dedup, uint32_t* record, int32_t* counts, cudaStream_t stream) {
    int k = p->k;
    int r = vec_search_impl(seg, queries, nq, ldq, qhost, false, p, record, reinterpret_cast<float*>(record + (size_t)nq * k), counts, stream);
    if (r) return r;
    if (dedup) {
        int n_res = nq * k;
        shard_keys_kernel<<<(n_res * 32 + 255) / 256, 256, 0, stream>>>(seg->vdev(), record, n_res, seg->d_par_keys, (uint32_t)rank, p->with_duplicates ? 0 : 1,
                                                                       reinterpret_cast<uint64_t*>(record + 2 * (size_t)nq * k),
                                                                       reinterpret_cast<uint64_t*>(record + 4 * (size_t)nq * k));
        LAUNCHED();
        CU(cudaGetLastError());
    }
    return 0;
}

int nidx_vec_shard_record(nidx_vec_segment* seg, const float* queries, int32_t nq, int32_t ldq, int mem, const nidx_vec_search_params* p, int32_t rank,
                          int32_t dedup, uint32_t* out_record, void* stream_) {
    if (!seg || !p || !out_record) return fail(NIDX_EINVAL, "null argument");
    if (nq <= 0) return 0;
    if (p->k <= 0) return fail(NIDX_EINVAL, "k must be positive");
    if (rank < 0) return fail(NIDX_EINVAL, "rank must not be negative");
    CU(cudaSetDevice(seg->cfg.device));
    return shard_record_impl(seg, queries, nq, ldq, mem == NIDX_MEM_HOST, p, rank, dedup != 0, out_record, nullptr, reinterpret_cast<cudaStream_t>(stream_));
}

int nidx_shard_merge(int32_t device, const uint32_t* records, int32_t n_parts, int32_t nq, int32_t k, int32_t dedup, int32_t with_duplicates, int mem,
                     uint32_t* out_ids, float* out_scores, int32_t* out_part, int32_t* out_counts, void* stream_) {
    int r = check_device(device);
    if (r) return r;
    if (!records || !out_ids || !out_scores || n_parts <= 0 || k <= 0) return fail(NIDX_EINVAL, "bad argument");
    if (nq <= 0) return 0;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    WorkspacePool* pool = plan_pool(device);
    if (!pool) return fail(NIDX_EINVAL, "device %d", device);
    WsGuard g(*pool, stream);
    const bool host = mem == NIDX_MEM_HOST;
    Stage st(stream, host, host);
    MergeOut o;
    stage_merge_outputs(st, o, nq, k, out_ids, out_scores, out_part, out_counts);
    r = st.place(g.w->stage);
    if (!r) r = shard_merge_impl(records, n_parts, nq, k, dedup ? PartsRule::fssc : PartsRule::kmerge, with_duplicates, o, stream);
    if (r) return r;
    return st.finish();
}

int nidx_vec_search_sharded(nidx_shard_comm* c, nidx_vec_segment* seg, const float* queries, int32_t nq, int32_t ldq, int mem, const nidx_vec_search_params* p,
                            int32_t dedup, uint32_t* out_ids, float* out_scores, int32_t* out_part, int32_t* out_counts, void* stream_) {
    if (!c || !seg || !p || !out_ids || !out_scores) return fail(NIDX_EINVAL, "null argument");
    if (nq <= 0) return 0;
    if (seg->cfg.device != c->device) return fail(NIDX_EINVAL, "segment on device %d, communicator on device %d", seg->cfg.device, c->device);
    int k = p->k;
    if (k <= 0) return fail(NIDX_EINVAL, "k must be positive");
    CU(cudaSetDevice(c->device));
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    bool host = mem == NIDX_MEM_HOST;
    std::lock_guard<std::mutex> lock(c->mu);
    size_t words;
    int r = shard_buffers(c, nq, k, dedup != 0, &words);
    Stage st(stream, false, host);
    MergeOut o;
    stage_merge_outputs(st, o, nq, k, out_ids, out_scores, out_part, out_counts);
    if (!r) r = st.place(c->stage);
    if (r) return r;
    uint32_t* local = c->local.as<uint32_t>();
    // 1. this rank's segment into the exchange record
    r = shard_record_impl(seg, queries, nq, ldq, host, p, c->rank, dedup != 0, local, reinterpret_cast<int*>(local + words), stream);
    // 2. + 3. exchange and merge
    if (!r) r = shard_exchange_and_merge(c, nq, k, dedup ? PartsRule::fssc : PartsRule::kmerge, p->with_duplicates, o, stream);
    if (r) return r;
    return st.finish();
}

int nidx_txt_search_sharded(nidx_shard_comm* c, nidx_txt_segment* seg, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem,
                            const nidx_txt_search_params* p, uint32_t* out_docs, float* out_scores, int32_t* out_part, int32_t* out_counts, uint64_t* out_total,
                            void* stream_) {
    if (!c || !seg || !p || !out_docs || !out_scores) return fail(NIDX_EINVAL, "null argument");
    if (nq <= 0) return 0;
    if (seg->ix->device != c->device) return fail(NIDX_EINVAL, "segment on device %d, communicator on device %d", seg->ix->device, c->device);
    int k = p->k;
    CU(cudaSetDevice(c->device));
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    bool host = mem == NIDX_MEM_HOST;
    std::lock_guard<std::mutex> lock(c->mu);
    NcclApi& N = nccl_api();
    size_t words;
    int r = shard_buffers(c, nq, k, false, &words);
    Stage st(stream, false, host);
    MergeOut o;
    uint64_t* d_total;
    stage_merge_outputs(st, o, nq, k, out_docs, out_scores, out_part, out_counts);
    st.out(out_total, (size_t)nq, &d_total);
    if (!r) r = st.place(c->stage);
    if (r) return r;
    uint32_t* local = c->local.as<uint32_t>();
    int* local_cnt = reinterpret_cast<int*>(local + words);
    // the min_score cut is applied to the merged list by the caller's convention (reader.rs:302-305 drops below min_score after top-k):
    // every part applies it locally, which commutes with the merge.
    r = txt_search_impl(seg, query_terms, query_off, nq, host, false, p, local, reinterpret_cast<float*>(local + (size_t)nq * k), local_cnt, d_total, stream);
    if (r) return r;
    NC(N.AllReduce(d_total, d_total, (size_t)nq, NCCL_UINT64, NCCL_SUM, c->comm, stream));   // Count collector over all parts
    LAUNCHED();
    r = shard_exchange_and_merge(c, nq, k, PartsRule::text, 1, o, stream);
    if (r) return r;
    return st.finish();
}

// ---- rank fusion + the fused shard search (SURVEY 8f rank 4) --------------------------------------------------------------
int nidx_txt_set_doc_keys(nidx_txt_segment* t, const uint64_t* keys) {
    int r = require_owner(t);
    if (r) return r;
    return set_rows(t->ix->device, t->ix->d_doc_keys, keys, t->ix->n_docs);
}

}  // extern "C"

// sources already on the device; outputs on the device
static int rrf_launch(const RrfSourceDev* src, int n_sources, int nq, double k, uint64_t* out_keys, double* out_scores, uint32_t* out_refs, int32_t* out_counts,
                      cudaStream_t stream) {
    RrfArgs a;
    memset(&a, 0, sizeof(a));
    int cap = 0;
    for (int i = 0; i < n_sources; ++i) { a.src[i] = src[i]; cap += src[i].k; }
    a.n_sources = n_sources; a.nq = nq; a.cap = cap; a.k = k;
    a.out_keys = out_keys; a.out_scores = out_scores; a.out_refs = out_refs; a.out_counts = out_counts;
    size_t smem = rf_smem_bytes(cap);
    if (smem > 200 * 1024) return fail(NIDX_EINVAL, "rank fusion of %d items per query needs %zu bytes of shared memory: too many", cap, smem);
    CU(cudaFuncSetAttribute(rrf_fuse_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    rrf_fuse_kernel<<<nq, RF_THREADS, smem, stream>>>(a);
    LAUNCHED();
    CU(cudaGetLastError());
    return 0;
}

// side streams of the fused shard search: one set per host thread and device (the reference runs the index searches of one request on
// scoped threads, shard_search.rs:215-239; here they are streams forked from, and joined back into, the caller's stream)
struct PlanStreams {
    cudaStream_t s[3] = {nullptr, nullptr, nullptr};
    cudaEvent_t fork = nullptr, join[3] = {nullptr, nullptr, nullptr};
    int device = -1;
    int init(int dev) {
        if (device == dev) return 0;
        if (device >= 0) return fail(NIDX_EINVAL, "a host thread uses nidx_shard_search on one device only (first %d, now %d)", device, dev);
        for (int i = 0; i < 3; ++i) {
            CU(cudaStreamCreateWithFlags(&s[i], cudaStreamNonBlocking));
            CU(cudaEventCreateWithFlags(&join[i], cudaEventDisableTiming));
        }
        CU(cudaEventCreateWithFlags(&fork, cudaEventDisableTiming));
        device = dev;
        return 0;
    }
};
static thread_local PlanStreams g_plan_streams;

extern "C" {

int nidx_rank_fusion_rrf(int32_t device, const nidx_rrf_source* sources, int32_t n_sources, int32_t nq, double k, int mem, uint64_t* out_keys,
                         double* out_scores, uint32_t* out_refs, int32_t* out_counts, void* stream_) {
    int r = check_device(device);
    if (r) return r;
    if (!sources || n_sources <= 0 || n_sources > RF_MAX_SOURCES) return fail(NIDX_EINVAL, "rank fusion takes 1..%d sources", RF_MAX_SOURCES);
    if (!out_keys || !out_scores || !out_refs || !out_counts) return fail(NIDX_EINVAL, "null output");
    if (nq <= 0) return 0;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    bool host = mem == NIDX_MEM_HOST;
    int cap = 0;
    for (int i = 0; i < n_sources; ++i) {
        if (sources[i].k <= 0 || !sources[i].keys || !sources[i].scores) return fail(NIDX_EINVAL, "rank fusion source %d: keys, scores and k > 0 are required", i);
        if (sources[i].k >= (1 << 24)) return fail(NIDX_EINVAL, "rank fusion source %d: k too large", i);
        cap += sources[i].k;
    }
    WorkspacePool* pool = plan_pool(device);
    if (!pool) return fail(NIDX_EINVAL, "device %d", device);
    WsGuard g(*pool, stream);
    Stage st(stream, host, host);
    RrfSourceDev dev[RF_MAX_SOURCES];
    for (int i = 0; i < n_sources; ++i) {
        const size_t nk = (size_t)nq * sources[i].k;
        dev[i] = RrfSourceDev{nullptr, nullptr, nullptr, sources[i].k, sources[i].weight};
        st.in(sources[i].keys, nk, &dev[i].keys);
        st.in(sources[i].scores, nk, &dev[i].scores);
        st.in(sources[i].counts, (size_t)nq, &dev[i].counts);
    }
    uint64_t* d_keys; double* d_sc; uint32_t* d_refs; int32_t* d_cnt;
    st.out(out_keys, (size_t)nq * cap, &d_keys);
    st.out(out_scores, (size_t)nq * cap, &d_sc);
    st.out(out_refs, (size_t)nq * cap, &d_refs);
    st.out(out_counts, (size_t)nq, &d_cnt);
    r = st.place(g.w->stage);
    if (!r) r = rrf_launch(dev, n_sources, nq, k, d_keys, d_sc, d_refs, d_cnt, stream);
    if (r) return r;
    return st.finish();
}

int nidx_shard_search(const nidx_shard_search_request* rq, nidx_shard_search_response* rs, int mem, void* stream_) {
    if (!rq || !rs) return fail(NIDX_EINVAL, "null argument");
    const int nq = rq->nq;
    if (nq <= 0) return 0;
    if (!rq->vec && !rq->par && !rq->doc) return fail(NIDX_EINVAL, "shard search without any index request");
    int device = rq->vec ? rq->vec->cfg.device : (rq->par ? rq->par->ix->device : rq->doc->ix->device);
    if ((rq->vec && rq->vec->cfg.device != device) || (rq->par && rq->par->ix->device != device) || (rq->doc && rq->doc->ix->device != device))
        return fail(NIDX_EINVAL, "the indexes of one shard search must live on one device");
    if (rq->vec && (!rq->vec_params || !rs->vec_ids || !rs->vec_scores || !rs->vec_counts)) return fail(NIDX_EINVAL, "vector request: params and outputs are required");
    if (rq->par && (!rq->par_params || !rs->par_docs || !rs->par_scores || !rs->par_counts)) return fail(NIDX_EINVAL, "paragraph request: params and outputs are required");
    if (rq->doc && (!rq->doc_params || !rs->doc_docs || !rs->doc_scores || !rs->doc_counts)) return fail(NIDX_EINVAL, "document request: params and outputs are required");
    const bool fuse = rq->rrf_k > 0.0 && rq->vec && rq->par;
    if (fuse && (!rs->fused_keys || !rs->fused_scores || !rs->fused_refs || !rs->fused_counts)) return fail(NIDX_EINVAL, "rank fusion: outputs are required");
    int r = check_device(device);
    if (r) return r;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    PlanStreams& ps = g_plan_streams;
    r = ps.init(device);
    if (r) return r;
    const int kv = rq->vec ? rq->vec_params->k : 0, kp = rq->par ? rq->par_params->k : 0, kd = rq->doc ? rq->doc_params->k : 0;
    if ((rq->vec && kv <= 0) || (rq->par && kp <= 0) || (rq->doc && kd <= 0)) return fail(NIDX_EINVAL, "k must be positive");
    WorkspacePool* pool = plan_pool(device);
    WsGuard g(*pool, stream);
    // device-side results (the callers' buffers, or staged when they are host buffers) + fusion scratch
    const size_t nv = (size_t)nq * kv, np = (size_t)nq * kp, nd = (size_t)nq * kd, nf = (size_t)nq * (kv + kp);
    Stage st(stream, host, host);
    uint32_t *d_vid, *d_pdoc, *d_ddoc, *d_frf;
    float *d_vsc, *d_psc, *d_dsc;
    int32_t *d_vcnt, *d_pcnt, *d_dcnt, *d_fcnt;
    uint64_t *d_ptot, *d_dtot, *d_fkey, *d_vkey = nullptr, *d_pkey = nullptr;
    double* d_fsc;
    if (rq->vec) { st.out(rs->vec_ids, nv, &d_vid); st.out(rs->vec_scores, nv, &d_vsc); st.out(rs->vec_counts, (size_t)nq, &d_vcnt); }
    if (rq->par) {
        st.out(rs->par_docs, np, &d_pdoc); st.out(rs->par_scores, np, &d_psc); st.out(rs->par_counts, (size_t)nq, &d_pcnt);
        st.out(rs->par_total, (size_t)nq, &d_ptot);
    }
    if (rq->doc) {
        st.out(rs->doc_docs, nd, &d_ddoc); st.out(rs->doc_scores, nd, &d_dsc); st.out(rs->doc_counts, (size_t)nq, &d_dcnt);
        st.out(rs->doc_total, (size_t)nq, &d_dtot);
    }
    if (fuse) {
        st.out(rs->fused_keys, nf, &d_fkey); st.out(rs->fused_scores, nf, &d_fsc); st.out(rs->fused_refs, nf, &d_frf);
        st.out(rs->fused_counts, (size_t)nq, &d_fcnt);
        st.out((uint64_t*)nullptr, nv, &d_vkey);   // scratch: the keys of the two fused lists
        st.out((uint64_t*)nullptr, np, &d_pkey);
    }
    r = st.place(g.w->stage);
    if (r) return r;

    // fork: the three index searches run on their own streams, each ordered after whatever the caller enqueued before this call
    CU(cudaEventRecord(ps.fork, stream));
    for (int i = 0; i < 3; ++i) CU(cudaStreamWaitEvent(ps.s[i], ps.fork, 0));
    // (text searches first: with host queries they enqueue without waiting; the vector search may wait for a filter count)
    for (int i : {1, 2, 0}) {
        if (i == 1 && rq->par)
            r = txt_search_impl(rq->par, rq->par_terms, rq->par_off, nq, host, false, rq->par_params, d_pdoc, d_psc, d_pcnt, d_ptot, ps.s[1]);
        else if (i == 2 && rq->doc)
            r = txt_search_impl(rq->doc, rq->doc_terms, rq->doc_off, nq, host, false, rq->doc_params, d_ddoc, d_dsc, d_dcnt, d_dtot, ps.s[2]);
        else if (i == 0 && rq->vec)
            r = vec_search_impl(rq->vec, rq->queries, nq, rq->ldq, host, false, rq->vec_params, d_vid, d_vsc, d_vcnt, ps.s[0], rq->formula, rq->n_formula);
        else continue;
        if (r) return r;
        CU(cudaEventRecord(ps.join[i], ps.s[i]));
        CU(cudaStreamWaitEvent(stream, ps.join[i], 0));
    }
    // join + rank fusion of the paragraph (keyword) and vector (semantic) results on the caller's stream
    if (fuse) {
        ids_to_keys_kernel<<<std::min<size_t>((nv + 255) / 256, 1024), 256, 0, stream>>>(d_vid, nv, rq->vec->d_par_of, rq->vec->d_par_keys, d_vkey);
        LAUNCHED();
        ids_to_keys_kernel<<<std::min<size_t>((np + 255) / 256, 1024), 256, 0, stream>>>(d_pdoc, np, nullptr, rq->par->ix->d_doc_keys, d_pkey);
        LAUNCHED();
        RrfSourceDev src[2];
        RrfSourceDev kw{d_pkey, d_psc, d_pcnt, kp, rq->weight_keyword}, sem{d_vkey, d_vsc, d_vcnt, kv, rq->weight_semantic};
        src[0] = rq->semantic_first ? sem : kw;
        src[1] = rq->semantic_first ? kw : sem;
        r = rrf_launch(src, 2, nq, rq->rrf_k, d_fkey, d_fsc, d_frf, d_fcnt, stream);
        if (r) return r;
    }
    return st.finish();
}

}  // extern "C"

// ---- graph search (graph.cuh) ---------------------------------------------------------------------------------------------------
struct nidx_graph {
    nidx_txt_segment* seg = nullptr;   // borrowed: alive bits, facets
    bool ready = false;
    DevArray<uint32_t> d_col[GF_COLS], d_tok_off[2], d_tok[2], d_value_cp, d_token_cp;
    DevArray<uint64_t> d_value_off, d_token_off;
    uint32_t n_values = 0, n_tokens = 0, n_node_keys = 0, n_rel_keys = 0;
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};   // call start, dictionary pass, scored pass, collection
    ~nidx_graph() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
};

// An expression (pre-order nidx_graph_node) as graph_eval_kernel runs it: post-order, with the deepest stack it reaches.
struct GraphPlan {
    std::vector<PfOp> prog;
    std::vector<uint32_t> ords;        // TOKSET lists
    bool val_bits = false, tok_bits = false;
    uint32_t level = 0, depth = 0;

    void push(const PfOp& o, int pops) { prog.push_back(o); level = level - pops + 1; depth = std::max(depth, level); }
    int compile(const nidx_graph_node* nodes, int n_nodes, int& i, int lvl, uint32_t n_terms, const std::vector<int>& term_dict) {
        if (i >= n_nodes) return fail(NIDX_EINVAL, "malformed graph expression (operand counts do not add up to %d nodes)", n_nodes);
        if (lvl > NIDX_PREFILTER_MAX_DEPTH) return fail(NIDX_EINVAL, "the graph expression nests deeper than %d levels", NIDX_PREFILTER_MAX_DEPTH);
        const nidx_graph_node& nd = nodes[i++];
        const int at = i - 1;
        PfOp o{};
        o.lo = nd.lo; o.hi = nd.hi; o.w = nd.w;
        // the per-key max (atomicMax on the bits) and the top-k keys (score bits << 32) order scores as unsigned integers: only
        // finite scores >= 0 (and -0, which is +0 there) keep their order
        if (!(nd.w >= 0.f) || !std::isfinite(nd.w)) return fail(NIDX_EINVAL, "graph node %d: the score must be finite and >= 0", at);
        if (nd.w == 0.f) o.w = 0.f;
        switch (nd.kind) {
            case NIDX_G_EQ:
                if (nd.arg < 0 || nd.arg >= GF_COLS) return fail(NIDX_EINVAL, "graph node %d: bad column", at);
                o.op = GF_EQ; o.arg = (uint32_t)nd.arg; break;
            case NIDX_G_COLBITS:
                if (nd.arg != NIDX_G_SRC_VALUE && nd.arg != NIDX_G_DST_VALUE) return fail(NIDX_EINVAL, "graph node %d: automaton leaves read a value column", at);
                if (nd.lo < 0 || nd.lo >= n_terms || term_dict[nd.lo] != NIDX_G_TERMS_VALUES) return fail(NIDX_EINVAL, "graph node %d: bad values term", at);
                o.op = GF_COLBITS; o.arg = (uint32_t)nd.arg; val_bits = true; break;
            case NIDX_G_TOKBITS:
                if (nd.arg != 0 && nd.arg != 1) return fail(NIDX_EINVAL, "graph node %d: bad side", at);
                if (nd.lo < 0 || nd.lo >= n_terms || term_dict[nd.lo] != NIDX_G_TERMS_TOKENS) return fail(NIDX_EINVAL, "graph node %d: bad tokens term", at);
                o.op = GF_TOKBITS; o.arg = (uint32_t)nd.arg; tok_bits = true; break;
            case NIDX_G_TOKSET:
                if ((nd.arg != 0 && nd.arg != 1) || nd.n < 0 || (nd.n && !nd.ords)) return fail(NIDX_EINVAL, "graph node %d: bad token set", at);
                o.op = GF_TOKSET; o.arg = (uint32_t)nd.arg; o.lo = (int64_t)ords.size();
                ords.insert(ords.end(), nd.ords, nd.ords + nd.n);
                o.hi = (int64_t)ords.size();
                break;
            case NIDX_G_FACET: o.op = GF_FACET; break;
            case NIDX_G_CONST: o.op = GF_CONST; o.arg = nd.lo ? 1u : 0u; break;
            case NIDX_G_AND: case NIDX_G_OR: {
                if (nd.n < 1) return fail(NIDX_EINVAL, "graph node %d: AND / OR take at least one operand", at);
                for (int c = 0; c < nd.n; ++c) {
                    int r = compile(nodes, n_nodes, i, lvl + 1, n_terms, term_dict);
                    if (r) return r;
                    if (c) { PfOp b{}; b.op = nd.kind == NIDX_G_AND ? GF_AND : GF_OR; push(b, 2); }
                }
                return 0;
            }
            case NIDX_G_NOT: case NIDX_G_CONST_SCORE: {
                if (nd.n != 1) return fail(NIDX_EINVAL, "graph node %d: NOT / CONST_SCORE take one operand", at);
                int r = compile(nodes, n_nodes, i, lvl + 1, n_terms, term_dict);
                if (r) return r;
                o.op = nd.kind == NIDX_G_NOT ? GF_NOT : GF_CONST_SCORE;
                push(o, 1);
                return 0;
            }
            default: return fail(NIDX_EINVAL, "graph node %d: bad kind %d", at, nd.kind);
        }
        push(o, 0);
        return 0;
    }
};

extern "C" {

int nidx_graph_create(nidx_txt_segment* seg, nidx_graph** out) {
    int r = require_handle(seg);
    if (r) return r;
    if (!out) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(seg->ix->device));
    std::unique_ptr<nidx_graph> g(new nidx_graph());
    g->seg = seg;
    for (cudaEvent_t& e : g->ev) CU(cudaEventCreate(&e));
    *out = g.release();
    return 0;
}

void nidx_graph_close(nidx_graph* g) {
    if (!g) return;
    cudaSetDevice(g->seg->ix->device);
    cudaDeviceSynchronize();
    delete g;
}

int nidx_graph_set_columns(nidx_graph* g, const nidx_graph_columns* c) {
    int r = require_handle(g);
    if (r) return r;
    if (!c) return fail(NIDX_EINVAL, "null argument");
    const uint32_t n = g->seg->ix->n_docs;
    if (n && std::any_of(c->col, c->col + GF_COLS, [](const uint32_t* p) { return !p; })) return fail(NIDX_EINVAL, "null column");
    if (!c->tok_off[0] || !c->tok_off[1] || !c->value_off || !c->token_off) return fail(NIDX_EINVAL, "null argument");
    if ((c->value_off[c->n_values] && !c->value_cp) || (c->token_off[c->n_tokens] && !c->token_cp)) return fail(NIDX_EINVAL, "null dictionary");
    const uint32_t limit[GF_COLS] = {c->n_values, c->n_values, 4, 4, NIDX_NIL, NIDX_NIL, 6, NIDX_NIL, c->n_node_keys, c->n_node_keys, c->n_rel_keys};
    for (int k = 0; k < GF_COLS; ++k)
        for (uint32_t d = 0; d < n; ++d)
            if (c->col[k][d] >= limit[k]) return fail(NIDX_EINVAL, "column %d, document %u: ord out of range", k, d);
    for (int s = 0; s < 2; ++s) {
        if (c->tok_off[s][n] >= (1ull << 32)) return fail(NIDX_EINVAL, "at most 2^32-1 tokens per side");
        if (c->tok_off[s][n] && !c->tok_ord[s]) return fail(NIDX_EINVAL, "null token ords");
        for (uint32_t d = 0; d < n; ++d) {
            if (c->tok_off[s][d + 1] < c->tok_off[s][d]) return fail(NIDX_EINVAL, "tok_off must be non-decreasing");
            for (uint64_t j = c->tok_off[s][d]; j < c->tok_off[s][d + 1]; ++j)
                if (c->tok_ord[s][j] >= c->n_tokens) return fail(NIDX_EINVAL, "document %u: token ord out of range", d);
        }
    }
    CU(cudaSetDevice(g->seg->ix->device));
    DevArray<uint32_t> col[GF_COLS], tok_off[2], tok[2], value_cp, token_cp;
    DevArray<uint64_t> value_off, token_off;
    for (int k = 0; k < GF_COLS; ++k) {
        ALLOC(col[k], std::max<size_t>(n, 1) * 4);
        if (n) CU(cudaMemcpy(col[k], c->col[k], (size_t)n * 4, cudaMemcpyHostToDevice));
    }
    for (int s = 0; s < 2; ++s) {
        const uint64_t nnz = c->tok_off[s][n];
        std::vector<uint32_t> off(n + 1);
        for (uint32_t d = 0; d <= n; ++d) off[d] = (uint32_t)c->tok_off[s][d];
        ALLOC(tok_off[s], ((size_t)n + 1) * 4);
        ALLOC(tok[s], std::max<uint64_t>(nnz, 1) * 4);
        CU(cudaMemcpy(tok_off[s], off.data(), off.size() * 4, cudaMemcpyHostToDevice));
        if (nnz) CU(cudaMemcpy(tok[s], c->tok_ord[s], nnz * 4, cudaMemcpyHostToDevice));
    }
    auto dict = [&](uint32_t nd, const uint32_t* cp, const uint64_t* off, DevArray<uint32_t>& dcp, DevArray<uint64_t>& doff) -> int {
        for (uint32_t e = 0; e < nd; ++e)
            if (off[e + 1] < off[e]) return fail(NIDX_EINVAL, "dictionary offsets must be non-decreasing");
        ALLOC(dcp, std::max<uint64_t>(off[nd], 1) * 4);
        ALLOC(doff, ((size_t)nd + 1) * 8);
        if (off[nd]) CU(cudaMemcpy(dcp, cp, off[nd] * 4, cudaMemcpyHostToDevice));
        CU(cudaMemcpy(doff, off, ((size_t)nd + 1) * 8, cudaMemcpyHostToDevice));
        return 0;
    };
    r = dict(c->n_values, c->value_cp, c->value_off, value_cp, value_off);
    if (!r) r = dict(c->n_tokens, c->token_cp, c->token_off, token_cp, token_off);
    if (r) return r;
    for (int k = 0; k < GF_COLS; ++k) g->d_col[k] = std::move(col[k]);   // only now: a failed call leaves the previous columns
    for (int s = 0; s < 2; ++s) { g->d_tok_off[s] = std::move(tok_off[s]); g->d_tok[s] = std::move(tok[s]); }
    g->d_value_cp = std::move(value_cp); g->d_value_off = std::move(value_off);
    g->d_token_cp = std::move(token_cp); g->d_token_off = std::move(token_off);
    g->n_values = c->n_values; g->n_tokens = c->n_tokens; g->n_node_keys = c->n_node_keys; g->n_rel_keys = c->n_rel_keys;
    g->ready = true;
    return 0;
}

int nidx_graph_search(nidx_graph* g, const nidx_graph_node* nodes, int32_t n_nodes, const nidx_graph_term* terms, int32_t n_terms, int32_t kind,
                      int32_t k, const uint64_t* mask, int mem, uint32_t* out_ids, float* out_scores, int32_t* out_count, void* stream_) {
    int r = require_handle(g);
    if (r) return r;
    if (!nodes || n_nodes <= 0 || !out_ids || !out_scores || !out_count) return fail(NIDX_EINVAL, "null argument");
    if (kind != NIDX_G_PATH && kind != NIDX_G_NODES && kind != NIDX_G_RELATIONS) return fail(NIDX_EINVAL, "bad kind %d", kind);
    if (k < 1 || k > NIDX_G_MAX_K) return fail(NIDX_EINVAL, "k must be in 1..%d", NIDX_G_MAX_K);
    if (n_terms < 0 || n_terms > GF_MAX_TERMS || (n_terms && !terms)) return fail(NIDX_EINVAL, "at most %d automaton terms", GF_MAX_TERMS);
    if (!g->ready) return fail(NIDX_ESTATE, "the graph has no columns (nidx_graph_set_columns)");
    TxtIndex* ix = g->seg->ix;
    // the automaton terms, grouped by dictionary: each dictionary's bitsets are [its terms][words]
    std::vector<int> term_dict(n_terms);
    std::vector<uint32_t> slot(n_terms), term_cp;
    std::vector<GraphTerm> dterms[2];
    for (int t = 0; t < n_terms; ++t) {
        const nidx_graph_term& T = terms[t];
        if (T.dict != NIDX_G_TERMS_VALUES && T.dict != NIDX_G_TERMS_TOKENS) return fail(NIDX_EINVAL, "term %d: bad dictionary", t);
        if (T.distance < 0 || T.distance > GF_MAX_DIST) return fail(NIDX_EINVAL, "term %d: the distance must be in 0..%d", t, GF_MAX_DIST);
        if (T.n_cp < 0 || (T.n_cp && !T.cp)) return fail(NIDX_EINVAL, "term %d: bad code points", t);
        term_dict[t] = T.dict;
        slot[t] = (uint32_t)dterms[T.dict].size();
        dterms[T.dict].push_back(GraphTerm{(uint32_t)term_cp.size(), (uint32_t)T.n_cp, (uint32_t)T.distance, T.prefix ? 1u : 0u});
        term_cp.insert(term_cp.end(), T.cp, T.cp + T.n_cp);
        if (term_cp.size() > (size_t)GF_MAX_TERM_CPS) return fail(NIDX_EINVAL, "the automaton terms have more than %d code points", GF_MAX_TERM_CPS);
    }
    GraphPlan P[2];
    const int n_prog = kind == NIDX_G_NODES ? 2 : 1;
    int at = 0;
    for (int p = 0; p < n_prog; ++p) {
        r = P[p].compile(nodes, n_nodes, at, 1, (uint32_t)n_terms, term_dict);
        if (r) return r;
        if (P[p].prog.size() > (size_t)PF_MAX_PROGRAM) return fail(NIDX_EINVAL, "the graph program has more than %d instructions", PF_MAX_PROGRAM);
        for (PfOp& o : P[p].prog)   // automaton leaves name their dictionary's bitset
            if (o.op == GF_COLBITS || o.op == GF_TOKBITS) o.lo = slot[o.lo];
    }
    if (at != n_nodes) return fail(NIDX_EINVAL, "malformed graph expression (operand counts do not add up to %d nodes)", n_nodes);
    for (int p = 0; p < n_prog; ++p)
        for (const PfOp& o : P[p].prog)
            if (o.op == GF_FACET && !ix->facets.d_off) return fail(NIDX_ESTATE, "the segment has no facets (nidx_txt_set_facets)");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    CU(cudaSetDevice(ix->device));
    WsGuard wg(ix->pool, stream);
    Workspace& w = *wg.w;
    const uint32_t n = ix->n_docs;
    const size_t words = ((size_t)n + 63) / 64;
    Stage st(stream, host, host);
    const uint64_t* d_mask;
    uint32_t* d_ids; float* d_sc; int32_t* d_cnt;
    st.in(mask, words, &d_mask);
    st.out(out_ids, (size_t)k, &d_ids);
    st.out(out_scores, (size_t)k, &d_sc);
    st.out(out_count, 1, &d_cnt);
    r = st.place(w.stage);
    if (r) return r;
    CU(cudaEventRecord(g->ev[0], stream));
    // scratch (w.prefilter): [values bitsets][token bitsets][term code points][terms][TOKSET ords][programs]
    const size_t vw = ((size_t)g->n_values + 63) / 64, tw = ((size_t)g->n_tokens + 63) / 64;
    const size_t nv = dterms[0].size(), nt = dterms[1].size();
    auto al = [](size_t b) { return (b + 15) & ~(size_t)15; };
    const size_t o_tb = al(nv * vw * 8), o_cp = o_tb + al(nt * tw * 8), o_terms = o_cp + al(term_cp.size() * 4),
                 o_ords = o_terms + al((nv + nt) * sizeof(GraphTerm)), o_prog0 = o_ords + al((P[0].ords.size() + P[1].ords.size()) * 4),
                 o_prog1 = o_prog0 + al(P[0].prog.size() * sizeof(PfOp)), o_end = o_prog1 + al(P[1].prog.size() * sizeof(PfOp));
    ENSURE(w.prefilter, o_end + 16);
    unsigned char* base = w.prefilter.p;
    uint64_t* val_bits = reinterpret_cast<uint64_t*>(base);
    uint64_t* tok_bits = reinterpret_cast<uint64_t*>(base + o_tb);
    uint32_t* d_term_cp = reinterpret_cast<uint32_t*>(base + o_cp);
    GraphTerm* d_terms = reinterpret_cast<GraphTerm*>(base + o_terms);
    uint32_t* d_ords = reinterpret_cast<uint32_t*>(base + o_ords);
    // the host temporaries are staged in one pinned-free copy each; the call synchronises before they go
    std::vector<GraphTerm> all_terms(dterms[0]);
    all_terms.insert(all_terms.end(), dterms[1].begin(), dterms[1].end());
    std::vector<uint32_t> all_ords(P[0].ords);
    for (PfOp& o : P[1].prog)
        if (o.op == GF_TOKSET) { o.lo += (int64_t)P[0].ords.size(); o.hi += (int64_t)P[0].ords.size(); }
    all_ords.insert(all_ords.end(), P[1].ords.begin(), P[1].ords.end());
    if (!term_cp.empty()) CU(cudaMemcpyAsync(d_term_cp, term_cp.data(), term_cp.size() * 4, cudaMemcpyHostToDevice, stream));
    if (!all_terms.empty()) CU(cudaMemcpyAsync(d_terms, all_terms.data(), all_terms.size() * sizeof(GraphTerm), cudaMemcpyHostToDevice, stream));
    if (!all_ords.empty()) CU(cudaMemcpyAsync(d_ords, all_ords.data(), all_ords.size() * 4, cudaMemcpyHostToDevice, stream));
    for (int p = 0; p < n_prog; ++p)
        CU(cudaMemcpyAsync(base + (p ? o_prog1 : o_prog0), P[p].prog.data(), P[p].prog.size() * sizeof(PfOp), cudaMemcpyHostToDevice, stream));
    const size_t cp_smem = term_cp.size() * 4;
    const int dict_threads = GF_THREADS;
    for (int dct = 0; dct < 2; ++dct) {
        const size_t nterm = dct ? nt : nv, dw = dct ? tw : vw;
        const uint32_t nd = dct ? g->n_tokens : g->n_values;
        if (!nterm || !dw) continue;
        uint64_t* outb = dct ? tok_bits : val_bits;
        CU(cudaMemsetAsync(outb, 0, nterm * dw * 8, stream));
        const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)ix->sm_count * 8, (nd + dict_threads - 1) / dict_threads));
        graph_dict_match_kernel<<<blocks, dict_threads, cp_smem, stream>>>(dct ? g->d_token_cp : g->d_value_cp, dct ? g->d_token_off : g->d_value_off, nd,
                                                                           d_terms + (dct ? nv : 0), (uint32_t)nterm, d_term_cp, (uint32_t)term_cp.size(), outb, dw);
        LAUNCHED();
    }
    CU(cudaEventRecord(g->ev[1], stream));
    // scores and bits per program, then the per-key max (NODES / RELATIONS)
    const uint32_t n_keys = kind == NIDX_G_PATH ? n : (kind == NIDX_G_NODES ? g->n_node_keys : g->n_rel_keys);
    ENSURE(w.scores, (size_t)std::max<uint32_t>(n, 1) * 4 + 2 * std::max<size_t>(words, 1) * 8 + (size_t)std::max<uint32_t>(n_keys, 1) * 4);
    float* d_score = w.scores.as<float>();
    uint32_t* d_bits = reinterpret_cast<uint32_t*>(w.scores.p + (size_t)std::max<uint32_t>(n, 1) * 4);
    uint32_t* d_kmax = reinterpret_cast<uint32_t*>(w.scores.p + (size_t)std::max<uint32_t>(n, 1) * 4 + 2 * std::max<size_t>(words, 1) * 8);
    if (kind != NIDX_G_PATH && n_keys) CU(cudaMemsetAsync(d_kmax, 0, (size_t)n_keys * 4, stream));
    GraphEvalArgs A{};
    A.G.n_docs = n;
    for (int c = 0; c < GF_COLS; ++c) A.G.col[c] = g->d_col[c];
    for (int s = 0; s < 2; ++s) { A.G.tok_off[s] = g->d_tok_off[s]; A.G.tok[s] = g->d_tok[s]; }
    A.G.fdoc_off = ix->facets.d_off; A.G.ford = ix->facets.d_ord;
    A.alive = g->seg->d_alive; A.mask = d_mask; A.val_bits = val_bits; A.tok_bits = tok_bits; A.val_words = vw; A.tok_words = tw; A.ords = d_ords;
    A.score = d_score; A.bits = d_bits;
    const int eval_blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)ix->sm_count * 8, (2 * words * 32 + GF_THREADS - 1) / GF_THREADS));
    const int uniq_blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)ix->sm_count * 8, ((size_t)n + 255) / 256));
    const uint32_t key_col[3] = {0, NIDX_G_SRC_NODE, NIDX_G_REL_KEY};
    for (int p = 0; p < n_prog; ++p) {
        if (!words) break;
        A.prog = reinterpret_cast<const PfOp*>(base + (p ? o_prog1 : o_prog0));
        A.n_prog = (uint32_t)P[p].prog.size();
        A.depth = P[p].depth;
        const size_t smem = P[p].prog.size() * sizeof(PfOp) + (size_t)P[p].depth * GF_THREADS * 4;
        CU(cudaFuncSetAttribute(graph_eval_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        graph_eval_kernel<<<eval_blocks, GF_THREADS, smem, stream>>>(A);
        LAUNCHED();
        if (kind != NIDX_G_PATH) {
            graph_unique_kernel<<<uniq_blocks, 256, 0, stream>>>(n, d_bits, d_score, g->d_col[p ? NIDX_G_DST_NODE : key_col[kind]], d_kmax);
            LAUNCHED();
        }
    }
    CU(cudaEventRecord(g->ev[2], stream));
    // the best k: per CTA, then one merge
    const int cap = topk_cap(k, GF_THREADS);
    const int tk_blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)ix->sm_count * 2, ((size_t)n_keys + GF_THREADS * 16 - 1) / (GF_THREADS * 16)));
    ENSURE(w.partial, (size_t)tk_blocks * k * 8);
    CU(cudaFuncSetAttribute(graph_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap * 8));
    CU(cudaFuncSetAttribute(graph_topk_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap * 8));
    if (n_keys && words) {
        graph_topk_kernel<<<tk_blocks, GF_THREADS, (size_t)cap * 8, stream>>>(n_keys, d_bits, d_score, kind == NIDX_G_PATH ? nullptr : d_kmax, k, cap,
                                                                             w.partial.as<uint64_t>());
        LAUNCHED();
    } else {
        CU(cudaMemsetAsync(w.partial, 0, (size_t)tk_blocks * k * 8, stream));
    }
    graph_topk_merge_kernel<<<1, GF_THREADS, (size_t)cap * 8, stream>>>(w.partial.as<uint64_t>(), tk_blocks * k, k, cap, d_ids, d_sc, d_cnt);
    LAUNCHED();
    CU(cudaEventRecord(g->ev[3], stream));
    CU(cudaGetLastError());
    return st.finish(true);   // the programs, terms and lists are host temporaries
}

int nidx_graph_last_times(nidx_graph* g, float* ms4) {
    int r = require_handle(g);
    if (r) return r;
    if (!ms4) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(g->seg->ix->device));
    CU(cudaEventSynchronize(g->ev[3]));
    CU(cudaEventElapsedTime(ms4 + 0, g->ev[0], g->ev[1]));
    CU(cudaEventElapsedTime(ms4 + 1, g->ev[1], g->ev[2]));
    CU(cudaEventElapsedTime(ms4 + 2, g->ev[2], g->ev[3]));
    CU(cudaEventElapsedTime(ms4 + 3, g->ev[0], g->ev[3]));
    return 0;
}

}  // extern "C"

// ---- suggest (suggest.cuh) -------------------------------------------------------------------------------------------------------
struct nidx_suggest_dict {
    int device = 0, sm_count = 0;
    uint32_t n_terms = 0;
    DevArray<uint32_t> d_cp;
    DevArray<uint64_t> d_off;
    cudaEvent_t ev[2] = {nullptr, nullptr};   // around the last dictionary pass
    WorkspacePool pool;
    ~nidx_suggest_dict() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
};

extern "C" {

int nidx_suggest_dict_create(int32_t device, uint32_t n_terms, const uint32_t* cp, const uint64_t* off, nidx_suggest_dict** out) {
    if (!off || !out || (off[n_terms] && !cp)) return fail(NIDX_EINVAL, "null argument");
    int r = check_device(device);
    if (r) return r;
    for (uint32_t e = 0; e < n_terms; ++e)
        if (off[e + 1] < off[e]) return fail(NIDX_EINVAL, "dictionary offsets must be non-decreasing");
    CU(cudaSetDevice(device));
    std::unique_ptr<nidx_suggest_dict> d(new nidx_suggest_dict());
    d->device = device;
    d->n_terms = n_terms;
    cudaDeviceProp prop;
    CU(cudaGetDeviceProperties(&prop, device));
    d->sm_count = prop.multiProcessorCount;
    ALLOC(d->d_cp, std::max<uint64_t>(off[n_terms], 1) * 4);
    ALLOC(d->d_off, ((size_t)n_terms + 1) * 8);
    if (off[n_terms]) CU(cudaMemcpy(d->d_cp, cp, off[n_terms] * 4, cudaMemcpyHostToDevice));
    CU(cudaMemcpy(d->d_off, off, ((size_t)n_terms + 1) * 8, cudaMemcpyHostToDevice));
    for (cudaEvent_t& e : d->ev) CU(cudaEventCreate(&e));
    *out = d.release();
    return 0;
}

void nidx_suggest_dict_close(nidx_suggest_dict* d) {
    if (!d) return;
    cudaSetDevice(d->device);
    cudaDeviceSynchronize();
    delete d;
}

int nidx_suggest_expand(nidx_suggest_dict* d, const nidx_graph_term* terms, int32_t n, uint64_t* out_bits, uint64_t* out_counts, void* stream_) {
    int r = require_handle(d);
    if (r) return r;
    if (n < 0 || n > GF_MAX_TERMS || (n && (!terms || !out_bits))) return fail(NIDX_EINVAL, "at most %d automaton terms", GF_MAX_TERMS);
    std::vector<GraphTerm> h_terms;
    std::vector<uint32_t> term_cp;
    for (int t = 0; t < n; ++t) {
        const nidx_graph_term& T = terms[t];
        if (T.distance < 0 || T.distance > GF_MAX_DIST) return fail(NIDX_EINVAL, "term %d: the distance must be in 0..%d", t, GF_MAX_DIST);
        if (T.n_cp < 0 || (T.n_cp && !T.cp)) return fail(NIDX_EINVAL, "term %d: bad code points", t);
        h_terms.push_back(GraphTerm{(uint32_t)term_cp.size(), (uint32_t)T.n_cp, (uint32_t)T.distance, T.prefix ? 1u : 0u});
        term_cp.insert(term_cp.end(), T.cp, T.cp + T.n_cp);
        if (term_cp.size() > (size_t)GF_MAX_TERM_CPS) return fail(NIDX_EINVAL, "the automaton terms have more than %d code points", GF_MAX_TERM_CPS);
    }
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    CU(cudaSetDevice(d->device));
    WsGuard g(d->pool, stream);
    Workspace& w = *g.w;
    const size_t words = ((size_t)d->n_terms + 63) / 64;
    const size_t o_terms = (term_cp.size() * 4 + 15) & ~(size_t)15, o_counts = o_terms + ((h_terms.size() * sizeof(GraphTerm) + 15) & ~(size_t)15);
    ENSURE(w.prefilter, o_counts + std::max<size_t>(n, 1) * 8);
    uint32_t* d_cp = w.prefilter.as<uint32_t>();
    GraphTerm* d_terms = reinterpret_cast<GraphTerm*>(w.prefilter.p + o_terms);
    unsigned long long* d_counts = reinterpret_cast<unsigned long long*>(w.prefilter.p + o_counts);
    CU(cudaEventRecord(d->ev[0], stream));
    if (n && words) {
        if (!term_cp.empty()) CU(cudaMemcpyAsync(d_cp, term_cp.data(), term_cp.size() * 4, cudaMemcpyHostToDevice, stream));
        CU(cudaMemcpyAsync(d_terms, h_terms.data(), h_terms.size() * sizeof(GraphTerm), cudaMemcpyHostToDevice, stream));
        CU(cudaMemsetAsync(out_bits, 0, (size_t)n * words * 8, stream));
        const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)d->sm_count * 8, ((size_t)d->n_terms + GF_THREADS - 1) / GF_THREADS));
        graph_dict_match_kernel<<<blocks, GF_THREADS, term_cp.size() * 4, stream>>>(d->d_cp, d->d_off, d->n_terms, d_terms, (uint32_t)n, d_cp,
                                                                                   (uint32_t)term_cp.size(), out_bits, words);
        LAUNCHED();
    }
    CU(cudaEventRecord(d->ev[1], stream));
    if (out_counts && n) {
        CU(cudaMemsetAsync(d_counts, 0, (size_t)n * 8, stream));
        if (words) {
            suggest_popc_kernel<<<(unsigned)std::max<size_t>(1, std::min<size_t>((size_t)d->sm_count * 4, (n * words + 255) / 256)), 256, 0, stream>>>(
                out_bits, words, (uint32_t)n, d_counts);
            LAUNCHED();
        }
        CU(cudaMemcpyAsync(out_counts, d_counts, (size_t)n * 8, cudaMemcpyDeviceToHost, stream));
        CU(cudaStreamSynchronize(stream));
    } else {
        CU(cudaStreamSynchronize(stream));   // the terms are host temporaries
    }
    CU(cudaGetLastError());
    return 0;
}

int nidx_suggest_last_ms(nidx_suggest_dict* d, float* ms) {
    int r = require_handle(d);
    if (r) return r;
    if (!ms) return fail(NIDX_EINVAL, "null argument");
    CU(cudaSetDevice(d->device));
    CU(cudaEventSynchronize(d->ev[1]));
    CU(cudaEventElapsedTime(ms, d->ev[0], d->ev[1]));
    return 0;
}

int nidx_txt_set_repeated(nidx_txt_segment* t, const uint64_t* bits) {
    int r = require_handle(t);
    if (!r) r = require_owner(t);
    if (r) return r;
    if (!bits) { t->ix->d_repeated.release(); return 0; }
    return set_rows(t->ix->device, t->ix->d_repeated, bits, ((size_t)t->ix->n_docs + 63) / 64);
}

int nidx_txt_suggest_mask(nidx_txt_segment* t, const uint64_t* sec_bits, const uint64_t* pf_bits, const uint64_t* joined_bits, int32_t op, uint64_t* out_bits,
                          int mem, uint64_t* out_matching, void* stream_) {
    int r = require_handle(t);
    if (r) return r;
    if (!out_bits) return fail(NIDX_EINVAL, "null argument");
    if (op != NIDX_F_AND && op != NIDX_F_OR) return fail(NIDX_EINVAL, "op must be NIDX_F_AND or NIDX_F_OR");
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    CU(cudaSetDevice(t->ix->device));
    WsGuard g(t->ix->pool, stream);
    Workspace& w = *g.w;
    const size_t words = ((size_t)t->ix->n_docs + 63) / 64;
    Stage st(stream, host, host);
    const uint64_t *d_sec, *d_pf, *d_joined;
    uint64_t* d_out;
    st.in(sec_bits, words, &d_sec);
    st.in(pf_bits, words, &d_pf);
    st.in(joined_bits, words, &d_joined);
    st.out(out_bits, words, &d_out);
    r = st.place(w.stage);
    if (r) return r;
    ENSURE(w.misc, 16);
    unsigned long long* d_count = w.misc.as<unsigned long long>();
    CU(cudaMemsetAsync(d_count, 0, 8, stream));
    if (words) {
        suggest_mask_kernel<<<(unsigned)std::max<size_t>(1, std::min<size_t>((words + 255) / 256, 1024)), 256, 0, stream>>>(
            t->ix->n_docs, t->ix->d_repeated, d_sec, d_pf, d_joined, op == NIDX_F_OR, d_out, d_count);
        LAUNCHED();
        CU(cudaGetLastError());
    }
    unsigned long long h = 0;
    CU(cudaMemcpyAsync(&h, d_count, 8, cudaMemcpyDeviceToHost, stream));
    r = st.finish(true);
    if (r) return r;
    if (out_matching) *out_matching = h;
    return 0;
}

int nidx_txt_suggest_fuzzy(nidx_txt_segment* t, const nidx_suggest_clause* clauses, int32_t n_clauses, const uint64_t* exp_bits, int32_t n_exp_rows,
                           uint64_t n_dict, const nidx_txt_phrases* phrases, int32_t k, int32_t match_hits, int mem, uint32_t* out_ids, float* out_scores,
                           int32_t* out_count, uint64_t* out_matches, uint32_t match_cap, uint32_t* out_n_matches, void* stream_) {
    int r = require_handle(t);
    if (r) return r;
    if (!clauses || !out_ids || !out_scores || !out_count || !out_n_matches || (match_cap && !out_matches)) return fail(NIDX_EINVAL, "null argument");
    if (n_clauses < 1 || n_clauses > SG_MAX_CLAUSES) return fail(NIDX_EINVAL, "a fuzzy pass has 1 to %d clauses", SG_MAX_CLAUSES);
    if (k < 1 || k > NIDX_G_MAX_K) return fail(NIDX_EINVAL, "k must be in 1..%d", NIDX_G_MAX_K);
    if (match_hits < 0 || match_hits > SG_MAX_HITS) return fail(NIDX_EINVAL, "match_hits must be in 0..%d", SG_MAX_HITS);
    if (n_exp_rows < 0 || (n_exp_rows && !exp_bits)) return fail(NIDX_EINVAL, "bad expansion bitsets");
    if (n_dict > t->ix->n_terms) return fail(NIDX_EINVAL, "the dictionary has more terms (%llu) than the segment (%u)", (unsigned long long)n_dict, t->ix->n_terms);
    const uint32_t n_ph = phrases ? (uint32_t)std::max(phrases->n, 0) : 0u;
    int n_exact = 0;
    for (int c = 0; c < n_clauses; ++c) {
        const nidx_suggest_clause& C = clauses[c];
        if (C.kind == NIDX_SG_FUZZY && C.arg >= (uint32_t)n_exp_rows) return fail(NIDX_EINVAL, "clause %d: no expansion row %u", c, C.arg);
        else if (C.kind == NIDX_SG_TERM) ++n_exact;
        else if (C.kind == NIDX_SG_PHRASE && C.arg >= n_ph) return fail(NIDX_EINVAL, "clause %d: no phrase %u", c, C.arg);
        else if (C.kind != NIDX_SG_FUZZY && C.kind != NIDX_SG_TERM && C.kind != NIDX_SG_PHRASE) return fail(NIDX_EINVAL, "clause %d: bad kind %d", c, C.kind);
    }
    PhrasePlan pp;
    if (n_ph) {
        nidx_txt_phrases one = *phrases;
        std::vector<uint32_t> query(n_ph, 0), h_off = {0, (uint32_t)n_exact};
        one.query = query.data();   // one query: the plan keeps the phrases in the caller's order
        r = phrase_plan(t, &one, 1, h_off, pp);
        if (r) return r;
    }
    // the clauses as the kernels read them: weights resolved here, warp tasks laid out clause by clause
    const float K1 = 1.2f;
    const size_t exp_words = (n_dict + 63) / 64;
    std::vector<SgClause> sc(n_clauses + 1);
    std::vector<uint32_t> fz_clause;
    uint64_t tasks = 0;
    const float* ph_w = n_ph ? reinterpret_cast<const float*>(pp.buf.data() + pp.o_weight) : nullptr;
    const uint64_t* ph_cap = n_ph ? reinterpret_cast<const uint64_t*>(pp.buf.data() + pp.o_cap_off) : nullptr;
    for (int c = 0; c < n_clauses; ++c) {
        const nidx_suggest_clause& C = clauses[c];
        SgClause& S = sc[c];
        S.task0 = (uint32_t)tasks;
        S.arg = C.arg;
        S.w = 0.f;
        uint64_t postings = 0;
        if (C.kind == NIDX_SG_FUZZY) {
            S.kind = SG_FUZZY;   // its chunks are counted on the device (suggest_chunk_count_kernel)
            fz_clause.push_back((uint32_t)c);
        } else if (C.kind == NIDX_SG_TERM) {
            S.kind = SG_TERM;
            if (C.arg < t->ix->n_terms) { postings = t->ix->own_df[C.arg]; S.w = t->ix->idf[C.arg] * (1.0f + K1); }   // txt_upload_stats' weight
            else S.arg = NIDX_NIL;
        } else {
            S.kind = SG_PHRASE;
            postings = ph_cap[C.arg + 1] - ph_cap[C.arg];
            S.w = ph_w[C.arg];
        }
        tasks += (postings + SG_CHUNK - 1) / SG_CHUNK;
        if (tasks >= (1ull << 32)) return fail(NIDX_EINVAL, "the fuzzy pass has too many posting chunks");
    }
    sc[n_clauses].task0 = (uint32_t)tasks;
    cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
    const bool host = mem == NIDX_MEM_HOST;
    CU(cudaSetDevice(t->ix->device));
    TxtIndex* ix = t->ix;
    for (cudaEvent_t& e : ix->ev_sg)
        if (!e) CU(cudaEventCreate(&e));
    WsGuard g(ix->pool, stream);
    Workspace& w = *g.w;
    const uint32_t n = ix->n_docs;
    const size_t words = ((size_t)n + 63) / 64;
    Stage st(stream, false, host);
    uint32_t* d_ids; float* d_sc; int32_t* d_cnt; uint64_t* d_matches; uint32_t* d_nm;
    st.out(out_ids, (size_t)k, &d_ids);
    st.out(out_scores, (size_t)k, &d_sc);
    st.out(out_count, 1, &d_cnt);
    st.out(out_matches, std::max<size_t>(match_cap, 1), &d_matches);
    st.out(out_n_matches, 1, &d_nm);
    r = st.place(w.stage);
    if (r) return r;
    CU(cudaEventRecord(ix->ev_sg[0], stream));
    TxtDev T;
    T.n_docs = n; T.n_terms = ix->n_terms; T.n_fine = ix->n_fine; T.term_off = ix->d_term_off; T.post = ix->d_post;
    T.skip_row = ix->d_skip_row; T.skip = ix->d_skip; T.alive = t->d_alive;
    Bm25Args a{};
    if (pp.nv) {
        r = phrase_pass(t, pp, T, w, stream, a);
        if (r) return r;
    }
    // scratch (w.scores): [clauses][words] bitsets, [n] scores, [2 words] hit bits, the clauses, the fuzzy clauses' indices;
    // (w.sched): the chunk counts per (fuzzy clause, word), their exclusive prefix sum and the scan's temporary storage
    const size_t o_score = (size_t)n_clauses * std::max<size_t>(words, 1) * 8, o_hits = o_score + ((std::max<size_t>(n, 1) * 4 + 15) & ~(size_t)15),
                 o_cl = o_hits + std::max<size_t>(words, 1) * 8, o_fz = o_cl + ((sc.size() * sizeof(SgClause) + 15) & ~(size_t)15);
    ENSURE(w.scores, o_fz + std::max<size_t>(fz_clause.size(), 1) * 4);
    const size_t n_fw = fz_clause.size() * exp_words;
    if (n_fw + 1 > (size_t)INT32_MAX) return fail(NIDX_EINVAL, "the expansion is too large");
    size_t scan_bytes = 0;
    if (n_fw) CU(cub::DeviceScan::ExclusiveSum(nullptr, scan_bytes, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)(n_fw + 1), stream));
    const size_t o_off = ((n_fw + 1) * 8 + 15) & ~(size_t)15, o_tmp = 2 * o_off;
    ENSURE(w.sched, o_tmp + scan_bytes + 16);
    SgArgs A{};
    A.term_off = ix->d_term_off; A.post = ix->d_post; A.ph_range = a.ph_range; A.ph_post = a.ph_post; A.norm_cache = ix->d_norm_cache;
    A.exp_bits = exp_bits; A.exp_words = exp_words; A.n_dict = (uint32_t)n_dict;
    A.clauses = reinterpret_cast<const SgClause*>(w.scores.p + o_cl); A.n_clauses = (uint32_t)n_clauses;
    A.fz_clause = reinterpret_cast<const uint32_t*>(w.scores.p + o_fz); A.n_fuzzy = (uint32_t)fz_clause.size();
    A.fz_off = reinterpret_cast<const uint64_t*>(w.sched.p + o_off);
    A.n_docs = n; A.words = words; A.bits = w.scores.as<uint64_t>(); A.alive = t->d_alive;
    A.score = reinterpret_cast<float*>(w.scores.p + o_score); A.hit_bits = reinterpret_cast<uint32_t*>(w.scores.p + o_hits);
    CU(cudaMemcpyAsync(w.scores.p + o_cl, sc.data(), sc.size() * sizeof(SgClause), cudaMemcpyHostToDevice, stream));
    if (!fz_clause.empty()) CU(cudaMemcpyAsync(w.scores.p + o_fz, fz_clause.data(), fz_clause.size() * 4, cudaMemcpyHostToDevice, stream));
    if (words) CU(cudaMemsetAsync(A.bits, 0, (size_t)n_clauses * words * 8, stream));
    const int sm = ix->sm_count;
    if (n_fw && words) {   // every expanded term's chunks: counted per word, then laid out by an exclusive prefix sum
        uint64_t* cnt = w.sched.as<uint64_t>();
        CU(cudaMemsetAsync(cnt + n_fw, 0, 8, stream));
        suggest_chunk_count_kernel<<<(unsigned)std::max<size_t>(1, std::min<size_t>((size_t)sm * 8, (n_fw + 255) / 256)), 256, 0, stream>>>(A, cnt);
        LAUNCHED();
        CU(cub::DeviceScan::ExclusiveSum(w.sched.p + o_tmp, scan_bytes, cnt, reinterpret_cast<uint64_t*>(w.sched.p + o_off), (int)(n_fw + 1), stream));
    }
    if ((n_fw || tasks) && words) {   // the fuzzy chunk count stays on the device: a full grid strides over the tasks
        const int blocks = n_fw ? sm * 8 : (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)sm * 8, (tasks * 32 + SG_THREADS - 1) / SG_THREADS));
        suggest_scatter_kernel<<<blocks, SG_THREADS, 0, stream>>>(A);
        LAUNCHED();
    }
    CU(cudaEventRecord(ix->ev_sg[1], stream));
    if (words) {
        const int blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)sm * 8, (2 * words * 32 + SG_THREADS - 1) / SG_THREADS));
        suggest_score_kernel<<<blocks, SG_THREADS, 0, stream>>>(A);
        LAUNCHED();
    }
    CU(cudaEventRecord(ix->ev_sg[2], stream));
    const int cap = topk_cap(k, GF_THREADS);
    const int tk_blocks = (int)std::max<size_t>(1, std::min<size_t>((size_t)sm * 2, ((size_t)n + GF_THREADS * 16 - 1) / (GF_THREADS * 16)));
    ENSURE(w.partial, (size_t)tk_blocks * k * 8);
    CU(cudaFuncSetAttribute(graph_topk_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap * 8));
    CU(cudaFuncSetAttribute(graph_topk_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, cap * 8));
    if (n) {
        graph_topk_kernel<<<tk_blocks, GF_THREADS, (size_t)cap * 8, stream>>>(n, A.hit_bits, A.score, nullptr, k, cap, w.partial.as<uint64_t>());
        LAUNCHED();
    } else {
        CU(cudaMemsetAsync(w.partial, 0, (size_t)tk_blocks * k * 8, stream));
    }
    graph_topk_merge_kernel<<<1, GF_THREADS, (size_t)cap * 8, stream>>>(w.partial.as<uint64_t>(), tk_blocks * k, k, cap, d_ids, d_sc, d_cnt);
    LAUNCHED();
    CU(cudaEventRecord(ix->ev_sg[3], stream));
    CU(cudaMemsetAsync(d_nm, 0, 4, stream));
    uint64_t fuzzy_tasks = 0;
    for (int c = 0; c < n_clauses; ++c) fuzzy_tasks += sc[c].kind == SG_FUZZY ? exp_words : 0;
    if (match_hits && fuzzy_tasks) {
        const int blocks = (int)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)sm * 8, (fuzzy_tasks * 32 + SG_THREADS - 1) / SG_THREADS));
        suggest_matches_kernel<<<blocks, SG_THREADS, 0, stream>>>(A, d_ids, d_cnt, match_hits, d_matches, match_cap, d_nm);
        LAUNCHED();
    }
    CU(cudaEventRecord(ix->ev_sg[4], stream));
    CU(cudaGetLastError());
    return st.finish(true);   // the phrase plan and the clauses are host temporaries
}

int nidx_txt_suggest_last_times(nidx_txt_segment* t, float* ms4) {
    int r = require_handle(t);
    if (r) return r;
    if (!ms4) return fail(NIDX_EINVAL, "null argument");
    if (!t->ix->ev_sg[4]) return fail(NIDX_ESTATE, "no fuzzy suggest pass has run on this segment");
    CU(cudaSetDevice(t->ix->device));
    CU(cudaEventSynchronize(t->ix->ev_sg[4]));
    for (int i = 0; i < 4; ++i) CU(cudaEventElapsedTime(ms4 + i, t->ix->ev_sg[i], t->ix->ev_sg[i + 1]));
    return 0;
}

}  // extern "C"
