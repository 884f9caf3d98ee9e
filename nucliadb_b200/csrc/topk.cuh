// nidx_b200 — block-wide streaming top-k over 64-bit rank keys (sm_90a).
//
// Used by the exact scan (segment.rs:611-617: sort desc + take k), the BM25 collector
// (TopDocs::with_limit(k).order_by_score, nidx_text/src/reader.rs:432) and the cross-segment merge
// (searcher.rs:150-199 / shard_merge.rs:332-348).  Keys are unique (they embed the id), larger
// key = better; key 0 is "nothing".
#pragma once
#include "common.cuh"

namespace nidx {

// In-place bitonic sort, descending, of `n` (power of two) keys in shared memory by the whole block.
__device__ inline void block_bitonic_sort_desc(uint64_t* keys, int n) {
    for (int size = 2; size <= n; size <<= 1) {
        for (int stride = size >> 1; stride > 0; stride >>= 1) {
            __syncthreads();
            for (int t = threadIdx.x; t < (n >> 1); t += blockDim.x) {
                int lo = 2 * t - (t & (stride - 1));
                int hi = lo + stride;
                bool desc = ((lo & size) == 0);
                uint64_t a = keys[lo], b = keys[hi];
                if ((a < b) == desc) { keys[lo] = b; keys[hi] = a; }
            }
        }
    }
    __syncthreads();
}

// Streaming top-k state in shared memory.  cap is a power of two >= 2*k and >= k + blockDim.x.
struct BlockTopK {
    uint64_t* buf;   // [cap]
    int* count;      // entries in buf
    uint64_t* thr;   // keys <= *thr cannot enter the top-k any more
    int k, cap;

    __device__ void init(uint64_t* buf_, int* count_, uint64_t* thr_, int k_, int cap_) {
        buf = buf_; count = count_; thr = thr_; k = k_; cap = cap_;
        if (threadIdx.x == 0) { *count = 0; *thr = 0; }
        __syncthreads();
    }
    // Sort, keep the best k, raise the threshold.  Must be called by all threads.
    __device__ void flush() {
        __syncthreads();
        int c = *count;
        for (int i = c + threadIdx.x; i < cap; i += blockDim.x) buf[i] = 0;
        block_bitonic_sort_desc(buf, cap);
        if (threadIdx.x == 0) {
            int kept = c < k ? c : k;
            *count = kept;
            if (kept == k) *thr = buf[k - 1];
        }
        __syncthreads();
    }
    // One round: every thread may offer one key (0 = none).  All threads must call.
    __device__ void offer(uint64_t key) {
        if (key > *thr) {
            int pos = atomicAdd(count, 1);
            buf[pos] = key;  // cap >= k + blockDim.x and count <= k after a flush
        }
        // The flush decision must be the same in every thread: the count is read between two barriers, so no thread can
        // reach the next round's atomicAdd before all threads have read it (flush() contains barriers).
        __syncthreads();
        int c = *count;
        __syncthreads();
        if (c > cap - (int)blockDim.x) flush();
    }
    // Final: sorted best-k in buf[0..min(count,k)).
    __device__ int finish() {
        flush();
        return *count;
    }
};

__host__ __device__ inline int topk_cap(int k, int block) {
    int need = 2 * k > k + block ? 2 * k : k + block;
    need = need < 2 * block ? 2 * block : need;
    int cap = 1;
    while (cap < need) cap <<= 1;
    return cap;
}

}  // namespace nidx
