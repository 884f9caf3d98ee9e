// nidx_b200 — K8: segments sharded over the GPUs of one node, behind the C ABI (sm_90a + NCCL over NVLink).
//
// Replaces the reference's scatter-gather over shards / segments:
//   nidx/src/searcher/grpc.rs:253-431            fan a request out to every shard's searcher, gather the responses
//   nidx/src/searcher/shard_merge.rs:332-348     merge_vector_responses: kmerge_by(score >=), take(limit)
//   nidx/src/searcher/shard_merge.rs:177-231     merge_document / merge_paragraph_responses (bm25 desc, shard, docaddr)
//   nidx/nidx_vector/src/searcher.rs:150-199     Fssc: the cross-SEGMENT collection of one index -- keyed by paragraph id,
//                                                optionally suppressing byte-identical vectors
// One process per GPU holds one segment; per batch every rank searches its segment for the same queries, the [nq][k]
// partial results travel in ONE ncclAllGather on the caller's stream (80 KB per rank at nq = 1024, k = 10: latency
// bound, so one collective per batch) and every rank merges the gathered parts with one kernel -- search, exchange and
// merge are enqueued back to back on one stream, no host synchronisation in between.
// NCCL is bound at run time (dlopen of libnccl.so.2, the copy already loaded in the process if there is one), so the
// library still loads -- and every single-GPU entry point works -- on a machine without NCCL.
#pragma once
#include <dlfcn.h>

#include <mutex>

#include "common.cuh"

namespace nidx {

// The slice of nccl.h this file uses (NCCL 2.x ABI: ncclUniqueId is 128 bytes, enums as below).
typedef struct ncclComm* nccl_comm_t;
typedef struct { char internal[128]; } nccl_unique_id;
constexpr int NCCL_SUCCESS = 0;
constexpr int NCCL_INT8 = 0, NCCL_UINT64 = 5, NCCL_SUM = 0;

struct NcclApi {
    void* handle = nullptr;
    int (*GetUniqueId)(nccl_unique_id*) = nullptr;
    int (*CommInitRank)(nccl_comm_t*, int, nccl_unique_id, int) = nullptr;
    int (*CommDestroy)(nccl_comm_t) = nullptr;
    int (*AllGather)(const void*, void*, size_t, int, nccl_comm_t, cudaStream_t) = nullptr;
    int (*AllReduce)(const void*, void*, size_t, int, int, nccl_comm_t, cudaStream_t) = nullptr;
    const char* (*GetErrorString)(int) = nullptr;
    bool ok = false;
};

inline NcclApi& nccl_api() {
    static NcclApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD);   // the copy the host process already uses (e.g. torch's)
        if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!h) return;
        api.handle = h;
        api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
        api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
        api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
        api.AllGather = reinterpret_cast<decltype(api.AllGather)>(dlsym(h, "ncclAllGather"));
        api.AllReduce = reinterpret_cast<decltype(api.AllReduce)>(dlsym(h, "ncclAllReduce"));
        api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
        api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.AllGather && api.AllReduce && api.GetErrorString;
    });
    return api;
}

// ---- exchange record of one part: [ids nq*k u32][scores nq*k f32] (+ [par_key nq*k u64][vec_key nq*k u64] with de-dup), in u32 words
// (nidx_vec_shard_record writes one, nidx_shard_merge merges n_parts of them laid end to end) ------------------------------------
__host__ __device__ __forceinline__ size_t shard_part_words(int nq, int k, bool dedup) { return (size_t)nq * k * (dedup ? 6 : 2); }

// 64-bit keys of the local results for the cross-segment de-duplication: par_key = the caller's paragraph key (the hash of the
// paragraph id, nidx_vec_set_paragraph_keys) or, without keys, (rank, paragraph address); vec_key = a 64-bit hash of the
// vector's bytes (the reference compares the bytes themselves, searcher.rs:183-189; 2^-64 per pair is the price of not
// shipping 3 KB per result).  One warp per result.
__global__ void shard_keys_kernel(VecDev V, const uint32_t* __restrict__ ids, int n_results, const uint64_t* __restrict__ par_keys, uint32_t rank,
                                  int hash_vectors, uint64_t* __restrict__ out_par, uint64_t* __restrict__ out_vec) {
    int r = (int)((blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
    if (r >= n_results) return;
    uint32_t id = ids[r];
    uint64_t h = 0, pk = 0;
    if (id != NIL) {
        const uint32_t* row = reinterpret_cast<const uint32_t*>(V.vecs + (size_t)id * V.ld);
        uint64_t acc = 0x9E3779B97F4A7C15ull;
        for (int i = lane; hash_vectors && i < V.d; i += 32) {
            uint64_t x = ((uint64_t)(uint32_t)(i + 1) << 32) | row[i];
            x ^= x >> 33; x *= 0xFF51AFD7ED558CCDull; x ^= x >> 33; x *= 0xC4CEB9FE1A85EC53ull; x ^= x >> 33;
            acc += x;                                   // order independent over the lanes: position is mixed into x
        }
        for (int off = 16; off >= 1; off >>= 1) acc += __shfl_xor_sync(0xFFFFFFFFu, acc, off);
        h = acc;
        uint32_t p = V.paragraph_of ? V.paragraph_of[id] : id;
        pk = par_keys ? par_keys[p] : (((uint64_t)rank << 32) | p);
    }
    if (lane == 0) { out_par[r] = pk; out_vec[r] = h; }
}

// Fssc (searcher.rs:150-199) over the gathered parts, one thread per query, state in shared memory: candidates are added
// part by part (the reference's segment loop), each part in its own order (score descending).
//   add(): with_duplicates == false and the vector was seen -> skip; full -> the lowest-scored entry that scores below the
//   candidate is evicted; the candidate is inserted unless its paragraph key is already present (HashSet::insert keeps the
//   old element), so an eviction followed by a present key shrinks the collection.  Among entries tied for the lowest score the
//   first in insertion order is evicted (the reference takes whichever its HashSet iterates first, which is not fixed).  Result
//   sorted by score descending, stable over the collection's order (insertion order here).
__global__ void shard_fssc_kernel(const uint32_t* __restrict__ gathered, int n_parts, size_t part_words, int nq, int k, int with_duplicates,
                                  uint32_t* __restrict__ out_ids, float* __restrict__ out_scores, int* __restrict__ out_part, int* __restrict__ out_counts) {
    extern __shared__ __align__(16) unsigned char fs_smem[];
    int q = blockIdx.x * blockDim.x + threadIdx.x;
    // per-thread slices: buff entries (score, slot) x k, par keys x k, seen vec keys x n_parts*k
    size_t per = (size_t)k * 16 + (size_t)n_parts * k * 8;
    unsigned char* base = fs_smem + (size_t)threadIdx.x * per;
    float* b_score = reinterpret_cast<float*>(base);
    uint32_t* b_slot = reinterpret_cast<uint32_t*>(base + (size_t)k * 4);
    uint64_t* b_par = reinterpret_cast<uint64_t*>(base + (size_t)k * 8);
    uint64_t* seen = reinterpret_cast<uint64_t*>(base + (size_t)k * 16);
    if (q >= nq) return;
    int nb = 0, nseen = 0;
    size_t nk = (size_t)nq * k;
    for (int part = 0; part < n_parts; ++part) {
        const uint32_t* P = gathered + (size_t)part * part_words;
        const uint32_t* ids = P + (size_t)q * k;
        const float* sc = reinterpret_cast<const float*>(P + nk) + (size_t)q * k;
        const uint64_t* pk = reinterpret_cast<const uint64_t*>(P + 2 * nk) + (size_t)q * k;
        const uint64_t* vk = reinterpret_cast<const uint64_t*>(P + 4 * nk) + (size_t)q * k;
        for (int pos = 0; pos < k; ++pos) {
            if (ids[pos] == NIL) break;
            float s = sc[pos];
            if (!with_duplicates) {
                uint64_t v = vk[pos];
                bool dup = false;
                for (int i = 0; i < nseen; ++i) dup |= seen[i] == v;
                if (dup) continue;
                seen[nseen++] = v;
            }
            uint64_t key = pk[pos];
            if (nb == k) {
                int victim = -1;
                for (int i = 0; i < nb; ++i)
                    if (s > b_score[i] && (victim < 0 || b_score[i] < b_score[victim])) victim = i;   // first minimum among the lower-scored
                if (victim < 0) continue;
                for (int i = victim; i + 1 < nb; ++i) { b_score[i] = b_score[i + 1]; b_slot[i] = b_slot[i + 1]; b_par[i] = b_par[i + 1]; }
                --nb;
            }
            bool present = false;
            for (int i = 0; i < nb; ++i) present |= b_par[i] == key;
            if (!present) { b_score[nb] = s; b_slot[nb] = (uint32_t)(part * k + pos); b_par[nb] = key; ++nb; }
        }
    }
    // stable sort by score descending (insertion sort; nb <= k)
    for (int i = 1; i < nb; ++i) {
        float s = b_score[i]; uint32_t sl = b_slot[i];
        int j = i - 1;
        while (j >= 0 && b_score[j] < s) { b_score[j + 1] = b_score[j]; b_slot[j + 1] = b_slot[j]; --j; }
        b_score[j + 1] = s; b_slot[j + 1] = sl;
    }
    for (int i = 0; i < k; ++i) {
        size_t dst = (size_t)q * k + i;
        if (i < nb) {
            int part = b_slot[i] / k, pos = b_slot[i] % k;
            out_ids[dst] = gathered[(size_t)part * part_words + (size_t)q * k + pos];
            out_scores[dst] = b_score[i];
            if (out_part) out_part[dst] = part;
        } else {
            out_ids[dst] = NIL; out_scores[dst] = 0.0f;
            if (out_part) out_part[dst] = -1;
        }
    }
    if (out_counts) out_counts[q] = nb;
}

// merge_vector_responses (shard_merge.rs:332-348): kmerge_by(|a, b| a.score >= b.score).take(k) over the parts, taken in the order
// given (the reference's `responses` vector).  itertools 0.14's KMergeBy restated: a binary heap, ordered by `less_than`, of the
// non-empty parts' iterators in part order, built by heapify; every next() yields the head of heap[0], advances that part or, when it
// is exhausted, swap_remove(0)s it, then sift_down(0) (the branchless form: the right child is taken when less_than(right, left)).
// The predicate holds both ways for equal scores, so ties do NOT come out lower part first: the heap's shape decides which equal
// head leads.  A part ends at its first NIL.  IEEE f32 >=: -0 and +0 are equal, a NaN is never >=.  One thread per query; its heap
// (part * k + position of each part's head) lives in shared memory, entry i of thread t at [i * blockDim.x + t].
__global__ void kmerge_parts_kernel(const uint32_t* __restrict__ ids, const float* __restrict__ scores, int n_parts, size_t part_stride, int nq, int k,
                                    uint32_t* __restrict__ out_ids, float* __restrict__ out_scores, int* __restrict__ out_part, int* __restrict__ out_counts) {
    extern __shared__ __align__(16) uint32_t km_heap[];
    int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    uint32_t* heap = km_heap + threadIdx.x;
    const size_t W = blockDim.x;
    auto src = [&](uint32_t slot) { return (size_t)(slot / (uint32_t)k) * part_stride + (size_t)q * k + slot % (uint32_t)k; };
    auto less = [&](uint32_t a, uint32_t b) { return scores[src(a)] >= scores[src(b)]; };
    auto swap = [&](int a, int b) { uint32_t t = heap[a * W]; heap[a * W] = heap[b * W]; heap[b * W] = t; };
    auto sift_down = [&](int pos, int len) {
        int child = 2 * pos + 1;
        while (child + 1 < len) {
            child += less(heap[(child + 1) * W], heap[child * W]) ? 1 : 0;
            if (!less(heap[child * W], heap[pos * W])) return;
            swap(pos, child);
            pos = child;
            child = 2 * pos + 1;
        }
        if (child + 1 == len && less(heap[child * W], heap[pos * W])) swap(pos, child);
    };
    int len = 0;
    for (int part = 0; part < n_parts; ++part)
        if (ids[(size_t)part * part_stride + (size_t)q * k] != NIL) heap[(size_t)(len++) * W] = (uint32_t)part * (uint32_t)k;
    for (int i = len / 2 - 1; i >= 0; --i) sift_down(i, len);
    int c = 0;
    for (; c < k && len > 0; ++c) {
        uint32_t top = heap[0];
        size_t s = src(top), dst = (size_t)q * k + c;
        out_ids[dst] = ids[s];
        out_scores[dst] = scores[s];
        if (out_part) out_part[dst] = (int)(top / (uint32_t)k);
        if (top % (uint32_t)k + 1 < (uint32_t)k && ids[s + 1] != NIL) heap[0] = top + 1;
        else heap[0] = heap[(size_t)(--len) * W];
        sift_down(0, len);
    }
    for (int i = c; i < k; ++i) {
        size_t dst = (size_t)q * k + i;
        out_ids[dst] = NIL; out_scores[dst] = 0.0f;
        if (out_part) out_part[dst] = -1;
    }
    if (out_counts) out_counts[q] = c;
}

__global__ void shard_count_kernel(const uint32_t* __restrict__ ids, int nq, int k, int* __restrict__ out_counts) {
    int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= nq) return;
    int c = 0;
    for (int i = 0; i < k; ++i) c += ids[(size_t)q * k + i] != NIL;
    out_counts[q] = c;
}

}  // namespace nidx
