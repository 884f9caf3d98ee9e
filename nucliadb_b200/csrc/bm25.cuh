// nidx_b200 — K7: BM25 top-k over device-resident postings (sm_90a).
//
// Replaces the tantivy collector call of the reference:
//   nidx/nidx_text/src/reader.rs:432-435        TopDocs::with_limit(k+1).order_by_score() + Count
//   nidx/nidx_paragraph/src/reader.rs:290-292   same, OR of TermQuery(Basic) (keyword_parser.rs:62-67)
// with tantivy 0.26's BM25 (restated in oracle/bm25.hpp; parity unpinned, SURVEY F9):
//   score(doc) = sum over matching query terms of  idf_t * (1 + k1) * tf / (tf + k1 * (1 - b + b * fieldnorm / avg))
//
// Index-time layout (once per segment):
//   * post[i] = (doc, tf << 8 | fieldnorm_id(doc)), ascending doc per term: ONE 8-byte record per posting, the document's
//     length code travels with it (no random gather of fieldnorm[doc]);
//   * skip[row][f] = first posting of the term with doc >= f * BM_FINE, for every term with df >= BM_SKIP_DF: the slice
//     of a term in ANY run of fine tiles is two table entries.
// Query time: one CTA per query walks the document space in tiles of up to BM_MAX_SPAN fine tiles, sized per query so that a
// tile holds about BM_SLOTS postings.  A query's postings touch a small fraction of a tile's documents (50 terms of
// df ~5 k over 5 M documents: 5 %), so the accumulator is COMPACT: a bitmap of the touched documents + a prefix
// popcount give every touched document a dense rank.  Per tile (every thread owns BM_PT posting slots, held in registers):
//   A  all of the tile's postings are requested at once (BM_PT independent 8-byte loads per thread: the memory-level
//      parallelism that hides HBM latency with only ~24 warps per SM), in 8-posting octets of ONE term each -- consecutive
//      lanes read consecutive postings -- and every posting sets its document's bit (shared-memory atomicOr);
//   S  exclusive prefix popcount of the bitmap words: rank base per word; the popcount itself is the Count collector
//      (ANDed with the alive bits);
//   C  the same postings, from registers: score, atomicAdd into acc[rank].  Contributions are fixed point (2^-shift):
//      the sum does not depend on the order, equal scores stay bit-equal and TopDocs' (score desc, doc asc) tie order is
//      deterministic.  The shift is the query's own (largest s <= 24 with max(1, nt * max_t w_t) * 2^s < 4e9, so no sum can
//      leave uint32): a query scores the same in any batch and on every segment that shares the index's statistics.
//      tests/bm25_model.py restates the arithmetic bit for bit and bounds its error against float64.  The thread whose add
//      carries a document's sum across the current top-k threshold (OR) or completes the conjunction (AND) records it as a
//      candidate: only documents that can still enter the top-k are looked at again;
//   D  candidates -> streaming top-k buffer (final sums, exact threshold test) while warp 0 resolves the next tile's
//      slices (skip entries prefetched one tile ahead); then the bitmap, the used accumulators and the counters are cleared.
// A tile that holds more postings than slots is redone with half the span; a single fine tile that still does not fit runs in
// several rounds of slots (postings re-read in phase C): distinct documents <= BM_FINE = the accumulator's capacity, whatever
// the posting count.
// No atomicCAS, no probing: one atomicOr + one atomicAdd per posting (scripts/ubench_smem.cu measures the shared-memory atomic
// rate; a hash-table accumulator would spend its instructions in divergent probe loops).
// HBM traffic = the query's postings once (8 B each) + one skip entry per (term, tile).
#pragma once
#include "common.cuh"
#include "topk.cuh"

namespace nidx {

// CTA shape: threads x posting slots per thread = 4096 slots per round; CTAs per SM (launch bounds).  512 x 8 x 2 (64 registers,
// 32 warps per SM) by default; 256 x 16 x 3 (80 registers, 24 warps per SM) gives the same outputs
// (make EXTRA="-DBM_THREADS_CFG=256 -DBM_PT_CFG=16 -DBM_MINB_CFG=3" builds it).
#ifndef BM_THREADS_CFG
#define BM_THREADS_CFG 512
#define BM_PT_CFG 8
#define BM_MINB_CFG 2
#endif
constexpr int BM_THREADS = BM_THREADS_CFG;
constexpr int BM_WARPS = BM_THREADS / 32;
constexpr int BM_MAX_TERMS = 128;
constexpr int BM_TPL = BM_MAX_TERMS / 32;  // query terms per lane of the resolving warp
constexpr int BM_FINE = 4096;              // skip-table granularity (documents)
constexpr int BM_SKIP_DF = 256;            // terms with at least this many postings get a skip row
constexpr int BM_PT = BM_PT_CFG;           // posting slots per thread and round (registers)
constexpr int BM_SLOTS = BM_THREADS * BM_PT;   // 4096 posting slots per round
constexpr int BM_OCT = BM_SLOTS / 8;       // 8-posting octets per round (one term each)
constexpr int BM_MAX_SPAN = 32;            // fine tiles per tile at most: 131 072 documents, a 16 KB bitmap
constexpr int BM_WORDS = BM_MAX_SPAN * BM_FINE / 32;   // bitmap words
constexpr int BM_ACC = 4096;               // distinct documents per tile the compact accumulator holds (>= BM_FINE and >= BM_SLOTS)

struct TxtDev {
    uint32_t n_docs, n_terms, n_fine;
    const uint64_t* term_off;
    const uint2* post;               // (doc, tf << 8 | fieldnorm id)
    const uint32_t* skip_row;        // [n_terms] row in skip[] or NIL
    const uint32_t* skip;            // [rows][n_fine + 1] posting index relative to term_off[term]
    const uint64_t* alive;
};

struct Bm25Args {
    const uint32_t* query_terms;
    const uint32_t* query_off;
    int nq;
    int k, cap;                 // cap: top-k buffer entries (power of two >= 2k, >= k + BM_THREADS)
    const float* term_weight;   // [n_terms] idf * (1 + k1) from the collection statistics
    const float* norm_cache;    // [256] k1 * (1 - b + b * fieldnorm(id) / avg)
    int after_mode;             // search-after (nidx_paragraph reader.rs:379-392): 0 none, 1 Drop, 2 KeepAfter, 3 Keep
    float after_score;
    uint64_t after_docaddr, docaddr_base;
    uint64_t* out_keys;         // [nq][k] rank keys (score desc, doc asc), 0 = none
    unsigned long long* out_total;  // [nq] matching documents (Count collector)
    // Phrases (phrase.cuh): query q's clauses are its terms, then the virtual posting lists ph_qoff[q] .. ph_qoff[q + 1), each
    // scored with its real frequency (a TF kernel runs; basic_terms keeps the terms at tf == 1).  ph_qoff == nullptr: no phrases.
    const uint32_t* ph_qoff;    // [nq + 1]
    const uint64_t* ph_range;   // [2 nv] (first, end) posting of list v in ph_post
    const uint2* ph_post;
    const uint32_t* ph_skip_row;   // [nv] row in ph_skip or NIL
    const uint32_t* ph_skip;       // [rows][n_fine + 1] posting index relative to the list's first
    const float* ph_weight;     // [nv] (sum of the terms' idf) * (1 + k1)
    int basic_terms;            // TF kernels: the query terms are Basic (tf == 1) and only the phrases count their frequency
};

// A query term's postings are addressed in 8-byte units of the address space, so that a term's slice is read the same way whether
// it lies in the segment's postings or in a phrase's virtual list.
__device__ __forceinline__ uint64_t post_addr(const uint2* p) { return (uint64_t)reinterpret_cast<uintptr_t>(p) >> 3; }
__device__ __forceinline__ const uint2* post_at(uint64_t a) { return reinterpret_cast<const uint2*>(a << 3); }

// ---- index-time kernels ---------------------------------------------------------------------------------
__global__ void bm25_pack_kernel(const uint32_t* __restrict__ post_doc, const uint32_t* __restrict__ post_tf, const unsigned char* __restrict__ fieldnorm,
                                 uint64_t n_post, uint2* __restrict__ post) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n_post; i += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t tf = post_tf ? post_tf[i] : 1u;
        if (tf > 0xFFFFFFu) tf = 0xFFFFFFu;
        uint32_t d = post_doc[i];
        post[i] = make_uint2(d, (tf << 8) | fieldnorm[d]);
    }
}
// one thread per (skip row, fine-tile boundary)
__global__ void bm25_build_skip_kernel(const uint64_t* __restrict__ term_off, const uint2* __restrict__ post, const uint32_t* __restrict__ row_term,
                                       uint32_t n_rows, uint32_t n_fine, uint32_t* __restrict__ skip) {
    uint64_t total = (uint64_t)n_rows * (n_fine + 1);
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        uint32_t row = (uint32_t)(i / (n_fine + 1)), t = (uint32_t)(i % (n_fine + 1));
        uint32_t term = row_term[row];
        uint64_t b = term_off[term], e = term_off[term + 1];
        uint64_t bound = (uint64_t)t * BM_FINE;
        uint64_t l = b, r = e;
        while (l < r) {
            uint64_t m = (l + r) >> 1;
            if ((uint64_t)post[m].x < bound) l = m + 1; else r = m;
        }
        skip[i] = (uint32_t)(l - b);
    }
}

// ---- facet counts (tantivy FacetCollector, nidx_text/src/reader.rs:388-450, nidx_paragraph/src/reader.rs:252-347) ----------
// The segment's facets are a dictionary in facet order (host side) and every document's facet ords, ascending, in CSR form
// (HBM).  A request maps every ord to the bucket of the requested facet's child it lies under, or NIL (the host's collapse
// table); buckets ascend with the ord, so the repeats of one bucket among a document's ords are adjacent and a document adds one
// to each of its buckets once.
struct FacetArgs {
    const uint32_t* doc_off;   // [n_docs + 1]
    const uint32_t* ords;      // [doc_off[n_docs]]
    const uint32_t* bucket;    // [n_facets] ord -> bucket or NIL
    uint32_t n_buckets;
    int smem;                  // 1: one CTA counts into shared memory and writes its row / adds its histogram; 0: global atomics
    uint32_t* out;             // [nq][n_buckets]
};
constexpr uint32_t FACET_SMEM_BUCKETS = 4096;   // 16 KB of shared counters at most (bm25: beside the ~80 KB of a k <= 128 search)

__device__ __forceinline__ void facet_doc(const FacetArgs& F, uint32_t doc, uint32_t* cnt) {
    const uint32_t e = F.doc_off[doc + 1];
    uint32_t prev = NIL;
    for (uint32_t i = F.doc_off[doc]; i < e; ++i) {
        uint32_t b = __ldg(F.bucket + __ldg(F.ords + i));
        if (b != NIL && b != prev) { atomicAdd(cnt + b, 1u); prev = b; }
    }
}

// FACET_BATCH documents at once (NIL = none): their offsets, then their ords step by step, are independent loads in flight
// together -- a document alone is a chain of three dependent loads, and a pass over many documents is bound by its latency.
constexpr int FACET_BATCH = 4;
__device__ __forceinline__ void facet_docs(const FacetArgs& F, const uint32_t (&doc)[FACET_BATCH], uint32_t* cnt) {
    uint32_t b[FACET_BATCH], e[FACET_BATCH], prev[FACET_BATCH];
#pragma unroll
    for (int j = 0; j < FACET_BATCH; ++j) {
        b[j] = doc[j] != NIL ? __ldg(F.doc_off + doc[j]) : 0;
        e[j] = doc[j] != NIL ? __ldg(F.doc_off + doc[j] + 1) : 0;
        prev[j] = NIL;
    }
    for (bool more = true; more;) {
        uint32_t bk[FACET_BATCH];
        more = false;
#pragma unroll
        for (int j = 0; j < FACET_BATCH; ++j) bk[j] = b[j] < e[j] ? __ldg(F.ords + b[j]) : NIL;
#pragma unroll
        for (int j = 0; j < FACET_BATCH; ++j) bk[j] = bk[j] != NIL ? __ldg(F.bucket + bk[j]) : NIL;
#pragma unroll
        for (int j = 0; j < FACET_BATCH; ++j) {
            if (b[j] < e[j]) { ++b[j]; more |= b[j] < e[j]; }
            if (bk[j] != NIL && bk[j] != prev[j]) { atomicAdd(cnt + bk[j], 1u); prev[j] = bk[j]; }
        }
    }
}

// The matched-everything count (AllQuery: empty body / only_faceted catalogue): one pass over the CSR and the alive bits, a
// histogram per block in shared memory (F.smem) added to F.out[0][*] at the end.
__global__ void facet_count_all_kernel(uint32_t n_docs, const uint64_t* __restrict__ alive, FacetArgs F) {
    extern __shared__ uint32_t hist[];
    uint32_t* cnt = F.smem ? hist : F.out;
    if (F.smem) for (uint32_t i = threadIdx.x; i < F.n_buckets; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const uint32_t stride = gridDim.x * blockDim.x;   // a thread takes FACET_BATCH documents `stride` apart: every load stays coalesced
    for (uint32_t d0 = blockIdx.x * blockDim.x + threadIdx.x; d0 < n_docs; d0 += FACET_BATCH * stride) {
        uint32_t dd[FACET_BATCH];
#pragma unroll
        for (int j = 0; j < FACET_BATCH; ++j) {
            uint32_t d = d0 + j * stride;
            dd[j] = d < n_docs && (!alive || ((alive[d >> 6] >> (d & 63)) & 1ull)) ? d : NIL;
        }
        facet_docs(F, dd, cnt);
    }
    if (F.smem) {
        __syncthreads();
        for (uint32_t i = threadIdx.x; i < F.n_buckets; i += blockDim.x)
            if (hist[i]) atomicAdd(F.out + i, hist[i]);
    }
}

// ---- order by date (TopDocs::order_by_fast_field("created" | "modified", Desc | Asc): nidx_text/src/reader.rs:208-224,
// nidx_paragraph/src/reader.rs:229-243) ------------------------------------------------------------------------------------------
// Every document of a segment holds the dense rank of its date among the segment's distinct dates (1..n_ranks, ascending seconds;
// 0 = no date), built once by nidx_txt_set_dates.  The rank in the requested direction takes the score's place in the 64-bit key:
//   key = dir_rank << 32 | (0x7FFFFFFF - doc) << 1,   dir_rank = rank (DESC) or n_ranks + 1 - rank (ASC), 0 without a date,
// so the existing top-k orders by (date in the requested direction, doc ascending), undated documents last, and key_id() still
// gives the document.  The order is exact over all of i64: the ranks come from a sort of the seconds themselves.
struct OrderArgs {
    const uint32_t* rank;      // [n_docs rounded up to 8] (padding 0)
    const int64_t* secs;       // [n_docs] seconds, NIDX_DATE_NONE = no date
    uint32_t n_ranks;
    int asc;
};
constexpr int64_t DATE_NONE = INT64_MIN;

__device__ __forceinline__ uint64_t order_key(uint32_t rank, uint32_t n_ranks, int asc, uint32_t doc) {
    const uint32_t dr = rank == 0 ? 0u : (asc ? n_ranks + 1u - rank : rank);
    return ((uint64_t)dr << 32) | (uint64_t)((0x7FFFFFFFu - doc) << 1);
}
__device__ __forceinline__ uint64_t order_key(const OrderArgs& O, uint32_t doc) { return order_key(__ldg(O.rank + doc), O.n_ranks, O.asc, doc); }

// nidx_txt_set_dates: sorted (seconds, doc) pairs -> first-of-its-date flags (NIDX_DATE_NONE sorts first and is never flagged); their
// inclusive prefix sum is the dense rank, scattered back to the documents.
__global__ void date_flag_kernel(const int64_t* __restrict__ sorted, uint32_t n, uint32_t* __restrict__ flag) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        flag[i] = sorted[i] != DATE_NONE && (i == 0 || sorted[i] != sorted[i - 1]);
}
__global__ void date_scatter_kernel(const uint32_t* __restrict__ incl, const uint32_t* __restrict__ doc_of, uint32_t n, uint32_t* __restrict__ rank) {
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) rank[doc_of[i]] = incl[i];
}

// The catalogue listing (empty body + order: AllQuery, nidx_text/src/search_query.rs:100-101): per CTA, the top-k by date key of
// a grid-stride slice of the alive documents, written to partial[blockIdx.x][k]; the Count of AllQuery (alive documents) is added
// to *total (zeroed by the caller).  A thread takes DATE_PT consecutive documents per round: two 16-byte rank loads and one byte of
// alive bits, all in flight together.  dynamic smem: cap * 8.
constexpr int DATE_PT = 8;
__global__ void date_topk_all_kernel(uint32_t n_docs, const uint64_t* __restrict__ alive, OrderArgs O, int k, int cap, uint64_t* __restrict__ partial,
                                     unsigned long long* __restrict__ total) {
    extern __shared__ __align__(16) uint64_t tk_buf[];
    __shared__ int tk_count;
    __shared__ uint64_t tk_thr;
    __shared__ unsigned long long s_hits;
    BlockTopK tk;
    if (threadIdx.x == 0) s_hits = 0;
    tk.init(tk_buf, &tk_count, &tk_thr, k, cap);
    unsigned int hits = 0;
    const uint32_t step = gridDim.x * blockDim.x * DATE_PT;
    for (uint32_t base = blockIdx.x * blockDim.x * DATE_PT; base < n_docs; base += step) {   // (uniform per CTA)
        const uint32_t d0 = base + threadIdx.x * DATE_PT;
        uint32_t r[DATE_PT];
        uint32_t live = 0;
        if (d0 < n_docs) {
            const uint4 a = __ldg(reinterpret_cast<const uint4*>(O.rank + d0)), b = __ldg(reinterpret_cast<const uint4*>(O.rank + d0) + 1);
            r[0] = a.x; r[1] = a.y; r[2] = a.z; r[3] = a.w; r[4] = b.x; r[5] = b.y; r[6] = b.z; r[7] = b.w;
            live = alive ? __ldg(reinterpret_cast<const unsigned char*>(alive) + (d0 >> 3)) : 0xFFu;
            if (n_docs - d0 < DATE_PT) live &= (1u << (n_docs - d0)) - 1u;
            hits += __popc(live);
        }
#pragma unroll
        for (int u = 0; u < DATE_PT; ++u) tk.offer((live >> u) & 1u ? order_key(r[u], O.n_ranks, O.asc, d0 + u) : 0);
    }
    for (int off = 16; off >= 1; off >>= 1) hits += __shfl_xor_sync(0xFFFFFFFFu, hits, off);
    if ((threadIdx.x & 31) == 0 && hits) atomicAdd(&s_hits, (unsigned long long)hits);
    int c = tk.finish();
    uint64_t* out = partial + (size_t)blockIdx.x * k;
    for (int i = threadIdx.x; i < k; i += blockDim.x) out[i] = i < c ? tk_buf[i] : 0;
    if (threadIdx.x == 0 && s_hits) atomicAdd(total, s_hits);
}

// Per query: top-k of n_in date keys (0 = empty) -> (doc, seconds) and the count.  dynamic smem: cap * 8.
__global__ void date_merge_kernel(const uint64_t* __restrict__ keys_in, int n_in, int k, int cap, const int64_t* __restrict__ secs, uint32_t* __restrict__ out_docs,
                                  int64_t* __restrict__ out_dates, int* __restrict__ out_counts) {
    extern __shared__ __align__(16) uint64_t tk_buf[];
    __shared__ int tk_count;
    __shared__ uint64_t tk_thr;
    const int q = blockIdx.x;
    BlockTopK tk;
    tk.init(tk_buf, &tk_count, &tk_thr, k, cap);
    const uint64_t* in = keys_in + (size_t)q * n_in;
    for (int base = 0; base < n_in; base += blockDim.x) {
        int i = base + threadIdx.x;
        tk.offer(i < n_in ? in[i] : 0);
    }
    int c = tk.finish();
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        const uint32_t doc = i < c ? key_id(tk_buf[i]) : NIL;
        out_docs[(size_t)q * k + i] = doc;
        out_dates[(size_t)q * k + i] = i < c ? secs[doc] : DATE_NONE;
    }
    if (threadIdx.x == 0) out_counts[q] = c;
}

__host__ __device__ __forceinline__ size_t bm_smem_bytes(int cap, bool conj) {
    return (size_t)cap * 8 + 2 * BM_MAX_TERMS * 8 /* run start */ + BM_WORDS * 4 /* bitmap */ + BM_ACC * 4 /* acc */ + BM_ACC * 4 /* candidates */ +
           2 * BM_MAX_TERMS * 4 /* run length */ + BM_MAX_TERMS * 4 /* weights */ + 1024 /* norm / ratio table */ + BM_WORDS * 2 /* rank bases */ +
           2 * (BM_MAX_TERMS + 2) * 4 /* octet prefix */ + 2 * BM_OCT /* octet -> run */ + (conj ? BM_ACC : 0) /* byte counters */ + 16 +
           4 * BM_MAX_TERMS * 8 /* term state */ + 64;
}

__device__ __forceinline__ uint2 ldg_post(const uint2* p) {
    uint2 r;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u32 {%0, %1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}

// CONJ: nidx_text (all terms must match).  TF: real term frequencies (else IndexRecordOption::Basic, tf == 1).
// FACET: the FacetCollector runs beside Count on the same matched documents (bm25_facet_kernel); with FACET false every facet
// statement compiles away and bm25_kernel is the search without facets.
// ORDER: TopDocs orders by date instead of score (bm25_order_kernel): every matched document -- the set Count counts -- is offered
// with its date key (OrderArgs) instead of a score key.  No score is computed: OR skips phase C and walks the tile bitmap AND alive
// after phase S instead (phase O); AND keeps phase C's conjunction counters only.  min_score and search-after do not apply.  With
// ORDER false every order statement compiles away.
template <bool CONJ, bool TF, bool FACET, bool ORDER>
__device__ __forceinline__ void bm25_body(const TxtDev& T, const Bm25Args& a, const FacetArgs& F, const OrderArgs& O) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int tk_count;
    __shared__ uint64_t tk_thr;
    __shared__ int s_ncand, s_tk_snapshot, s_noct[2], s_ptile[2], s_minlen[2], s_ndistinct, s_shift;
    __shared__ uint32_t s_wsum[BM_WARPS];
    __shared__ unsigned long long s_hits;
    unsigned char* p = smem;
    uint64_t* tk_buf = reinterpret_cast<uint64_t*>(p); p += (size_t)a.cap * 8;
    uint64_t* run_b = reinterpret_cast<uint64_t*>(p); p += 2 * BM_MAX_TERMS * 8;       // [2][terms] first posting of the tile (absolute)
    uint32_t* bitmap = reinterpret_cast<uint32_t*>(p); p += BM_WORDS * 4;              // touched documents of the tile
    uint32_t* acc = reinterpret_cast<uint32_t*>(p); p += BM_ACC * 4;                   // fixed-point sums by rank
    uint32_t* cand = reinterpret_cast<uint32_t*>(p); p += BM_ACC * 4;                  // rank << 17 | tile-relative document
    uint32_t* run_len = reinterpret_cast<uint32_t*>(p); p += 2 * BM_MAX_TERMS * 4;     // [2][terms]
    float* tw = reinterpret_cast<float*>(p); p += BM_MAX_TERMS * 4;
    float* ntab = reinterpret_cast<float*>(p); p += 1024;                              // TF: norm cache; else 1 / (1 + norm) per fieldnorm id
    unsigned short* base = reinterpret_cast<unsigned short*>(p); p += BM_WORDS * 2;    // rank of the first set bit of every bitmap word
    uint32_t* pre8 = reinterpret_cast<uint32_t*>(p); p += 2 * (BM_MAX_TERMS + 2) * 4;   // [2][terms + 1] exclusive prefix of the runs' octet counts
    unsigned char* omap = p; p += 2 * BM_OCT;                                          // [2][BM_OCT] run of every octet
    uint32_t* cnts = reinterpret_cast<uint32_t*>(p); if (CONJ) p += BM_ACC;            // matched-term counters, one BYTE per rank (AND only)
    p = smem + (((size_t)(p - smem) + 15) & ~(size_t)15);
    // per-term state of the resolving warp (kept out of the registers: every thread would pay for them)
    uint64_t* t_base = reinterpret_cast<uint64_t*>(p); p += BM_MAX_TERMS * 8;          // post_addr of the term's first posting
    uint64_t* t_end = reinterpret_cast<uint64_t*>(p); p += BM_MAX_TERMS * 8;           // post_addr past its last
    uint64_t* t_cur = reinterpret_cast<uint64_t*>(p); p += BM_MAX_TERMS * 8;           // first posting not yet assigned to a tile
    uint64_t* t_skip = reinterpret_cast<uint64_t*>(p);                                 // address of the term's skip row, 0 = none
    const int q = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t* fcnt = nullptr;   // FACET: this query's bucket counts (shared memory past the term state, or its row of F.out)
    if (FACET) {
        fcnt = F.smem ? reinterpret_cast<uint32_t*>(t_skip + BM_MAX_TERMS) : F.out + (size_t)q * F.n_buckets;
        if (F.smem) for (uint32_t i = threadIdx.x; i < F.n_buckets; i += BM_THREADS) fcnt[i] = 0;
    }

    const uint32_t* terms = a.query_terms + a.query_off[q];
    const int n_real = (int)(a.query_off[q + 1] - a.query_off[q]);   // the clauses from n_real on are phrases
    const uint32_t ph0 = a.ph_qoff ? a.ph_qoff[q] : 0u;
    int nt = n_real + (a.ph_qoff ? (int)(a.ph_qoff[q + 1] - ph0) : 0);
    if (nt > BM_MAX_TERMS) nt = BM_MAX_TERMS;
    BlockTopK tk;
    tk.init(tk_buf, &tk_count, &tk_thr, a.k, a.cap);
    for (int i = threadIdx.x; i < 256; i += blockDim.x) {
        float nc = a.norm_cache[i];
        ntab[i] = TF ? nc : __fdiv_rn(1.0f, __fadd_rn(1.0f, nc));   // tf == 1: tf / (tf + norm), the same two roundings as the division per posting
    }
    for (int i = threadIdx.x; i < BM_WORDS; i += blockDim.x) bitmap[i] = 0;
    for (int i = threadIdx.x; i < BM_ACC; i += blockDim.x) { acc[i] = 0; if (CONJ && i < BM_ACC / 4) cnts[i] = 0; }

    // ---- warp 0 owns the terms: lane l handles terms l, l + 32, ...; only the prefetched skip entries live in registers ----
    uint32_t t_pf[BM_TPL];
    bool missing = false;
    unsigned long long my_total = 0;
    float wmax = 0.0f;   // the query's largest term weight (unknown terms weigh 0): it sets the query's fixed-point scale
#pragma unroll
    for (int j = 0; j < BM_TPL; ++j) t_pf[j] = 0;
    if (warp == 0) {
#pragma unroll
        for (int j = 0; j < BM_TPL; ++j) {
            int i = lane + 32 * j;
            if (i < nt) {
                uint64_t b, e;
                float w;
                const uint32_t* sk = nullptr;
                if (i < n_real) {
                    uint32_t t = terms[i];
                    bool ok = t < T.n_terms;
                    b = post_addr(T.post) + (ok ? T.term_off[t] : 0);
                    e = post_addr(T.post) + (ok ? T.term_off[t + 1] : 0);
                    w = ok ? a.term_weight[t] : 0.0f;
                    uint32_t row = ok ? T.skip_row[t] : NIL;
                    if (row != NIL) sk = T.skip + (uint64_t)row * (T.n_fine + 1);
                } else {
                    const uint32_t v = ph0 + (uint32_t)(i - n_real);
                    b = post_addr(a.ph_post) + a.ph_range[2 * v];
                    e = post_addr(a.ph_post) + a.ph_range[2 * v + 1];
                    w = a.ph_weight[v];
                    uint32_t row = a.ph_skip_row[v];
                    if (row != NIL) sk = a.ph_skip + (uint64_t)row * (T.n_fine + 1);
                }
                t_base[i] = b; t_end[i] = e; t_cur[i] = b;
                tw[i] = w;   // scaled by 2^shift below (exact: a power of two), so a posting costs one multiply
                if (!ORDER) wmax = fmaxf(wmax, w);
                t_skip[i] = (uint64_t)reinterpret_cast<uintptr_t>(sk);
                missing |= b == e;
                my_total += e - b;
            }
        }
        for (int off = 16; off >= 1; off >>= 1) my_total += __shfl_xor_sync(0xFFFFFFFFu, my_total, off);
        if (!ORDER) for (int off = 16; off >= 1; off >>= 1) wmax = fmaxf(wmax, __shfl_xor_sync(0xFFFFFFFFu, wmax, off));
    }
    if (threadIdx.x == 0) {
        s_hits = 0; s_ncand = 0; s_tk_snapshot = 0; s_ptile[0] = (int)min(my_total, (unsigned long long)INT_MAX);
        if (!ORDER) {   // fixed-point scale: a sum is at most nt * wmax * 2^s + nt / 2 (frac <= 1), kept below 4e9 < 2^32
            const float bound = fmaxf(1.0f, __fmul_rn((float)nt, wmax));
            int s = 24;
            while (s > 4 && __fmul_rn(bound, (float)(1u << s)) >= 4.0e9f) --s;
            s_shift = s;
        }
    }
    int any_missing = __syncthreads_or(missing);   // an AND query with a term without postings matches nothing
    const bool dead = (CONJ && any_missing) || nt == 0;
    const float scale = ORDER ? 1.0f : (float)(1u << s_shift);
    if (threadIdx.x < nt) {   // rn(rn(w * frac) * 2^s) == rn((w * 2^s) * frac)
        const float ws = __fmul_rn(tw[threadIdx.x], scale);
        tw[threadIdx.x] = TF && a.basic_terms && (int)threadIdx.x < n_real ? -ws : ws;   // a negative weight marks a Basic term
    }
    const uint32_t n_fine = dead ? 0 : T.n_fine;
    // tile span (fine tiles): the query's postings spread evenly would fill ~80 % of the slots per tile (octet padding takes some)
    uint32_t m = 1;
    {
        unsigned long long P = (unsigned long long)(unsigned)s_ptile[0];
        unsigned long long nf = n_fine ? n_fine : 1, mm = P ? (unsigned long long)(BM_SLOTS * 4 / 5) * nf / P : nf;
        if (mm < 1) mm = 1;
        if (mm > BM_MAX_SPAN) mm = BM_MAX_SPAN;
        if (mm > nf) mm = nf;
        m = (uint32_t)mm;
    }
    __syncthreads();

    // resolve(f1, buf) by warp 0: slices of every term in fine tiles [cursor position, f1) -> run_b / run_len / pre8 / omap of `buf`
    auto resolve = [&](uint32_t f1, uint32_t m_next, int buf) {
        uint32_t hi = (uint64_t)f1 * BM_FINE < T.n_docs ? f1 * BM_FINE : T.n_docs;
        uint32_t run = 0;
        int mn = INT_MAX, tot = 0;
#pragma unroll
        for (int j = 0; j < BM_TPL; ++j) {
            if (32 * j >= nt) break;            // (uniform) a 50-term query needs two of the four term groups
            int i = lane + 32 * j;
            uint32_t len = 0;
            if (i < nt) {
                uint64_t bgn = t_cur[i], end;
                if (t_skip[i] != 0) {
                    end = t_base[i] + t_pf[j];
                } else {                                                   // rare term: a few postings in total
                    uint64_t l = bgn, e = t_end[i];
                    while (l < e && post_at(l)->x < hi) ++l;
                    end = l;
                }
                run_b[buf * BM_MAX_TERMS + i] = bgn;
                len = (uint32_t)(end - bgn);
                run_len[buf * BM_MAX_TERMS + i] = len;
                t_cur[i] = end;
                mn = min(mn, (int)len);
                tot += (int)len;
            }
            // exclusive scan of the octet counts over the terms (term order = lane + 32 j: scan lanes, then carry `run`)
            uint32_t c = (len + 7) >> 3, x = c;
            for (int off = 1; off < 32; off <<= 1) { uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, off); if (lane >= off) x += y; }
            uint32_t first = run + x - c;
            if (i < nt) pre8[buf * (BM_MAX_TERMS + 2) + i] = first;
            run += __shfl_sync(0xFFFFFFFFu, x, 31);
        }
        for (int off = 16; off >= 1; off >>= 1) { mn = min(mn, __shfl_xor_sync(0xFFFFFFFFu, mn, off)); tot += __shfl_xor_sync(0xFFFFFFFFu, tot, off); }
        if (lane == 0) { pre8[buf * (BM_MAX_TERMS + 2) + nt] = run; s_noct[buf] = (int)run; s_ptile[buf] = tot; s_minlen[buf] = mn; }
        // request the skip entries of the tile after this one
        uint32_t f2 = f1 + m_next < T.n_fine ? f1 + m_next : T.n_fine;
#pragma unroll
        for (int j = 0; j < BM_TPL; ++j) { int i = lane + 32 * j; if (i < nt && t_skip[i] != 0) t_pf[j] = __ldg(reinterpret_cast<const uint32_t*>(t_skip[i]) + f2); }
    };
    auto load_pf = [&](uint32_t f1) {   // synchronous (re)load of the skip entries for boundary f1
#pragma unroll
        for (int j = 0; j < BM_TPL; ++j) { int i = lane + 32 * j; if (i < nt && t_skip[i] != 0) t_pf[j] = __ldg(reinterpret_cast<const uint32_t*>(t_skip[i]) + f1); }
    };

    // omap[o] = run of octet o (last run with pre8[r] <= o), two octets per thread; pre8 of `b` must be complete (barrier)
    auto fill_omap = [&](int b) {
        const uint32_t* pr = pre8 + b * (BM_MAX_TERMS + 2);
        int total = min((int)pr[nt], BM_OCT);
        for (int o = threadIdx.x; o < total; o += BM_THREADS) {
            int l2 = 0, h2 = nt - 1;
            while (l2 < h2) { int mid = (l2 + h2 + 1) >> 1; if ((int)pr[mid] <= o) l2 = mid; else h2 = mid - 1; }
            omap[b * BM_OCT + o] = (unsigned char)l2;
        }
    };

    uint32_t thr_fx = 1;   // sums >= thr_fx may still enter the top-k (1 = everything that is touched)
    unsigned int my_hits = 0;
    // a candidate -> top-k buffer (final sum; exact threshold, alive, search-after)
    auto offer_cand = [&](uint32_t cd, uint32_t lo) {
        uint32_t v = acc[cd >> 17], doc = lo + (cd & 0x1FFFFu);
        bool match = true;
        if (T.alive) match = (T.alive[doc >> 6] >> (doc & 63)) & 1;
        if (CONJ && match) my_hits++;
        if (FACET && CONJ && match) facet_doc(F, doc, fcnt);   // AND: every completed conjunction is a candidate
        if (ORDER) {
            if (match) {
                const uint64_t key = order_key(O, doc);
                if (key > tk_thr) tk_buf[atomicAdd(&tk_count, 1)] = key;
            }
        } else if (match) {
            float score = __fdiv_rn((float)v, scale);
            bool after = true;   // is_after(): strictly lower score, or an equal score that the tie break keeps
            if (a.after_mode != 0) {
                uint32_t so = ordered_bits(score), ao = ordered_bits(a.after_score);
                after = so < ao || (so == ao && (a.after_mode == 3 || (a.after_mode == 2 && a.docaddr_base + doc > a.after_docaddr)));
            }
            uint64_t key = make_key(score, doc, 0);
            if (after && key > tk_thr) tk_buf[atomicAdd(&tk_count, 1)] = key;
        }
    };

    uint32_t f0 = 0;
    int buf = 0;
    if (n_fine) {
        if (warp == 0) { load_pf(min(m, n_fine)); resolve(min(m, n_fine), m, 0); }
        __syncthreads();
        fill_omap(0);
        __syncthreads();
    }
    while (f0 < n_fine) {
        uint32_t f1 = min(f0 + m, n_fine);
        if (f1 - f0 > 1 && (s_ptile[buf] > BM_ACC || s_noct[buf] > BM_OCT)) {   // (uniform) does not fit one round: redo from f0 with half the span
            __syncthreads();
            m = m / 2 > 1 ? m / 2 : 1;
            if (warp == 0) {
#pragma unroll
                for (int j = 0; j < BM_TPL; ++j) { int i = lane + 32 * j; if (i < nt) t_cur[i] = run_b[buf * BM_MAX_TERMS + i]; }
                load_pf(min(f0 + m, n_fine));
                resolve(min(f0 + m, n_fine), m, buf);
            }
            __syncthreads();
            fill_omap(buf);
            __syncthreads();
            continue;
        }
        const uint32_t lo = f0 * BM_FINE;
        const uint32_t docs_t = (f1 * BM_FINE < T.n_docs ? f1 * BM_FINE : T.n_docs) - lo;
        const int nwords = (int)((docs_t + 31) >> 5);
        const bool skip_tile = s_ptile[buf] == 0 || (CONJ && s_minlen[buf] == 0);   // AND: some term has nothing in this tile
        if (!skip_tile) {
            const int noct = s_noct[buf];
            const int nrounds = (noct + BM_OCT - 1) / BM_OCT;
            const bool one_round = nrounds == 1;
            const uint32_t* pr8 = pre8 + buf * (BM_MAX_TERMS + 2);
            uint2 pd[BM_PT];
            uint32_t rpack[BM_PT / 4];
            uint32_t actm = 0;
            // the slots of this thread in `round`: slot = round * BM_SLOTS + u * BM_THREADS + tid
            auto load_round = [&](int round) {
                actm = 0;
#pragma unroll
                for (int u = 0; u < BM_PT; ++u) {
                    if ((u & 3) == 0) rpack[u >> 2] = 0;
                    int s = round * BM_SLOTS + u * BM_THREADS + (int)threadIdx.x;
                    int o = s >> 3;
                    pd[u] = make_uint2(0, 0);
                    if (o < noct) {
                        int r;
                        if (one_round) r = omap[buf * BM_OCT + o];
                        else {   // dense tile: last run with pre8[r] <= o
                            int l2 = 0, h2 = nt - 1;
                            while (l2 < h2) { int mid = (l2 + h2 + 1) >> 1; if ((int)pr8[mid] <= o) l2 = mid; else h2 = mid - 1; }
                            r = l2;
                        }
                        uint32_t within = (uint32_t)(o - (int)pr8[r]) * 8u + (uint32_t)(s & 7);
                        if (within < run_len[buf * BM_MAX_TERMS + r]) {
                            actm |= 1u << u;
                            rpack[u >> 2] |= (uint32_t)r << (8 * (u & 3));
                            pd[u] = ldg_post(post_at(run_b[buf * BM_MAX_TERMS + r] + within));
                        }
                    }
                }
            };
            // ---- phase A: request everything, mark the touched documents ----
            for (int round = 0; round < nrounds; ++round) {
                load_round(round);
#pragma unroll
                for (int u = 0; u < BM_PT; ++u)
                    if (actm & (1u << u)) { uint32_t off = pd[u].x - lo; atomicOr(&bitmap[off >> 5], 1u << (off & 31)); }
            }
            __syncthreads();
            // ---- phase S: rank base of every bitmap word (exclusive prefix popcount); Count collector ----
            {
                constexpr int WPT = BM_WORDS / BM_THREADS;   // consecutive words per thread (a multiple of 8), read twice (registers hold the postings)
                const int w0 = (int)threadIdx.x * WPT;
                const bool mine = w0 < nwords;
                uint32_t sum = 0;
                if (mine) {
                    const uint32_t* al = T.alive ? reinterpret_cast<const uint32_t*>(T.alive) + (lo >> 5) + w0 : nullptr;
                    uint32_t hits = 0;
#pragma unroll
                    for (int i = 0; i < WPT; i += 4) {
                        uint4 v = *reinterpret_cast<const uint4*>(bitmap + w0 + i);
                        sum += __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w);
                        if (!CONJ && al) {   // a word is read only where the tile has documents: the alive array ends with the documents
                            if (v.x) hits += __popc(v.x & al[i]);
                            if (v.y) hits += __popc(v.y & al[i + 1]);
                            if (v.z) hits += __popc(v.z & al[i + 2]);
                            if (v.w) hits += __popc(v.w & al[i + 3]);
                        }
                    }
                    if (!CONJ) my_hits += al ? hits : sum;
                }
                uint32_t x = sum;
                for (int off = 1; off < 32; off <<= 1) { uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, off); if (lane >= off) x += y; }
                if (lane == 31) s_wsum[warp] = x;
                __syncthreads();
                uint32_t pre = x - sum;
                for (int ww = 0; ww < warp; ++ww) pre += s_wsum[ww];
                if (threadIdx.x == BM_THREADS - 1) s_ndistinct = (int)(pre + sum);
                if (mine) {
#pragma unroll
                    for (int i = 0; i < WPT; i += 8) {
                        uint4 v0 = *reinterpret_cast<const uint4*>(bitmap + w0 + i), v1 = *reinterpret_cast<const uint4*>(bitmap + w0 + i + 4);
                        uint32_t b0 = pre; pre += __popc(v0.x);
                        uint32_t b1 = pre; pre += __popc(v0.y);
                        uint32_t b2 = pre; pre += __popc(v0.z);
                        uint32_t b3 = pre; pre += __popc(v0.w);
                        uint32_t b4 = pre; pre += __popc(v1.x);
                        uint32_t b5 = pre; pre += __popc(v1.y);
                        uint32_t b6 = pre; pre += __popc(v1.z);
                        uint32_t b7 = pre; pre += __popc(v1.w);
                        *reinterpret_cast<uint4*>(base + w0 + i) = make_uint4(b0 | (b1 << 16), b2 | (b3 << 16), b4 | (b5 << 16), b6 | (b7 << 16));
                    }
                }
            }
            __syncthreads();
            // ---- phase C: score and accumulate by rank ----
            // All of a thread's postings are scored and added first (independent chains: the loads of the bitmap word, the rank
            // base, the weight and the norm entry of different postings overlap); which adds crossed the threshold is kept in a
            // per-thread mask and the candidates are appended afterwards -- a warp vote per posting only where some lane has one
            // (rare once the top-k threshold is established).
            // ORDER: no scores; AND keeps the conjunction counters, OR has nothing to do here (phase O below).
            for (int round = 0; round < (ORDER && !CONJ ? 0 : nrounds); ++round) {
                if (!one_round) load_round(round);
                uint32_t cmask = 0;
                uint32_t cds[BM_PT];
#pragma unroll
                for (int u = 0; u < BM_PT; ++u) {
                    cds[u] = 0;
                    if (actm & (1u << u)) {
                        uint32_t off = pd[u].x - lo, tfn = pd[u].y;
                        uint32_t wd = bitmap[off >> 5];
                        uint32_t rank = (uint32_t)base[off >> 5] + __popc(wd & ((1u << (off & 31)) - 1u));
                        bool crossed;
                        if (ORDER) {
                            if (CONJ) {
                                uint32_t oldw = atomicAdd(&cnts[rank >> 2], 1u << (8 * (rank & 3)));
                                crossed = (int)(((oldw >> (8 * (rank & 3))) & 0xFFu) + 1) == nt;
                            } else {
                                crossed = false;
                            }
                        } else {
                            float wgt = tw[(rpack[u >> 2] >> (8 * (u & 3))) & 0xFFu];
                            float frac;
                            if (TF) {
                                float tff = (float)(tfn >> 8);
                                if (wgt < 0.0f) { tff = 1.0f; wgt = -wgt; }   // a Basic term beside phrases (a.basic_terms)
                                frac = __fdiv_rn(tff, __fadd_rn(tff, ntab[tfn & 0xFFu]));
                            } else frac = ntab[tfn & 0xFFu];
                            uint32_t fx = (uint32_t)__float2uint_rn(__fmul_rn(wgt, frac));
                            if (fx == 0) fx = 1;
                            uint32_t oldv = atomicAdd(&acc[rank], fx);
                            if (CONJ) {
                                uint32_t oldw = atomicAdd(&cnts[rank >> 2], 1u << (8 * (rank & 3)));   // byte counter (nt <= 128) inside its 32-bit word
                                crossed = (int)(((oldw >> (8 * (rank & 3))) & 0xFFu) + 1) == nt;       // the posting that completes the conjunction hands the document on
                            } else {
                                crossed = oldv < thr_fx && oldv + fx >= thr_fx;
                            }
                        }
                        cds[u] = (rank << 17) | off;
                        if (crossed) cmask |= 1u << u;
                    }
                }
                if (__any_sync(0xFFFFFFFFu, cmask != 0)) {
#pragma unroll
                    for (int u = 0; u < BM_PT; ++u) {
                        const bool crossed = (cmask >> u) & 1u;
                        unsigned mk = __ballot_sync(0xFFFFFFFFu, crossed);
                        if (mk) {
                            int basepos = 0;
                            if (lane == 0) basepos = atomicAdd(&s_ncand, __popc(mk));
                            basepos = __shfl_sync(0xFFFFFFFFu, basepos, 0);
                            if (crossed) cand[basepos + __popc(mk & ((1u << lane) - 1))] = cds[u];
                        }
                    }
                }
            }
            if (FACET && !CONJ) {   // OR: the documents phase S counted (bitmap AND alive), FACET_BATCH at a time per thread
                const uint32_t* al = T.alive ? reinterpret_cast<const uint32_t*>(T.alive) + (lo >> 5) : nullptr;
                int w = (int)threadIdx.x - BM_THREADS;   // this thread's words: threadIdx.x, + BM_THREADS, ...
                uint32_t v = 0;
                for (;;) {
                    uint32_t dd[FACET_BATCH];
#pragma unroll
                    for (int j = 0; j < FACET_BATCH; ++j) {
                        while (v == 0 && w + BM_THREADS < nwords) { w += BM_THREADS; v = bitmap[w]; if (v && al) v &= al[w]; }
                        dd[j] = v ? lo + 32u * (uint32_t)w + (uint32_t)(__ffs(v) - 1) : NIL;
                        v &= v - 1;
                    }
                    if (dd[0] == NIL) break;
                    facet_docs(F, dd, fcnt);
                }
            }
            if (ORDER && !CONJ) {   // phase O: every document phase S counted (bitmap AND alive) whose date key can still enter the top-k
                const uint32_t* al = T.alive ? reinterpret_cast<const uint32_t*>(T.alive) + (lo >> 5) : nullptr;
                for (int w = threadIdx.x; w < nwords; w += BM_THREADS) {
                    uint32_t v = bitmap[w];
                    if (v && al) v &= al[w];
                    while (v) {
                        const uint32_t off = 32u * (uint32_t)w + (uint32_t)(__ffs(v) - 1);
                        v &= v - 1;
                        if (order_key(O, lo + off) > tk_thr) cand[atomicAdd(&s_ncand, 1)] = off;   // a tile holds <= BM_ACC documents
                    }
                }
            }
            __syncthreads();
            // ---- phase D: candidates -> top-k buffer; warp 0 resolves the next tile meanwhile ----
            // The branch below must be uniform: it is taken on the buffer fill recorded at the end of the previous tile
            // (no other phase touches the buffer), never on tk_count itself, which the other warps are already incrementing.
            const int ncand = s_ncand;
            const int room = a.cap - a.k;
            if (s_tk_snapshot + ncand > a.cap) {     // (uniform) rare: the buffer cannot take them all at once -> rounds with a flush each
                for (int b0 = 0; b0 < ncand; b0 += room) {
                    tk.flush();
                    int end = min(ncand, b0 + room);
                    for (int i = b0 + threadIdx.x; i < end; i += BM_THREADS) offer_cand(cand[i], lo);
                    __syncthreads();
                }
                if (ncand > room) tk.flush();        // several rounds (the first tiles): raise the threshold right away
                if (warp == 0 && f1 < n_fine) resolve(min(f1 + m, n_fine), m, buf ^ 1);
            } else if (warp == 0) {
                if (f1 < n_fine) resolve(min(f1 + m, n_fine), m, buf ^ 1);
            } else {
                for (int i = threadIdx.x - 32; i < ncand; i += BM_THREADS - 32) offer_cand(cand[i], lo);
            }
            __syncthreads();
            // ---- reset: bitmap words, used accumulators (and counters) ----
            if (!ORDER && tk_thr != 0) {   // threshold in fixed point, conservative (float(v) is within 2^-24 of v)
                float ts = key_score(tk_thr);
                float lowb = __fmul_rn(__fmul_rn(ts, scale), 0.9999990f);
                thr_fx = lowb >= 1.0f ? (uint32_t)lowb : 1u;
            }
            const uint4 z4 = make_uint4(0, 0, 0, 0);
            const int nd4 = (s_ndistinct + 3) >> 2;
            for (int i = threadIdx.x; i < (nwords + 3) >> 2; i += BM_THREADS) reinterpret_cast<uint4*>(bitmap)[i] = z4;
            if (!ORDER) for (int i = threadIdx.x; i < nd4; i += BM_THREADS) reinterpret_cast<uint4*>(acc)[i] = z4;
            if (CONJ) for (int i = threadIdx.x; i < (nd4 + 3) >> 2; i += BM_THREADS) reinterpret_cast<uint4*>(cnts)[i] = z4;
            if (threadIdx.x == 0) { s_ncand = 0; s_tk_snapshot = tk_count; }
            if (f1 < n_fine) fill_omap(buf ^ 1);   // the next tile's octet map (its prefix was completed before the last barrier)
            __syncthreads();
        } else {
            if (warp == 0 && f1 < n_fine) resolve(min(f1 + m, n_fine), m, buf ^ 1);
            __syncthreads();
            if (f1 < n_fine) fill_omap(buf ^ 1);
            __syncthreads();
        }
        f0 = f1;
        buf ^= 1;
    }
    for (int off = 16; off >= 1; off >>= 1) my_hits += __shfl_xor_sync(0xFFFFFFFFu, my_hits, off);
    if (lane == 0 && my_hits) atomicAdd(&s_hits, (unsigned long long)my_hits);
    int c = tk.finish();
    uint64_t* out = a.out_keys + (size_t)q * a.k;
    for (int i = threadIdx.x; i < a.k; i += blockDim.x) out[i] = i < c ? tk_buf[i] : 0;
    if (threadIdx.x == 0 && a.out_total) a.out_total[q] = s_hits;
    // every tile ends with a barrier, so the shared counts are complete here
    if (FACET && F.smem) for (uint32_t i = threadIdx.x; i < F.n_buckets; i += BM_THREADS) F.out[(size_t)q * F.n_buckets + i] = fcnt[i];
}

template <bool CONJ, bool TF>
__global__ void __launch_bounds__(BM_THREADS, BM_MINB_CFG) bm25_kernel(TxtDev T, Bm25Args a) {
    bm25_body<CONJ, TF, false, false>(T, a, FacetArgs{}, OrderArgs{});
}

// bm25_kernel + the FacetCollector: same top-k and Count, plus F.out[q][bucket] (shared counters: smem = bm_smem_bytes + 4 n_buckets)
template <bool CONJ, bool TF>
__global__ void __launch_bounds__(BM_THREADS, BM_MINB_CFG) bm25_facet_kernel(TxtDev T, Bm25Args a, FacetArgs f) {
    bm25_body<CONJ, TF, true, false>(T, a, f, OrderArgs{});
}

// bm25_kernel ordered by date (TopDocs::order_by_fast_field): same matched set and Count, keys from OrderArgs (no scores, so no TF)
template <bool CONJ>
__global__ void __launch_bounds__(BM_THREADS, BM_MINB_CFG) bm25_order_kernel(TxtDev T, Bm25Args a, OrderArgs o) {
    bm25_body<CONJ, false, false, true>(T, a, FacetArgs{}, o);
}

// bm25_order_kernel + the FacetCollector in the same pass
template <bool CONJ>
__global__ void __launch_bounds__(BM_THREADS, BM_MINB_CFG) bm25_order_facet_kernel(TxtDev T, Bm25Args a, FacetArgs f, OrderArgs o) {
    bm25_body<CONJ, false, true, true>(T, a, f, o);
}

// date keys -> (doc, seconds, count); no min_score under an order (convert_int_order, nidx_text/src/reader.rs:226-287).
__global__ void date_finish_kernel(const uint64_t* keys, int nq, int k, const int64_t* secs, uint32_t* out_docs, int64_t* out_dates, int* out_counts) {
    int q = blockIdx.x;
    __shared__ int s_count;
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        uint64_t key = keys[(size_t)q * k + i];
        uint32_t doc = key != 0 ? key_id(key) : NIL;
        out_docs[(size_t)q * k + i] = doc;
        out_dates[(size_t)q * k + i] = key != 0 ? secs[doc] : DATE_NONE;
        if (key != 0) atomicAdd(&s_count, 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) out_counts[q] = s_count;
}

// keys -> (doc, score, count) with the min_score cut applied after top-k (reader.rs:302-305).
__global__ void bm25_finish_kernel(const uint64_t* keys, int nq, int k, float min_score, uint32_t* out_docs, float* out_scores, int* out_counts) {
    int q = blockIdx.x;
    __shared__ int s_count;
    if (threadIdx.x == 0) s_count = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < k; i += blockDim.x) {
        uint64_t key = keys[(size_t)q * k + i];
        bool ok = key != 0 && !(key_score(key) < min_score);
        out_docs[(size_t)q * k + i] = ok ? key_id(key) : NIL;
        out_scores[(size_t)q * k + i] = ok ? key_score(key) : 0.0f;
        if (ok) atomicAdd(&s_count, 1);
    }
    __syncthreads();
    if (threadIdx.x == 0) out_counts[q] = s_count;
}

}  // namespace nidx
