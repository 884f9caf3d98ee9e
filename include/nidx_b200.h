/* nidx_b200 — C ABI of the H100-native (sm_90a) nidx search hot path (libnidx_b200.so).
 *
 * This is the drop-in boundary: every entry point replaces one Rust interface of the reference
 * (cited per function) and is what a cgo/FFI/ctypes binding on the reference side binds
 * (INTEGRATION.md shows the Rust `extern "C"` block).  Plain pointers and sizes only; the caller
 * owns every buffer it passes, the library owns the handles and all device memory.
 *
 * Conventions
 *   - every function returns 0 on success, a negative NIDX_E* code on failure;
 *     nidx_last_error() returns the message of the calling thread's last failure
 *     (reference: anyhow::Error / VectorErr strings, nidx_vector/src/lib.rs:203-232).
 *   - `mem` arguments say where the caller's buffers live: NIDX_MEM_HOST (the library copies
 *     host<->device inside the call) or NIDX_MEM_DEVICE (pointers are device pointers on the
 *     index's GPU; nothing is copied).  `stream` is a cudaStream_t (NULL = default stream); calls
 *     with NIDX_MEM_DEVICE are asynchronous on it, calls with NIDX_MEM_HOST return after the
 *     results are in the host buffers.
 *   - search entry points are re-entrant: they may be called concurrently from many threads on
 *     one handle (reference: searchers are Sync+Send behind an Arc, index_cache.rs:41-47).
 *   - there is NO CPU fallback: without a CUDA device every call fails with NIDX_ENODEVICE.
 */
#ifndef NIDX_B200_H
#define NIDX_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NIDX_OK 0
#define NIDX_EINVAL (-1)     /* bad argument (VectorErr::InconsistentDimensions, ...) */
#define NIDX_ENODEVICE (-2)  /* no usable CUDA device */
#define NIDX_ECUDA (-3)      /* CUDA runtime error */
#define NIDX_EIO (-4)        /* segment file error */
#define NIDX_ESTATE (-5)     /* e.g. HNSW search on an index without a graph */
#define NIDX_EOVERFLOW (-6)  /* an internal bounded structure overflowed; results incomplete */

#define NIDX_MEM_HOST 0
#define NIDX_MEM_DEVICE 1

#define NIDX_SIM_DOT 0     /* config.rs:33-37 Similarity::Dot */
#define NIDX_SIM_COSINE 1  /* Similarity::Cosine */
#define NIDX_SIM_L2 2      /* extension (north_star): -|a - b|^2 as a similarity; the reference has no L2 (config.rs:33-37), so parity is
                              against the oracle's restatement and a float64 brute force only */

#define NIDX_METHOD_AUTO 0   /* segment.rs:538 use_hnsw() cost model decides */
#define NIDX_METHOD_HNSW 1   /* hnsw/search.rs:306-383 */
#define NIDX_METHOD_BRUTE 2  /* segment.rs:569-623 */
#define NIDX_METHOD_BRUTE_RABITQ 3 /* segment.rs:581-608 with a RaBitQ query: quantised scan + exact rerank (rabitq.rs:222-244) */
#define NIDX_METHOD_HNSW_RABITQ 4  /* hnsw/search.rs:306-383 with a RaBitQ query: the walk ranks by the estimate, layer 0 returns
                                      min(100 k, 2000) nodes, rerank_top + closest_up_nodes on exact similarities.  What AUTO takes
                                      when the segment carries codes (segment.rs:506-513) and the cost model picks the graph */

#define NIDX_NIL 0xFFFFFFFFu

const char* nidx_last_error(void);
/* Number of CUDA devices the library can use (0 => every other call fails). */
int nidx_device_count(void);
/* Kernel launches issued by this process through the library (bench.py's gpu_launches). */
uint64_t nidx_launch_count(void);

/* ------------------------------------------------------------------------------------------
 * Vector segment  (reference: nidx_vector OpenSegment + VectorConfig, segment.rs / config.rs)
 * ------------------------------------------------------------------------------------------ */
typedef struct nidx_vec_segment nidx_vec_segment;

typedef struct nidx_vec_config {
    int32_t dimension;        /* VectorType::DenseF32{dimension}, config.rs:102-124 */
    int32_t similarity;       /* NIDX_SIM_* */
    int32_t multi_vector;     /* VectorCardinality::Multi: one result per paragraph */
    int32_t m;                /* params.rs:40 M (also M_MAX);   0 => 30 */
    int32_t m0;               /* params.rs:34 M_MAX_0;          0 => 60 */
    int32_t ef_construction;  /* params.rs:43;                  0 => 100 */
    int32_t ef_search;        /* params.rs:46;                  0 => 30 */
    int32_t device;           /* CUDA device ordinal */
} nidx_vec_config;

/* segment::create's data-store half (segment.rs:199-239, data_store/v2.rs:54-80): take n vectors
 * ([n][ld] f32, ld >= dimension) and, optionally, the paragraph address of every vector
 * (vectors of one paragraph must be contiguous; NULL = one vector per paragraph).  Vectors are
 * re-laid out in HBM as [n][ld4] rows (16-byte aligned) and their norms are precomputed.
 * No graph yet: brute force works, HNSW needs nidx_vec_build_hnsw or nidx_vec_set_graph. */
int nidx_vec_create(const nidx_vec_config* cfg, const float* vectors, uint64_t n, int32_t ld, int mem, const uint32_t* paragraph_of,
                    nidx_vec_segment** out);

/* Open a segment directory written by the reference (or by nidx_vec_save): vectors.bin
 * (data_store/v2/vector_store.rs:33-68) + hnsw.graph (hnsw/disk/v2.rs:16-49) [+ hnsw.edges].
 * Replaces segment::open (segment.rs:39-90) for the hot path's needs. */
int nidx_vec_open(const nidx_vec_config* cfg, const char* dir, nidx_vec_segment** out);
/* Write vectors.bin / hnsw.graph / hnsw.edges in the reference's formats (DiskHnswV2::serialize_to,
 * hnsw/disk/v2.rs:213-218; VectorStoreWriter, vector_store.rs:113-146). */
int nidx_vec_save(nidx_vec_segment* seg, const char* dir);
void nidx_vec_close(nidx_vec_segment* seg);

uint64_t nidx_vec_len(const nidx_vec_segment* seg);
/* Device pointers of the resident data, for zero-copy consumers (bench, tests). */
const float* nidx_vec_device_vectors(const nidx_vec_segment* seg, int32_t* ld_out);

/* HnswBuilder (hnsw/build.rs:36-166) on the GPU: levels for all nodes first (initialize_graph),
 * then batch-synchronous insertion (DESIGN.md "build"): batches of at most max_batch nodes search
 * the frozen graph and are linked in ascending id.  seed: level RNG seed (reference uses 2). */
int nidx_vec_build_hnsw(nidx_vec_segment* seg, uint64_t seed, int32_t max_batch, void* stream);

/* The top layer of every node as HnswBuilder::initialize_graph draws them (build.rs:40,49-55,97-101: SmallRng seeded with
 * `seed` (the reference uses 2), level = round(-ln(u) / ln(M))), capped at the library's layer limit.  nidx_vec_build_hnsw uses
 * exactly these.  Pure host function: needs no device. */
int nidx_hnsw_levels(uint64_t n, int32_t m, uint64_t seed, uint8_t* out_level);

/* utils::normalize_vector (nidx_vector/src/utils.rs:20-23) for n rows of d floats ([n][ld], in place): x / sqrt(fold(acc + x*x)),
 * the fold sequential in f32 exactly as the reference's iterator (bit-identical results).  Used at index time when
 * VectorConfig.normalize_vectors is set (indexer.rs:94-146) and on the query (searcher.rs:246-252).  mem = NIDX_MEM_HOST copies
 * in and out and waits; NIDX_MEM_DEVICE works in place on `stream`. */
int nidx_normalize_vectors(int32_t device, float* vectors, uint64_t n, int32_t d, int32_t ld, int mem, void* stream);

/* The planner's cost model (use_hnsw, segment.rs:626-660): 1 if the HNSW walk is estimated cheaper than the exhaustive scan
 * for `matching_nodes` of `total_nodes` paragraphs passing the filter.  has_rabitq = the segment carries 1-bit codes.  m = the
 * graph's M (the reference's compile-time hnsw::M = 30).  Pure host function: needs no device.  nidx_vec_search applies it for
 * NIDX_METHOD_AUTO. */
int nidx_use_hnsw(uint64_t total_nodes, uint64_t matching_nodes, uint64_t top_k, int has_rabitq, int m);

/* merge_indexes' fast path (segment.rs:143-167): the first n_existing vectors of this segment already have a graph
 * (the largest input segment of a merge, without deletions) given in the flat layout below for n_existing nodes; only the
 * remaining vectors are inserted.  Levels of the new nodes come from a fresh RNG (HnswBuilder::new + initialize_graph with
 * skip_nodes = n_existing, build.rs:36-55); the entry point moves only if a higher layer appears (ram_hnsw.rs:99-107).
 * The edge similarities (w0, wU: the contents of hnsw.edges) are required -- the reverse-link prune ranks by them.  Links
 * in a layer > 0 to a node that is not in that layer are dropped first (fix_broken_graph, ram_hnsw.rs:118-123). */
int nidx_vec_extend_hnsw(nidx_vec_segment* seg, uint64_t n_existing, const uint8_t* level_existing, const uint32_t* adj0, const float* w0,
                         const uint32_t* adjU, const float* wU, uint32_t entry_node, uint32_t entry_layer, uint64_t seed, int32_t max_batch,
                         void* stream);

/* Flat graph import / export (the layout in DESIGN.md; the oracle uses the same one).
 * level[n] u8; adj0[n][s0] u32, adjU[rows][su] u32, NIDX_NIL padded; w0/wU edge similarities
 * (may be NULL on import: search does not need them, merge/build does). Host pointers. */
int nidx_vec_graph_dims(const nidx_vec_segment* seg, int32_t* s0, int32_t* su, uint64_t* upper_rows, uint32_t* entry_node,
                        uint32_t* entry_layer);
int nidx_vec_set_graph(nidx_vec_segment* seg, const uint8_t* level, const uint32_t* adj0, const float* w0, const uint32_t* adjU,
                       const float* wU);
int nidx_vec_get_graph(const nidx_vec_segment* seg, uint8_t* level, uint32_t* adj0, float* w0, uint32_t* adjU, float* wU);

/* OpenSegment::apply_deletions (segment.rs:428-445): bit per paragraph, 1 = alive; NULL = all alive. */
int nidx_vec_set_alive(nidx_vec_segment* seg, const uint64_t* alive_bits, int mem);

typedef struct nidx_vec_search_params {
    int32_t k;                /* VectorSearchRequest.result_per_page (request_types.rs:18-35) */
    int32_t ef;               /* layer-0 width = max(k, ef) (hnsw/search.rs:338-345); 0 => config */
    float min_score;          /* VectorSearchRequest.min_score */
    int32_t with_duplicates;  /* VectorSearchRequest.with_duplicates */
    int32_t method;           /* NIDX_METHOD_* */
    const uint64_t* filter_bits; /* filter formula evaluated to a bitset over paragraphs
                                    (segment.rs:516-534); NULL = no filter. Same `mem` as queries. */
    uint64_t filter_matching; /* number of set bits in filter_bits ∧ alive (segment.rs:531), only read
                                 by the NIDX_METHOD_AUTO cost model; 0 = unknown (count on device) */
} nidx_vec_search_params;

/* OpenSegment::search (segment.rs:477-567) for a batch of nq queries ([nq][ldq] f32).
 * out_ids/out_scores are [nq][k] (vector address + similarity, descending; NIDX_NIL padded),
 * out_counts[nq] the number of valid results per query. */
int nidx_vec_search(nidx_vec_segment* seg, const float* queries, int32_t nq, int32_t ldq, int mem, const nidx_vec_search_params* p,
                    uint32_t* out_ids, float* out_scores, int32_t* out_counts, void* stream);

/* ------------------------------------------------------------------------------------------
 * Filters on the device (reference: ParagraphInvertedIndexes, inverted_index/paragraph.rs:39-186 over fst_index.rs + map.rs)
 * ------------------------------------------------------------------------------------------ */
#define NIDX_INV_LABELS 0  /* label index: key = labels_key(label) (paragraph.rs:64-66), looked up by PREFIX (get_prefix) */
#define NIDX_INV_FIELDS 1  /* field index: key = FieldKey bytes (utils.rs:80-117), looked up EXACTLY (get) */
/* One inverted index of the segment: n_keys byte strings, strictly ascending in memcmp order (the fst's order), key i =
 * key_bytes[key_off[i] .. key_off[i + 1]), its paragraph addresses = postings[post_off[i] .. post_off[i + 1]).  The keys stay on the
 * host side of the library (the lookup is the fst's job: a binary search), the postings live in HBM.  Host pointers.  A call that
 * fails (rejected input included) leaves the segment's previous index in place. */
int nidx_vec_set_inverted_index(nidx_vec_segment* seg, int32_t which, uint32_t n_keys, const uint8_t* key_bytes, const uint64_t* key_off,
                                const uint64_t* post_off, const uint32_t* postings);

#define NIDX_F_LABEL 0  /* AtomClause::Label: n = 1 key, every label key that starts with it (formula.rs:21, paragraph.rs:140-142) */
#define NIDX_F_KEYS 1   /* AtomClause::KeyPrefixSet: n field keys, each looked up exactly (paragraph.rs:143-147) */
#define NIDX_F_AND 2    /* CompoundClause And: intersection of the n operand nodes that follow */
#define NIDX_F_OR 3     /* CompoundClause Or: union */
#define NIDX_F_NOT 4    /* CompoundClause Not: complement of the INTERSECTION of its n operands (paragraph.rs:160-178) */
typedef struct nidx_filter_node {   /* a Formula / Clause tree in pre-order (formula.rs:40-100); a Formula with several clauses is an AND / OR root */
    int32_t kind;                   /* NIDX_F_* */
    int32_t n;                      /* LABEL: 1; KEYS: number of keys; AND / OR / NOT: number of operand subtrees that follow */
    const uint8_t* const* keys;     /* LABEL / KEYS: n byte strings (host pointers) */
    const uint32_t* key_len;
} nidx_filter_node;

/* ParagraphInvertedIndexes::filter + the intersection with the alive set (segment.rs:516-531): the formula's bitset over the
 * paragraphs, computed in HBM (postings -> bits, then one pass of the formula as a program, ANDed with alive and counted).  out_bits
 * (`mem`; (paragraphs + 63) / 64 words) may be NULL; *out_matching = number of set bits (the reference's `bitset.iter().count()`).
 * A formula whose program has more than 4096 instructions is NIDX_EINVAL: the atoms that are operands of one OR are one leaf,
 * and every other atom, and every operand of an AND / OR / NOT after its first, is one instruction (a NOT adds one more). */
int nidx_vec_filter(nidx_vec_segment* seg, const nidx_filter_node* nodes, int32_t n_nodes, uint64_t* out_bits, int mem, uint64_t* out_matching, void* stream);

/* nidx_vec_search with the filter given as a formula: evaluated on the device and fed to the search without a host round trip
 * (p->filter_bits must be NULL; NIDX_METHOD_AUTO reads the match count back, 8 bytes, for the cost model as segment.rs:531 does).
 * The formula has nidx_vec_filter's limit of 4096 instructions. */
int nidx_vec_search_formula(nidx_vec_segment* seg, const float* queries, int32_t nq, int32_t ldq, int mem, const nidx_vec_search_params* p,
                            const nidx_filter_node* nodes, int32_t n_nodes, uint32_t* out_ids, float* out_scores, int32_t* out_counts, void* stream);

/* The text merge: n_parts partial results [n_parts][nq][k] (score desc, NIDX_NIL padded) of the segments of ONE
 * document-partitioned index -> [nq][k] ranked (score desc, part asc, position asc).  Inside one index the parts are segments in
 * docaddr order, so this is merge_document_responses' order (bm25 desc, docaddr asc; shard_merge.rs:211-231) for them.  It is NOT
 * the vector merge: use nidx_merge_vector_parts for vector shards.  out_part[nq][k] receives the index of the part each winner
 * came from.  part_stride = elements between consecutive parts in ids / scores (0 = nq*k, i.e. dense), so an all-gather buffer can
 * be merged in place.  k <= 1024.  Device pointers. */
int nidx_merge_topk(int32_t device, const uint32_t* ids, const float* scores, int32_t n_parts, int64_t part_stride, int32_t nq, int32_t k,
                    uint32_t* out_ids, float* out_scores, int32_t* out_part, void* stream);
/* merge_vector_responses (shard_merge.rs:332-348) with nidx_merge_topk's arguments: kmerge_by(|a, b| a.score >= b.score), take(k),
 * exactly as itertools 0.14 runs it, over the parts in the order given (the reference's `responses` vector).  A part ends at its
 * first NIDX_NIL.  Equal scores (f32 ==, so -0 == +0) are NOT resolved lower part first: itertools' heap decides which equal head
 * leads (e.g. 2 parts of scores (1, 1, 0.5) -> (part, position) = (1,0) (0,0) (1,1) (0,1) ...).  n_parts * k < 2^31.  Device pointers. */
int nidx_merge_vector_parts(int32_t device, const uint32_t* ids, const float* scores, int32_t n_parts, int64_t part_stride, int32_t nq, int32_t k,
                            uint32_t* out_ids, float* out_scores, int32_t* out_part, void* stream);

/* Counters of the last HNSW search / build on this segment (for the roofline accounting, SURVEY 8d): [0] similarity
 * evaluations, [1] node expansions, [2] visited-set overflows.  Every search call resets them, whatever its method, so they are
 * 0 after a search that does not walk the graph (a scan, an empty segment, nothing matching).  Every search call counts into
 * its own workspace, so concurrent searches never mix their counts; "last" = the call that was issued last. */
int nidx_vec_counters(nidx_vec_segment* seg, uint64_t out[3]);
/* The same with the quantised walk's: [0] exact similarities computed, [1] expansions, [2] visited-set overflows, [3] closest_up
 * overflows, [4] RaBitQ estimates, [5] exact similarities the sequential rerank_top needed (<= the share of [0] spent there). */
int nidx_vec_counters_ex(nidx_vec_segment* seg, uint64_t out[6]);
/* f32 vector rows the last HNSW search / build read to compute a similarity.  The walk screens neighbours on an fp16 copy of
 * the vectors with a proven error bound and reads the f32 row only of those that can enter its list, so this is at most
 * the similarity count of nidx_vec_counters (equal when the segment has no fp16 copy). */
int nidx_vec_exact_rows(nidx_vec_segment* seg, uint64_t* out);
/* The tensor-core filter of the last exhaustive scan (batches of >= 64 queries, k <= 16): [0] vectors re-scored exactly as
 * survivors of the filter, [1] queries scanned exactly in full instead (a list that may have overflowed, too many survivors, or
 * a query outside the filter's error bound).  Both are 0 when the scan did not use the filter. */
int nidx_vec_scan_counters(nidx_vec_segment* seg, uint64_t out[2]);
/* Queries the last search's dense HNSW walk (NIDX_METHOD_HNSW, or AUTO choosing it) walked a second time because their first
 * walk overflowed its visited set or dropped a candidate it would have popped.  The second walk cannot overflow and its results
 * are returned; the counters describe it in place of the first.  0 after any other search, a build, or a walk that needed none. */
int nidx_vec_walk_reruns(nidx_vec_segment* seg, uint64_t* out);

/* RaBitQ 1-bit codes (vector_types/rabitq.rs; Dot similarity and dimension % 64 == 0 only, config.rs:170-173).
 * nidx_vec_rabitq_encode builds the reference's vectors.quant records ([f32 dot_quant_original][u32 sum_bits][dim/8 sign
 * bits], quant_vector_store.rs:29,57-60) in HBM; nidx_vec_rabitq_codes copies them out ([n][dim/8 + 8] bytes, host);
 * nidx_vec_rabitq_estimate evaluates QueryVector::similarity (estimate, error bound; rabitq.rs:202-218) of every stored
 * vector for nq queries into out_estimate / out_error [nq][n] (same `mem` as the queries).  NIDX_METHOD_BRUTE_RABITQ in
 * and NIDX_METHOD_HNSW_RABITQ in nidx_vec_search need the codes. */
int nidx_vec_rabitq_encode(nidx_vec_segment* seg, void* stream);
int nidx_vec_rabitq_codes(const nidx_vec_segment* seg, uint8_t* out_codes);
int nidx_vec_rabitq_estimate(nidx_vec_segment* seg, const float* queries, int32_t nq, int32_t ldq, int mem, float* out_estimate, float* out_error,
                             void* stream);

/* Device time (CUDA events on the caller's stream) of the dominant kernel of the last nidx_vec_search on
 * this segment: hnsw_search_kernel, or the first scan_scores_kernel of a brute-force call.  Diagnostics
 * for the roofline line of bench.py; not meaningful under concurrent searches. */
int nidx_vec_last_kernel_ms(nidx_vec_segment* seg, float* ms);

/* ------------------------------------------------------------------------------------------
 * Text segment: BM25 over device-resident postings
 * (reference: tantivy TopDocs::order_by_score called at nidx_text/src/reader.rs:433-435 and
 *  nidx_paragraph/src/reader.rs:290-292; statistics over the union of segments,
 *  nidx_tantivy/src/index_reader.rs:39-77)
 * ------------------------------------------------------------------------------------------ */
typedef struct nidx_txt_segment nidx_txt_segment;

#define NIDX_BM25_OR 0   /* nidx_paragraph keyword query: Occur::Should (keyword_parser.rs:62-67) */
#define NIDX_BM25_AND 1  /* nidx_text: QueryParser::set_conjunction_by_default (reader.rs:372-377) */

/* Postings in CSR form: term_off[n_terms+1], post_doc/post_tf[term_off[n_terms]] (doc ids ascending
 * per term), fieldnorm_id[n_docs] (tantivy's 1-byte fieldnorm code).  Host pointers; copied to HBM. */
int nidx_txt_create(int32_t device, uint32_t n_docs, uint32_t n_terms, const uint64_t* term_off, const uint32_t* post_doc,
                    const uint32_t* post_tf, const uint8_t* fieldnorm_id, nidx_txt_segment** out);
/* Collection statistics of the whole index (all segments, all GPUs): total docs, total tokens,
 * doc_freq[n_terms].  Defaults to the segment's own statistics. */
int nidx_txt_set_stats(nidx_txt_segment* seg, uint64_t total_docs, uint64_t total_tokens, const uint64_t* doc_freq);
int nidx_txt_set_alive(nidx_txt_segment* seg, const uint64_t* alive_bits);
/* Closes a segment or a view.  Closing a view frees only its alive bits. */
void nidx_txt_close(nidx_txt_segment* seg);

/* A view of seg under a document mask: a handle whose alive set is seg's alive set AND mask_bits ((n_docs + 63) / 64 words, `mem`;
 * on the device path typically nidx_txt_prefilter's output, which never leaves HBM).  Every search entry point of a text segment
 * (nidx_txt_search*, nidx_txt_list_ordered, nidx_txt_facet_count_all, nidx_txt_prefilter, ...) accepts the view and runs over the
 * masked set only: matches, totals, facet counts and listings are those of a copy of seg whose alive bits were set to alive AND mask.
 * Scores keep seg's statistics (nidx_txt_set_stats): masked-out documents still count in N, document frequencies and the average
 * length, as under a filter in the reference.  The view shares every other array of seg read-only and owns only its
 * (n_docs + 63) / 64 alive words, computed on `stream` (a call on another stream must be ordered after it by the caller).  Setters on
 * a view are NIDX_EINVAL.  seg must outlive the view, and must not be changed while the view is in use; close the view with
 * nidx_txt_close. */
int nidx_txt_view(nidx_txt_segment* seg, const uint64_t* mask_bits, int mem, nidx_txt_segment** out_view, void* stream);

typedef struct nidx_txt_search_params {
    int32_t k;       /* result_per_page + 1 in the reference (reader.rs:386-387) */
    int32_t mode;    /* NIDX_BM25_* */
    int32_t use_tf;  /* 0: IndexRecordOption::Basic (tf == 1), 1: real term frequencies */
    float min_score; /* results below are dropped after top-k (reader.rs:302-305) */
    /* nidx_paragraph search-after (reader.rs:350-392 build_topdocs_search_after_collector / is_after): documents that
     * are not "after" (after_score, tie break) are scored -inf by the reference's tweak_score; here they are counted
     * in out_total but never enter the top-k. */
    int32_t after_mode;      /* 0 = no search_after; 1 = SearchAfterTieBreak::Drop; 2 = KeepAfter(after_docaddr); 3 = Keep */
    float after_score;       /* SearchAfter.score */
    uint64_t after_docaddr;  /* KeepAfter payload */
    uint64_t docaddr_base;   /* segment_ord << 32: docaddr = docaddr_base + doc (reader.rs:366-371) */
} nidx_txt_search_params;

/* nq queries; query i is query_terms[query_off[i] .. query_off[i+1]) (term ids).
 * out_docs/out_scores [nq][k] (score desc, then doc asc), out_counts[nq], out_total[nq] = number of
 * matching documents (the Count collector, reader.rs:433).  `mem` applies to queries and outputs. */
int nidx_txt_search(nidx_txt_segment* seg, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem,
                    const nidx_txt_search_params* p, uint32_t* out_docs, float* out_scores, int32_t* out_counts, uint64_t* out_total,
                    void* stream);

/* Device time (CUDA events on the caller's stream) of bm25_kernel in the last nidx_txt_search on this segment (bench roofline),
 * or of the facet kernel of the last nidx_txt_search_faceted / nidx_txt_facet_count_all, of the order kernel of the last
 * nidx_txt_search_ordered, of the two listing kernels of the last nidx_txt_list_ordered, or of the pass of the last nidx_txt_prefilter;
 * not meaningful under concurrent searches. */
int nidx_txt_last_kernel_ms(nidx_txt_segment* seg, float* ms);

/* ---- Facet counts: tantivy's FacetCollector next to Count and TopDocs
 * (reference: the (Count, facet_collector, topdocs) tuples of nidx_text/src/reader.rs:388-450 and
 *  nidx_paragraph/src/reader.rs:252-347; groups produced by produce_facets, nidx_text/src/reader.rs:43-62 and
 *  nidx_paragraph/src/search_response.rs:48-77)
 * A facet is given in tantivy's encoded form: the path's segments joined by 0x00 bytes, without the leading '/'
 * ("/l/set/a" -> "l\0set\0a"); the root "/" is the empty string.  Facet order = memcmp order of the encoded bytes. */

/* The segment's facet dictionary and every document's facets: n_facets keys, strictly ascending in facet order, key i =
 * key_bytes[key_off[i] .. key_off[i + 1]); document d carries the ords doc_ords[doc_off[d] .. doc_off[d + 1]) (strictly
 * ascending; doc_off has n_docs + 1 entries).  The keys stay on the host side of the library (a request is resolved by binary
 * search: the descendants of a facet are one ord range), the ords live in HBM.  Segments of one index should be given the same
 * dictionary, so that a bucket means the same child in every segment and per-segment counts add up as arrays.  Host pointers.  A
 * call that fails (rejected input included) leaves the segment's previous facets in place. */
int nidx_txt_set_facets(nidx_txt_segment* seg, uint32_t n_facets, const uint8_t* key_bytes, const uint64_t* key_off, const uint64_t* doc_off,
                        const uint32_t* doc_ords);

typedef struct nidx_txt_facet_request {   /* FacetCollector::add_facet for each facet: facet i = key_bytes[key_off[i] .. key_off[i + 1]) */
    int32_t n;
    const uint8_t* key_bytes;
    const uint64_t* key_off;
} nidx_txt_facet_request;

/* The buckets of a request: one per direct child of a requested facet that the dictionary holds, requested facets taken in facet
 * order (duplicates collapse), children in facet order.  out_bucket_req[b] = index of the request that bucket b belongs to,
 * out_bucket_ord[b] = the first dictionary ord under its child (the child is that key cut after the requested facet's depth + 1).
 * At most `cap` entries are written (n_facets is always enough); *out_n_buckets = the number of buckets.  A requested facet that
 * is an ancestor of another is NIDX_EINVAL (tantivy asserts).  Host pointers; needs no device work. */
int nidx_txt_facet_buckets(nidx_txt_segment* seg, const nidx_txt_facet_request* facets, uint32_t* out_bucket_req, uint32_t* out_bucket_ord,
                           uint32_t cap, uint32_t* out_n_buckets);

/* nidx_txt_search + the FacetCollector in the same pass: docs / scores / counts / totals are those of nidx_txt_search, and
 * out_facet_counts[nq][n_buckets] (`mem`, u32) = for each bucket the number of matched documents (query match AND alive: the set
 * out_total counts, whatever k, min_score or search-after) that carry its child or a descendant of it, once per document.
 * A facet equal to the requested one counts nothing. */
int nidx_txt_search_faceted(nidx_txt_segment* seg, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem,
                            const nidx_txt_search_params* p, const nidx_txt_facet_request* facets, uint32_t* out_docs, float* out_scores,
                            int32_t* out_counts, uint64_t* out_total, uint32_t* out_facet_counts, void* stream);

/* The same counts over every alive document (the AllQuery of an empty body, nidx_text/src/search_query.rs:100-101: the
 * only_faceted catalogue request): out_facet_counts[n_buckets] (`mem`, u32). */
int nidx_txt_facet_count_all(nidx_txt_segment* seg, const nidx_txt_facet_request* facets, int mem, uint32_t* out_facet_counts, void* stream);

/* ---- Order by date: TopDocs::order_by_fast_field("created" | "modified", Desc | Asc) next to Count (and the FacetCollector)
 * (reference: nidx_text/src/reader.rs:208-287, 415-431 and nidx_paragraph/src/reader.rs:229-243, 270-287, 310-327).
 * Dates are seconds (the reference stores DateTime::from_timestamp_secs(ts.seconds) and returns {seconds, nanos: 0}:
 * nidx_text/src/schema.rs:48-57).  Results are ordered by (date in the requested direction, then doc ascending); documents without
 * a date come after every dated document in both directions.  The order is exact over the whole i64 range of seconds. */
#define NIDX_DATE_NONE INT64_MIN   /* the document has no date */
#define NIDX_ORDER_CREATED 0       /* OrderBy.OrderField (nodereader.proto) */
#define NIDX_ORDER_MODIFIED 1
#define NIDX_ORDER_DESC 0          /* OrderBy.OrderType */
#define NIDX_ORDER_ASC 1

typedef struct nidx_txt_order {
    int32_t field;   /* NIDX_ORDER_CREATED | NIDX_ORDER_MODIFIED */
    int32_t type;    /* NIDX_ORDER_DESC | NIDX_ORDER_ASC */
} nidx_txt_order;

/* Every document's created and modified seconds (n_docs each, NIDX_DATE_NONE = none; host pointers).  The seconds and, per field,
 * each document's dense rank among the segment's distinct dates (built on the device) live in HBM.  A call that fails leaves the
 * segment's previous dates in place. */
int nidx_txt_set_dates(nidx_txt_segment* seg, const int64_t* created, const int64_t* modified);

/* nidx_txt_search (facets == NULL) or nidx_txt_search_faceted with TopDocs ordered by date: the matched set, out_total and the facet
 * counts are theirs; out_docs / out_dates [nq][p->k] (`mem`; dates in seconds, i64) follow the order above, out_counts[nq] entries
 * are filled (NIDX_NIL / NIDX_DATE_NONE padded).  p->min_score and search-after are ignored, as in the reference (convert_int_order);
 * p->use_tf does not matter.  A segment without dates (nidx_txt_set_dates) is NIDX_EINVAL. */
int nidx_txt_search_ordered(nidx_txt_segment* seg, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem,
                            const nidx_txt_search_params* p, const nidx_txt_order* order, const nidx_txt_facet_request* facets, uint32_t* out_docs,
                            int64_t* out_dates, int32_t* out_counts, uint64_t* out_total, uint32_t* out_facet_counts, void* stream);

/* ---- Exact phrases: tantivy's PhraseQuery (slop 0) as one clause of the keyword query (reference: the quoted groups of
 * nidx_paragraph's body, query_parser/keyword_parser.rs:27-91).  A phrase t_0 .. t_{m-1} occurs in a document freq times, freq = the
 * number of start positions s such that t_i is at position s + i for every i; the document matches when freq >= 1 and scores
 * weight * freq / (freq + norm(fieldnorm)), weight = (f32 sum of the terms' idf, in phrase order, repeats counted) * (1 + k1), from
 * the statistics of nidx_txt_set_stats -- whatever p->use_tf says for the plain terms.  A phrase with a term of no posting in the
 * segment matches nothing (a term id >= n_terms also weighs 0).  OR: the phrase is one more optional clause; AND: one more required
 * clause. */

/* Every posting's token positions, in posting order (term by term, doc ascending), each posting's tf of them strictly ascending
 * (n_positions = the sum of the tf given to nidx_txt_create).  A token's position is its index in the token stream before long
 * tokens are dropped, so a dropped token leaves a gap.  Host pointer; HBM: 4 bytes per position + 8 per posting.  A segment whose
 * tf does not fit 24 bits, a count that does not add up or positions out of order are NIDX_EINVAL; a call that fails leaves the
 * previous positions in place. */
int nidx_txt_set_positions(nidx_txt_segment* seg, const uint32_t* positions, uint64_t n_positions);

typedef struct nidx_txt_phrases {   /* host memory, whatever `mem` says */
    const uint32_t* terms;   /* every phrase's term ids, concatenated */
    const uint32_t* off;     /* [n + 1]: phrase i = terms[off[i] .. off[i + 1]), 2 to 64 terms */
    const uint32_t* query;   /* [n]: the query of the batch phrase i is a clause of */
    int32_t n;
} nidx_txt_phrases;

/* nidx_txt_search (order == NULL, facets == NULL), nidx_txt_search_faceted (facets != NULL) or nidx_txt_search_ordered
 * (order != NULL: out_dates instead of out_scores) with phrase clauses besides each query's terms.  A query holds at most 128
 * clauses, a phrase counting as one; the segment needs positions (nidx_txt_set_positions) when phrases->n > 0, else NIDX_EINVAL.
 * With phrases->n == 0 the outputs are exactly those of the call it stands for. */
int nidx_txt_search_phrases(nidx_txt_segment* seg, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem,
                            const nidx_txt_search_params* p, const nidx_txt_phrases* phrases, const nidx_txt_order* order,
                            const nidx_txt_facet_request* facets, uint32_t* out_docs, float* out_scores, int64_t* out_dates, int32_t* out_counts,
                            uint64_t* out_total, uint32_t* out_facet_counts, void* stream);

/* The empty body with an order (AllQuery, nidx_text/src/search_query.rs:100-101: the catalogue listing): the top k (1..1024) of every
 * alive document by the order above -> out_docs / out_dates [k], *out_count; *out_total = the alive documents (Count). `mem` applies
 * to the outputs. */
int nidx_txt_list_ordered(nidx_txt_segment* seg, const nidx_txt_order* order, int32_t k, int mem, uint32_t* out_docs, int64_t* out_dates,
                          int32_t* out_count, uint64_t* out_total, void* stream);

/* ---- Prefilter: SearchRequest.field_filter evaluated over every document of the segment (reference: TextReaderService::prefilter,
 * nidx_text/src/reader.rs:147-180, over filter_to_query, nidx_text/src/search_query.rs:156-217).  The strings of the expression are
 * resolved on the caller's side into ranges of ords of the segment's dictionaries (facets: nidx_txt_set_facets; resources and field
 * paths: nidx_txt_set_doc_columns), so the device never sees a string. */

/* Every document's resource ord and field ord (n_docs each, host pointers): indexes into the caller's dictionaries of resource ids
 * and field paths.  The columns live in HBM (8 bytes per document).  A call that fails leaves the previous columns in place. */
int nidx_txt_set_doc_columns(nidx_txt_segment* seg, const uint32_t* resource_ord, const uint32_t* field_ord);

/* Every document's access groups (reference: Resource.security, nidx_text/src/resource_indexer.rs:49-62), in the shape of
 * nidx_txt_set_facets: n_groups keys strictly ascending in facet order (each a group id with a leading '/' added when it lacks one,
 * encoded as a facet), document d carries the ords doc_ords[doc_off[d] .. doc_off[d + 1]) (strictly ascending).  A document without
 * ords is public.  The ords live in HBM; host pointers.  A call that fails (rejected input included) leaves the previous groups in
 * place. */
int nidx_txt_set_doc_groups(nidx_txt_segment* seg, uint32_t n_groups, const uint8_t* key_bytes, const uint64_t* key_off, const uint64_t* doc_off,
                            const uint32_t* doc_ords);

#define NIDX_P_FACET 0     /* the document carries a facet ord in [lo, hi) */
#define NIDX_P_FIELD 1     /* the document's field ord is in [lo, hi) */
#define NIDX_P_RESOURCE 2  /* the document's resource ord is in [lo, hi) */
#define NIDX_P_DATE 3      /* n = NIDX_ORDER_CREATED | NIDX_ORDER_MODIFIED: lo <= seconds <= hi; a document without that date never matches */
#define NIDX_P_KEYWORD 4   /* n term ids in `terms`: 1 = the term occurs in the document, 2..64 = the phrase (slop 0) occurs in it (the
                              segment needs positions), 0 = nothing; an id that is not a term of the segment matches nothing */
#define NIDX_P_ALL 5       /* every document */
#define NIDX_P_AND 6       /* intersection of the n operand subtrees that follow; n = 0 matches nothing */
#define NIDX_P_OR 7        /* union of the n operand subtrees that follow; n = 0 matches nothing */
#define NIDX_P_NOT 8       /* n = 1: every document that the operand does not match */
#define NIDX_P_PUBLIC 9    /* the document has no access group (nidx_txt_set_doc_groups) */
#define NIDX_P_GROUP 10    /* the document carries an access group ord in [lo, hi): a group and its descendants are one range, so a
                              requested group grants the resources of its descendant groups (SearchRequest.security is
                              OR(PUBLIC, GROUP of each requested group)) */
#define NIDX_PREFILTER_MAX_DEPTH 64   /* levels of nesting: a leaf is one level, each AND / OR / NOT adds one */
typedef struct nidx_prefilter_node {   /* an expression in pre-order */
    int32_t kind;                      /* NIDX_P_* */
    int32_t n;                         /* AND / OR / NOT: operands; KEYWORD: terms; DATE: the date field */
    int64_t lo, hi;                    /* FACET / FIELD / RESOURCE: ord range [lo, hi); DATE: since, until in seconds, both inclusive */
    const uint32_t* terms;             /* KEYWORD: n term ids (host pointer) */
} nidx_prefilter_node;

/* The expression AND the alive set over the segment's documents -> out_bits ((n_docs + 63) / 64 words, `mem`, bits past n_docs
 * zero; may be NULL) and *out_matching (host) = the number of set bits.  The call returns when both are in place.  The program
 * (at most 4096 instructions: one per leaf and per operand after an operand's first) runs in one pass over the columns; FACET
 * needs nidx_txt_set_facets, FIELD / RESOURCE nidx_txt_set_doc_columns, DATE nidx_txt_set_dates, a phrase nidx_txt_set_positions,
 * PUBLIC / GROUP nidx_txt_set_doc_groups (else NIDX_ESTATE).  A malformed expression, one deeper than NIDX_PREFILTER_MAX_DEPTH or a longer program is NIDX_EINVAL. */
int nidx_txt_prefilter(nidx_txt_segment* seg, const nidx_prefilter_node* nodes, int32_t n_nodes, uint64_t* out_bits, int mem, uint64_t* out_matching,
                       void* stream);

/* The hand-off to one vector segment (reference: nidx_vector/src/searcher.rs:300-314 with PrefilterResult::Some) of a text part,
 * a resource part (SearchRequest.json_filter, below) or both:
 *   text: doc_bits over n_docs text documents and join[n_docs] (u32: the document's key in this segment's NIDX_INV_FIELDS index, or
 *     NIDX_NIL) -> the paragraphs of the matched documents' keys; doc_bits NULL = no text part;
 *   resources: res_bits over n_res resources -> their paragraphs: resource r's are the postings res_ranges[2 r] .. res_ranges[2 r + 1]
 *     of the NIDX_INV_FIELDS index (every key with r's 16 uuid bytes as prefix, one contiguous run of keys); res_bits NULL = no
 *     resource part;
 * combined under doc_op (NIDX_F_AND | NIDX_F_OR; read only when both parts are given), then with a filter formula (nodes, n_nodes > 0;
 * nidx_vec_filter's format) under op (NIDX_F_AND | NIDX_F_OR: SearchRequest.filter_operator), then ANDed with the alive set ->
 * out_bits ((paragraphs + 63) / 64 words; may be NULL) and *out_matching (host), to be passed to nidx_vec_search as filter_bits and
 * filter_matching.  No part at all is NIDX_EINVAL; a part with no documents or resources is an empty set.  All buffers `mem`; the call
 * returns when both outputs are in place.  The formula has nidx_vec_filter's limit, less one instruction per part, one for doc_op
 * when both are given and one for op. */
int nidx_vec_prefilter_bits(nidx_vec_segment* seg, const uint64_t* doc_bits, uint64_t n_docs, const uint32_t* join, int32_t doc_op,
                            const uint64_t* res_bits, uint64_t n_res, const uint64_t* res_ranges, const nidx_filter_node* nodes, int32_t n_nodes,
                            int32_t op, uint64_t* out_bits, int mem, uint64_t* out_matching, void* stream);

/* ---- JSON filters: SearchRequest.json_filter (reference: nidx_json, JsonSearcher::search -> a set of resources, combined with the
 * text prefilter by PrefilterResult::combine, nidx_types/src/prefilter.rs:49-92).  The JSON index is a text segment without terms:
 * one document per resource's JSON document, each flattened (path, value) an ord of a dictionary sorted by (path, kind, value) and
 * carried as a facet ord (nidx_txt_set_facets), the resource ord in the resource column (nidx_txt_set_doc_columns) and the resource's
 * access groups (nidx_txt_set_doc_groups).  A leaf is then one NIDX_P_FACET range, NOT ranges over the alive JSON documents, and the
 * expression runs in nidx_txt_prefilter's one pass.  The entry points below turn its output into a resource bitset and hand that to
 * the paragraph search; nidx_vec_prefilter_bits takes it as its resource part.  None of the bitsets leaves HBM on the device path. */

/* doc_bits ((n_docs + 63) / 64 words: typically nidx_txt_prefilter's output) -> out_res_bits ((n_resources + 63) / 64 words, zeroed
 * first): bit r set when a set document's resource ord (nidx_txt_set_doc_columns) is r; ords >= n_resources are dropped.  `mem` applies
 * to both. */
int nidx_txt_resource_bits(nidx_txt_segment* seg, const uint64_t* doc_bits, uint64_t n_resources, uint64_t* out_res_bits, int mem, void* stream);

/* One mask over seg's documents (for nidx_txt_view): bit d = and_bits[d] AND op(doc_bits[doc_join[d]], res_bits[res_join[d]]), op =
 * NIDX_F_AND | NIDX_F_OR.  and_bits NULL = every bit set; doc_bits NULL = every bit set (doc_join unread); a join entry of NIDX_NIL,
 * or past n_doc_bits / n_res, reads 0.  doc_join / res_join are [n_docs] u32 (the document's bit in doc_bits, its resource ord).
 * -> out_bits ((n_docs + 63) / 64 words, padding bits zero), *out_matching = its set bits (the alive set is not applied: the view does
 * that).  All buffers `mem`; the call returns when both are in place. */
int nidx_txt_join_mask(nidx_txt_segment* seg, const uint64_t* and_bits, const uint64_t* doc_bits, uint64_t n_doc_bits, const uint32_t* doc_join,
                       const uint64_t* res_bits, uint64_t n_res, const uint32_t* res_join, int32_t op, uint64_t* out_bits, int mem,
                       uint64_t* out_matching, void* stream);

/* ---- Graph search: NidxSearcher.GraphSearch (reference: nidx_relation).  One document per relation, in a text segment without
 * terms: its facets (nidx_txt_set_facets), resource / field ords (nidx_txt_set_doc_columns) and alive bits, so the prefilter mask
 * is nidx_txt_join_mask's.  The graph columns live in a handle that borrows that segment: the segment must outlive it. */
typedef struct nidx_graph nidx_graph;

#define NIDX_G_SRC_VALUE 0    /* per-document u32 ord columns: the source / target normalised value (values dictionary) */
#define NIDX_G_DST_VALUE 1
#define NIDX_G_SRC_TYPE 2     /* node types (0..3) */
#define NIDX_G_DST_TYPE 3
#define NIDX_G_SRC_SUBTYPE 4  /* subtype ords */
#define NIDX_G_DST_SUBTYPE 5
#define NIDX_G_REL_TYPE 6     /* relation type (0..5) */
#define NIDX_G_LABEL 7        /* label ord */
#define NIDX_G_SRC_NODE 8     /* node key ords (value, type, subtype) */
#define NIDX_G_DST_NODE 9
#define NIDX_G_REL_KEY 10     /* relation key ord (type, label) */
#define NIDX_G_COLUMNS 11

typedef struct nidx_graph_columns {   /* host pointers */
    const uint32_t* col[NIDX_G_COLUMNS];   /* [n_docs] each */
    const uint64_t* tok_off[2];            /* [n_docs + 1]: source (0) / target (1) default tokens as ords of the token dictionary */
    const uint32_t* tok_ord[2];
    uint32_t n_values;                     /* the values dictionary: entry e is value_cp[value_off[e] .. value_off[e + 1]) (code points) */
    const uint32_t* value_cp;
    const uint64_t* value_off;
    uint32_t n_tokens;                     /* the token dictionary, as the values' */
    const uint32_t* token_cp;
    const uint64_t* token_off;
    uint32_t n_node_keys, n_rel_keys;      /* NODE columns are < n_node_keys, REL_KEY < n_rel_keys */
} nidx_graph_columns;

/* A graph handle over seg (which must outlive it), without columns. */
int nidx_graph_create(nidx_txt_segment* seg, nidx_graph** out);
/* Checks and uploads the columns and dictionaries to HBM; a rejected or failed call leaves the previous ones in place. */
int nidx_graph_set_columns(nidx_graph* g, const nidx_graph_columns* cols);
void nidx_graph_close(nidx_graph* g);

#define NIDX_G_EQ 0          /* column arg == lo; score w */
#define NIDX_G_COLBITS 1     /* column arg (a value column) has an ord matched by automaton term lo; score w */
#define NIDX_G_TOKBITS 2     /* some token of side arg (0 source, 1 target) is matched by automaton term lo; score w */
#define NIDX_G_TOKSET 3      /* some token of side arg is one of the n ords `ords` (host pointer); score w */
#define NIDX_G_FACET 4       /* a facet ord in [lo, hi); score w */
#define NIDX_G_CONST 5       /* every document (lo = 1) or none (lo = 0); score w */
#define NIDX_G_AND 6         /* n >= 1 operands: all match; score = their sum, in order */
#define NIDX_G_OR 7          /* n >= 1 operands: any matches; score = the sum of the matched ones, in order */
#define NIDX_G_NOT 8         /* n = 1: the operand does not match; score 0 */
#define NIDX_G_CONST_SCORE 9 /* n = 1: the operand, scored w where it matches */
typedef struct nidx_graph_node {      /* an expression in pre-order */
    int32_t kind;                     /* NIDX_G_* */
    int32_t n;                        /* AND / OR / NOT / CONST_SCORE: operands; TOKSET: ords */
    int32_t arg;                      /* EQ / COLBITS: the column; TOKBITS / TOKSET: the side */
    float w;
    int64_t lo, hi;
    const uint32_t* ords;
} nidx_graph_node;

#define NIDX_G_TERMS_VALUES 0   /* an automaton term over the values dictionary */
#define NIDX_G_TERMS_TOKENS 1   /* over the token dictionary */
#define NIDX_G_MAX_TERMS 64     /* automaton terms per search, 4096 code points in all */
typedef struct nidx_graph_term {
    int32_t dict;                     /* NIDX_G_TERMS_* */
    int32_t distance;                 /* 0..2: restricted Damerau-Levenshtein on code points */
    int32_t prefix;                   /* 1: some prefix of the entry is within distance */
    int32_t n_cp;
    const uint32_t* cp;               /* host pointer */
} nidx_graph_term;

#define NIDX_G_PATH 0        /* ids: documents (ties: lower document first) */
#define NIDX_G_NODES 1       /* two expressions follow each other in nodes: the source side and the destination side; ids: node key
                                ords, each scored with the max over both sides' matched documents (ties: lower ord first) */
#define NIDX_G_RELATIONS 2   /* ids: relation key ords, the max over the matched documents (ties: lower ord first) */
#define NIDX_G_MAX_K 1024
/* The scored expression(s) over the documents alive AND mask (n_docs bits, `mem`; NULL: alive) -> the best k (1..NIDX_G_MAX_K) ids by
 * score descending: out_ids [k] (NIDX_NIL padded), out_scores [k], *out_count (all `mem`).  An expression deeper than
 * NIDX_PREFILTER_MAX_DEPTH or longer than 4096 instructions, more automaton terms or code points than above, a distance > 2 and a k
 * out of range, and a node whose w is negative, NaN or infinite are NIDX_EINVAL (sums of finite scores >= 0 order as their bits);
 * a handle without columns is NIDX_ESTATE.  The call returns when the outputs are in place (host) or
 * are enqueued on `stream` (device). */
int nidx_graph_search(nidx_graph* g, const nidx_graph_node* nodes, int32_t n_nodes, const nidx_graph_term* terms, int32_t n_terms, int32_t kind,
                      int32_t k, const uint64_t* mask, int mem, uint32_t* out_ids, float* out_scores, int32_t* out_count, void* stream);
/* The times (ms) of the last search's dictionary pass, scored pass(es), collection (unique max + top-k) and whole call. */
int nidx_graph_last_times(nidx_graph* g, float* ms4);

/* ---- Suggest: the paragraph pass of NidxSearcher.Suggest (reference: nidx_paragraph/src/reader.rs:58-90, search_query.rs:87-183,
 * query_parser/fuzzy_parser.rs, fuzzy_query.rs:88-116).  The keyword pass is nidx_txt_search(_phrases) on views (nidx_txt_view) under
 * the suggest mask below; when it finds nothing, the fuzzy pass runs over the same views: every fuzzy literal is expanded over the
 * paragraph index's vocabulary (one dictionary per index, shared by its segments) and each clause becomes a constant-score union of
 * the postings of the terms it accepts. */
typedef struct nidx_suggest_dict nidx_suggest_dict;

/* The vocabulary as code points: term id e is cp[off[e] .. off[e + 1]) (host pointers, copied to HBM). */
int nidx_suggest_dict_create(int32_t device, uint32_t n_terms, const uint32_t* cp, const uint64_t* off, nidx_suggest_dict** out);
void nidx_suggest_dict_close(nidx_suggest_dict* d);
/* The n (0..NIDX_G_MAX_TERMS) automaton terms (nidx_graph_term, host; `dict` is not read) -> out_bits [n][(n_terms + 63) / 64]
 * (a DEVICE pointer): bit e of row i when term e is within row i's distance (prefix: some prefix of term e is).  out_counts (host,
 * may be NULL) = the set bits of each row.  The call returns when the bits are in place. */
int nidx_suggest_expand(nidx_suggest_dict* d, const nidx_graph_term* terms, int32_t n, uint64_t* out_bits, uint64_t* out_counts, void* stream);
/* The time (ms) of the last nidx_suggest_expand's dictionary pass. */
int nidx_suggest_last_ms(nidx_suggest_dict* d, float* ms);

/* The paragraphs repeated in their field (IndexParagraph.repeated_in_field): (n_docs + 63) / 64 words (host); NULL = none. */
int nidx_txt_set_repeated(nidx_txt_segment* seg, const uint64_t* bits);
/* The suggest mask over seg's documents: bit d = NOT repeated AND sec_bits AND op(pf_bits, joined_bits), op = NIDX_F_AND | NIDX_F_OR; a
 * NULL operand is dropped (not read as "all": op applies only when both pf_bits and joined_bits are given).  Every bitset has
 * (n_docs + 63) / 64 words -> out_bits (padding bits zero) and *out_matching = its set bits (the alive set is not applied: the view
 * does that).  All buffers `mem`; the call returns when both are in place. */
int nidx_txt_suggest_mask(nidx_txt_segment* seg, const uint64_t* sec_bits, const uint64_t* pf_bits, const uint64_t* joined_bits, int32_t op,
                          uint64_t* out_bits, int mem, uint64_t* out_matching, void* stream);

#define NIDX_SG_FUZZY 0        /* arg = a row of the expansion bitsets: the union of its terms' postings, scored 1.0 */
#define NIDX_SG_TERM 1         /* arg = a term id (>= n_terms: matches nothing): BM25 at tf = 1 */
#define NIDX_SG_PHRASE 2       /* arg = a phrase of `phrases` (slop 0): BM25 at the phrase frequency */
#define NIDX_SG_MAX_CLAUSES 64
#define NIDX_SG_MAX_HITS 16
typedef struct nidx_suggest_clause {
    int32_t kind;              /* NIDX_SG_* */
    uint32_t arg;
} nidx_suggest_clause;

/* The fuzzy pass over seg's alive documents (a view: under its mask).  A document matches when a clause does, and scores
 * 0.5 * (the f32 sum, in clause order, of 1.0 per matched FUZZY clause, w_t * (1 / (1 + norm)) per matched TERM and
 * w_p * (freq / (freq + norm)) per matched PHRASE), with the weights and norms of nidx_txt_set_stats and of nidx_txt_search_phrases.
 * exp_bits: n_exp_rows rows over the n_dict terms of the dictionary (<= the segment's terms), a DEVICE pointer (nidx_suggest_expand's
 * output); phrases: as nidx_txt_search_phrases (`query` unread; NULL = none; the segment needs positions when there are some).
 * -> out_ids [k] (1..NIDX_G_MAX_K; score descending, ties to the lower document; NIDX_NIL padded), out_scores [k], *out_count, and
 * for the first min(count, match_hits) hits (match_hits 0..NIDX_SG_MAX_HITS) every (hit, FUZZY clause, expanded term) whose term
 * occurs in the hit, packed as hit << 40 | clause << 32 | term id, in no fixed order: the first match_cap of them in out_matches,
 * their number in *out_n_matches (larger than match_cap when some did not fit).  Outputs `mem`; the call returns when they are in
 * place (host) or enqueued on `stream` (device). */
int nidx_txt_suggest_fuzzy(nidx_txt_segment* seg, const nidx_suggest_clause* clauses, int32_t n_clauses, const uint64_t* exp_bits, int32_t n_exp_rows,
                           uint64_t n_dict, const nidx_txt_phrases* phrases, int32_t k, int32_t match_hits, int mem, uint32_t* out_ids, float* out_scores,
                           int32_t* out_count, uint64_t* out_matches, uint32_t match_cap, uint32_t* out_n_matches, void* stream);
/* The times (ms) of the last fuzzy pass on seg (or on a view of it): clause bitsets (phrase lists included), scored pass, top-k,
 * matches. */
int nidx_txt_suggest_last_times(nidx_txt_segment* seg, float* ms4);

/* ------------------------------------------------------------------------------------------
 * Segments sharded over the GPUs of one node: one process (or thread) per GPU, one segment each
 * (reference: the searcher's scatter-gather, nidx/src/searcher/grpc.rs:253-431, merged by
 *  shard_merge.rs:332-348 / 177-231; inside one index the cross-segment collection Fssc, nidx_vector/src/searcher.rs:150-199)
 * ------------------------------------------------------------------------------------------ */
typedef struct nidx_shard_comm nidx_shard_comm;

/* ncclGetUniqueId: rank 0 creates the 128-byte id and hands it to the other ranks by whatever channel the host has
 * (the reference's searchers already know each other through their gRPC addresses). */
int nidx_shard_unique_id(uint8_t out_id[128]);
/* ncclCommInitRank on `device`; collective: every rank of `world` must call it with the same id.  NCCL is bound at run time
 * (libnccl.so.2); without it these entry points fail with NIDX_ESTATE and everything else keeps working. */
int nidx_shard_init(const uint8_t unique_id[128], int32_t rank, int32_t world, int32_t device, nidx_shard_comm** out);
void nidx_shard_destroy(nidx_shard_comm* comm);

/* Paragraph keys for the cross-segment de-duplication: keys[p] identifies paragraph p's id across segments (the reference keys
 * Fssc by the paragraph id string, searcher.rs:62-90: pass a 64-bit hash of it).  NULL = (rank, paragraph address). Host pointer. */
int nidx_vec_set_paragraph_keys(nidx_vec_segment* seg, const uint64_t* keys);

/* OpenSegment::search on this rank's segment + exchange + merge, identical results on every rank.  Collective: every rank calls
 * it with the same queries, nq, k and dedup, in the same order (one call at a time per communicator).  It is
 * nidx_vec_shard_record (rank = this rank), an all-gather of the records in rank order, then nidx_shard_merge.
 *   dedup = 0: the parts are shards -- merge_vector_responses (kmerge_by(score >=), shard_merge.rs:332-348), parts in rank
 *              order standing for the reference's `responses` order; ties as nidx_merge_vector_parts;
 *   dedup = 1: the parts are segments of ONE index -- Fssc (searcher.rs:150-199): one entry per paragraph key, and with
 *              p->with_duplicates == 0 byte-identical vectors are suppressed across segments (by a 64-bit hash of the bytes).
 * out_ids are vector addresses local to the part in out_part[nq][k] (-1 = none); out_counts[nq] may be NULL.
 * `mem` applies to queries and outputs; device calls are asynchronous on `stream`. */
int nidx_vec_search_sharded(nidx_shard_comm* comm, nidx_vec_segment* seg, const float* queries, int32_t nq, int32_t ldq, int mem,
                            const nidx_vec_search_params* p, int32_t dedup, uint32_t* out_ids, float* out_scores, int32_t* out_part, int32_t* out_counts,
                            void* stream);

/* The two halves of nidx_vec_search_sharded without the exchange, for a host that gathers the records by other means (or one GPU
 * holding several parts).  A record of nq queries at k = p->k is, in 32-bit words:
 *     [ids nq*k u32][scores nq*k f32]                                    dedup = 0   (2 * nq * k words)
 *     [ids nq*k u32][scores nq*k f32][par_key nq*k u64][vec_key nq*k u64] dedup = 1   (6 * nq * k words)
 * ids / scores are nidx_vec_search's (vector addresses local to the segment, score desc, NIDX_NIL padded).  par_key = the
 * paragraph key of nidx_vec_set_paragraph_keys, or (rank << 32) | paragraph address without keys; vec_key = a 64-bit hash of the
 * vector's bytes when p->with_duplicates == 0, else one constant for every vector (the merge does not read it then); both 0 for
 * NIDX_NIL entries.
 * nidx_vec_shard_record: search `seg` into out_record (device memory on the segment's GPU).  `mem` applies to the queries (and
 * p->filter_bits); asynchronous on `stream`. */
int nidx_vec_shard_record(nidx_vec_segment* seg, const float* queries, int32_t nq, int32_t ldq, int mem, const nidx_vec_search_params* p, int32_t rank,
                          int32_t dedup, uint32_t* out_record, void* stream);
/* nidx_shard_merge: merge n_parts records laid end to end (device memory, part i at records + i * record words) with the rule of
 * nidx_vec_search_sharded for `dedup` (with_duplicates: Fssc's flag; ignored for dedup = 0) -> out_ids / out_scores /
 * out_part [nq][k], out_counts[nq] (out_part, out_counts may be NULL).  The de-duplicating merge keeps 16 k + 8 n_parts k bytes per
 * query in shared memory and refuses more than 96 KiB (NIDX_EINVAL).  `mem` applies to the outputs; NIDX_MEM_HOST returns when they
 * are in place, NIDX_MEM_DEVICE is asynchronous on `stream`. */
int nidx_shard_merge(int32_t device, const uint32_t* records, int32_t n_parts, int32_t nq, int32_t k, int32_t dedup, int32_t with_duplicates, int mem,
                     uint32_t* out_ids, float* out_scores, int32_t* out_part, int32_t* out_counts, void* stream);
/* BM25 over a document-partitioned index (every part scores with the statistics of the whole index, nidx_txt_set_stats):
 * merge_document_responses' order (bm25 desc, part asc, doc asc; shard_merge.rs:227-231); out_total = Count over all parts. */
int nidx_txt_search_sharded(nidx_shard_comm* comm, nidx_txt_segment* seg, const uint32_t* query_terms, const uint32_t* query_off, int32_t nq, int mem,
                            const nidx_txt_search_params* p, uint32_t* out_docs, float* out_scores, int32_t* out_part, int32_t* out_counts, uint64_t* out_total,
                            void* stream);

/* ------------------------------------------------------------------------------------------
 * One shard search as ONE device-side plan + rank fusion on the device (SURVEY 8f rank 4)
 * (reference: run_index_searches, nidx/src/searcher/shard_search.rs:176-241 -- the paragraph, document and vector searches of a
 *  request run on scoped threads; the ranked lists are fused afterwards in Python,
 *  nucliadb/src/nucliadb/search/search/rank_fusion.py:78-186)
 * ------------------------------------------------------------------------------------------ */
/* Caller keys of a text segment's documents (for the paragraph index: the paragraph id, as a 64-bit hash or table index -- the
 * same key space as nidx_vec_set_paragraph_keys), used to match keyword and semantic results.  NULL = the document number. */
int nidx_txt_set_doc_keys(nidx_txt_segment* seg, const uint64_t* keys);

typedef struct nidx_rrf_source {
    const uint64_t* keys;     /* [nq][k] item keys, best first (every source sorted by its score, descending); ~0 = no item */
    const float* scores;      /* [nq][k] the source's scores: reported as they are when only one source has results (rank_fusion.py:86-89) */
    const int32_t* counts;    /* [nq] valid items per query; NULL = k minus trailing ~0 keys */
    int32_t k;
    double weight;            /* the retriever's boost w(r) (rank_fusion.py:133-141) */
} nidx_rrf_source;

/* ReciprocalRankFusion.fuse (rank_fusion.py:78-96, 143-186) for nq queries: score(d) = sum over the sources, in the order given, of
 * 1 / (k + rank) * weight in IEEE double arithmetic (bit-identical to the reference's Python floats); one output item per key (the
 * first occurrence), sorted by score descending, ties in first-insertion order (Python's stable sort).  Rows of out_* are
 * sum(k_i) long: out_refs = first occurrence's source << 28 | mask of contributing sources << 24 | its position in that source;
 * out_counts[nq] = number of fused items.  At most 4 sources. */
int nidx_rank_fusion_rrf(int32_t device, const nidx_rrf_source* sources, int32_t n_sources, int32_t nq, double k, int mem, uint64_t* out_keys,
                         double* out_scores, uint32_t* out_refs, int32_t* out_counts, void* stream);

typedef struct nidx_shard_search_request {
    int32_t nq;
    /* vectors_request (shard_search.rs:211-213): vec == NULL = not requested */
    nidx_vec_segment* vec; const float* queries; int32_t ldq; const nidx_vec_search_params* vec_params;
    const nidx_filter_node* formula; int32_t n_formula;     /* optional filter formula evaluated on the device (nidx_vec_search_formula) */
    /* paragraphs_request (shard_search.rs:189-191): the keyword search, BM25 over the paragraph index */
    nidx_txt_segment* par; const uint32_t* par_terms; const uint32_t* par_off; const nidx_txt_search_params* par_params;
    /* texts_request (shard_search.rs:185-187): BM25 over the document (field) index */
    nidx_txt_segment* doc; const uint32_t* doc_terms; const uint32_t* doc_off; const nidx_txt_search_params* doc_params;
    /* rank fusion of the paragraph (keyword) and vector (semantic) lists; rrf_k <= 0: none */
    double rrf_k, weight_keyword, weight_semantic;
    int32_t semantic_first;   /* order of the sources (the reference iterates a dict: insertion order decides ties and which item object survives) */
} nidx_shard_search_request;

typedef struct nidx_shard_search_response {
    uint32_t* vec_ids; float* vec_scores; int32_t* vec_counts;                          /* [nq][vec_params->k] as nidx_vec_search */
    uint32_t* par_docs; float* par_scores; int32_t* par_counts; uint64_t* par_total;    /* [nq][par_params->k] as nidx_txt_search */
    uint32_t* doc_docs; float* doc_scores; int32_t* doc_counts; uint64_t* doc_total;    /* [nq][doc_params->k] */
    uint64_t* fused_keys; double* fused_scores; uint32_t* fused_refs; int32_t* fused_counts;   /* [nq][kv + kp] as nidx_rank_fusion_rrf */
} nidx_shard_search_response;

/* run_index_searches for a batch of nq requests against one shard's indexes: the requested searches run concurrently on side
 * streams forked from `stream`, are joined back, and (rrf_k > 0, vector and paragraph requests present) the two ranked lists
 * are fused on the device -- keys through nidx_vec_set_paragraph_keys / nidx_txt_set_doc_keys.  `mem` applies to all inputs
 * and outputs; with host buffers the call returns when the results are in them (one synchronisation at the end). */
int nidx_shard_search(const nidx_shard_search_request* req, nidx_shard_search_response* resp, int mem, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* NIDX_B200_H */
