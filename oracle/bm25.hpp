// ORACLE — TEST INFRASTRUCTURE ONLY (see distance.hpp).     *** PARITY UNPINNED ***
//
// CPU restatement of the BM25 top-k that nidx_text / nidx_paragraph obtain from tantivy:
//   nidx/nidx_text/src/reader.rs:432-449        TopDocs::with_limit(k+1).order_by_score() over the parsed
//                                               query (QueryParser::set_conjunction_by_default => AND, real tf)
//   nidx/nidx_text/src/reader.rs:289-355        convert_bm25_order: drop score < min_score, next_page = len > k
//   nidx/nidx_paragraph/src/reader.rs:290-292, 350-377   same collector (+ search-after tweak)
//   nidx/nidx_paragraph/src/query_parser/keyword_parser.rs:34-38,62-67   OR of TermQuery(IndexRecordOption::Basic)
//   nidx/nidx_tantivy/src/index_reader.rs:39-77 statistics are those of the UNION of all segments
//   nidx/src/searcher/shard_merge.rs:227-231    order: bm25 desc, shard id, lower docaddr first
//
// The arithmetic lives in tantivy 0.26.1 (nidx/Cargo.lock:4894), which is NOT in the reference tree,
// and no reference test asserts a BM25 value (SURVEY F9, 8c) => parity unpinned.  Restated from
// tantivy's published algorithm [recalled]:
//   K1 = 1.2, B = 0.75
//   idf(n, N)        = ln(1 + (N - n + 0.5) / (n + 0.5))                      (f32)
//   weight           = idf * (1 + K1)
//   norm(fn_id)      = K1 * (1 - B + B * id_to_fieldnorm(fn_id) / avg_fieldnorm)   (256-entry cache)
//   score(fn_id, tf) = weight * (tf / (tf + norm(fn_id)))
//   avg_fieldnorm    = total_num_tokens / total_num_docs  over all segments (deleted docs included)
//   fieldnorm        = token count of the field, stored as one byte: id = largest i with TABLE[i] <= count,
//                      TABLE[i] = i for i < 24, else 24 + ((8 | (j & 7)) << ((j >> 3) - 1)) with j = i - 24
//                      (j >> 3 == 0: j itself)  -- Lucene SmallFloat.byte4ToInt
//   TermQuery(Basic): term frequencies are not decoded, tf == 1.
//   Boolean OR sums the matching terms' scores, AND requires all terms; sums are f32, here in query-term order
//   (tantivy's order depends on its scorer arrangement; differences are last-ulp).
//   TopDocs: score desc, then (segment_ord, doc) asc.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

namespace nidx_oracle {

static inline uint32_t fieldnorm_id_to_value(uint32_t id) {
    if (id < 24) return id;
    uint32_t j = id - 24, bits = j & 7, shift = j >> 3;
    uint32_t v = shift == 0 ? bits : ((bits | 8u) << (shift - 1));
    return 24 + v;
}
static inline uint8_t fieldnorm_to_id(uint32_t fieldnorm) {
    int lo = 0, hi = 255;  // largest id with value <= fieldnorm
    while (lo < hi) {
        int mid = (lo + hi + 1) / 2;
        if (fieldnorm_id_to_value(mid) <= fieldnorm) lo = mid; else hi = mid - 1;
    }
    return (uint8_t)lo;
}

static const float BM25_K1 = 1.2f, BM25_B = 0.75f;
static inline float bm25_idf(uint64_t doc_freq, uint64_t doc_count) {
    float x = ((float)(doc_count - doc_freq) + 0.5f) / ((float)doc_freq + 0.5f);
    return std::log(1.0f + x);
}
static inline void bm25_norm_cache(float avg_fieldnorm, float cache[256]) {
    for (int i = 0; i < 256; ++i)
        cache[i] = BM25_K1 * (1.0f - BM25_B + BM25_B * (float)fieldnorm_id_to_value(i) / avg_fieldnorm);
}
static inline float bm25_term_score(float weight, float norm, uint32_t tf) {
    float t = (float)tf;
    return weight * (t / (t + norm));
}

// One segment's postings (CSR by term) + per-doc fieldnorm ids.
struct PostingsView {
    uint32_t n_docs = 0, n_terms = 0;
    const uint64_t* term_off = nullptr;  // [n_terms + 1]
    const uint32_t* doc = nullptr;       // sorted per term
    const uint32_t* tf = nullptr;
    const uint8_t* fieldnorm_id = nullptr;  // [n_docs]
    const uint64_t* alive_bits = nullptr;   // nullptr = all alive (deletions, index_reader.rs:48-52)
};
// Collection statistics over the union of segments.
struct Bm25Stats {
    uint64_t total_docs = 0, total_tokens = 0;
    const uint64_t* doc_freq = nullptr;  // [n_terms] summed over segments
    float avg_fieldnorm() const { return (float)total_tokens / (float)total_docs; }
};

struct DocScore {
    uint32_t doc;
    float score;
};

enum Bm25Mode : int { BM25_OR = 0, BM25_AND = 1 };

// Per-thread scratch that survives between queries: accumulators are reset through the list of touched documents, so a query
// costs O(its postings), not O(n_docs) -- closer to what tantivy's document-at-a-time scorers spend, which matters when this
// restatement is timed as the CPU baseline.  The arithmetic (and therefore every output bit) is that of the plain version.
struct Bm25Scratch {
    std::vector<float> acc;
    std::vector<uint16_t> cnt;
    std::vector<uint32_t> touched;
    void ensure(uint32_t n_docs) {
        if (acc.size() < n_docs) { acc.assign(n_docs, 0.0f); cnt.assign(n_docs, 0); }
    }
};

// One query on one segment.  use_tf=false reproduces IndexRecordOption::Basic (tf == 1).
static inline std::vector<DocScore> bm25_search(const PostingsView& P, const Bm25Stats& S, const uint32_t* terms, int n_terms, int mode,
                                                bool use_tf, size_t k, uint64_t* total_hits, Bm25Scratch& sc) {
    float cache[256];
    bm25_norm_cache(S.avg_fieldnorm(), cache);
    sc.ensure(P.n_docs);
    sc.touched.clear();
    float* acc = sc.acc.data();
    uint16_t* cnt = sc.cnt.data();
    for (int t = 0; t < n_terms; ++t) {          // term at a time, in query-term order: the f32 sum of a document is in that order
        uint32_t term = terms[t];
        if (term >= P.n_terms) continue;
        float weight = bm25_idf(S.doc_freq[term], S.total_docs) * (1.0f + BM25_K1);
        for (uint64_t i = P.term_off[term]; i < P.term_off[term + 1]; ++i) {
            uint32_t d = P.doc[i];
            uint32_t tf = use_tf ? P.tf[i] : 1;
            if (cnt[d] == 0) sc.touched.push_back(d);
            acc[d] = acc[d] + bm25_term_score(weight, cache[P.fieldnorm_id[d]], tf);
            cnt[d]++;
        }
    }
    auto cmp = [](const DocScore& a, const DocScore& b) { return a.score != b.score ? a.score > b.score : a.doc < b.doc; };
    std::vector<DocScore> heap;                  // the k best so far, worst on top (TopDocs' collector)
    heap.reserve(k + 1);
    uint64_t total = 0;
    for (uint32_t d : sc.touched) {
        bool match = mode == BM25_AND ? cnt[d] == n_terms : true;
        DocScore h{d, acc[d]};
        acc[d] = 0.0f;
        cnt[d] = 0;
        if (!match) continue;
        if (P.alive_bits && !((P.alive_bits[d >> 6] >> (d & 63)) & 1)) continue;
        ++total;
        if (k == 0) continue;
        if (heap.size() < k) { heap.push_back(h); std::push_heap(heap.begin(), heap.end(), cmp); }
        else if (cmp(h, heap.front())) { std::pop_heap(heap.begin(), heap.end(), cmp); heap.back() = h; std::push_heap(heap.begin(), heap.end(), cmp); }
    }
    if (total_hits) *total_hits = total;
    std::sort(heap.begin(), heap.end(), cmp);
    return heap;
}
static inline std::vector<DocScore> bm25_search(const PostingsView& P, const Bm25Stats& S, const uint32_t* terms, int n_terms, int mode,
                                                bool use_tf, size_t k, uint64_t* total_hits) {
    Bm25Scratch sc;
    return bm25_search(P, S, terms, n_terms, mode, use_tf, k, total_hits, sc);
}

}  // namespace nidx_oracle
