// ORACLE — TEST INFRASTRUCTURE ONLY (see distance.hpp).
//
// CPU restatement of the HNSW of nidx_vector:
//   nidx/nidx_vector/src/hnsw/params.rs:20-46      level_factor, m_max_for_layer, prune_m, constants
//   nidx/nidx_vector/src/hnsw/search.rs:242-304    layer_search
//   nidx/nidx_vector/src/hnsw/search.rs:306-383    search (descent k=1, layer 0 k=max(top_k, ef))
//   nidx/nidx_vector/src/hnsw/search.rs:188-240    closest_up_nodes (filter / dedup aware expansion)
//   nidx/nidx_vector/src/hnsw/search.rs:135-171    NodeFilter::passes
//   nidx/nidx_vector/src/hnsw/build.rs:49-55       initialize_graph (levels for all nodes first)
//   nidx/nidx_vector/src/hnsw/build.rs:57-95       select_neighbours_heuristic
//   nidx/nidx_vector/src/hnsw/build.rs:97-101      get_random_layer  (round, not floor)
//   nidx/nidx_vector/src/hnsw/build.rs:104-119     layer_insert
//   nidx/nidx_vector/src/hnsw/build.rs:123-166     insert (search top-down, link bottom-up)
//   nidx/nidx_vector/src/hnsw/ram_hnsw.rs:88-107   add_node, update_entry_point
//
// Deliberate, documented differences from the reference (all where the reference itself is
// unspecified / non-deterministic, SURVEY F3/F5/Q7):
//   * M, M0, efC, ef are run-time parameters (compile-time constants 30/60/100/30 in params.rs).
//   * Exactly equal scores are ordered (score desc, id asc); the reference's order under ties is
//     whatever BinaryHeap / sort_unstable give.
//   * Entry point = lowest node id of the top layer (reference: first key of an FxHashMap).
//   * The reference inserts with rayon and per-node RwLocks (segment.rs:254-256), which is not
//     deterministic.  Here insertion is "batch synchronous": a batch of nodes searches the graph
//     frozen at the start of the batch (build.rs:123-150 per node), then the batch is linked in
//     ascending node id (build.rs:157-165, 104-119).  Batch size 1 is exactly the reference's
//     sequential semantics.  The entry-point node is inserted first.
//   * RNG for levels: rand 0.10 SmallRng = xoshiro256++ seeded with SplitMix64 from 2
//     [recalled: rand is not vendored]; only the distribution matters for graph quality.
//
// Graph storage is the flat layout shared with the CUDA library (DESIGN.md "graph layout"):
//   adj0[n][s0] u32 (0xFFFFFFFF padded), w0[n][s0] f32, level[n] u8,
//   upper_off[n] u64 = first row of the node in the upper pool, row (l-1) is layer l,
//   adjU[rows][su], wU[rows][su].
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <queue>
#include <vector>

#include "distance.hpp"

namespace nidx_oracle {

static const uint32_t NIL = 0xFFFFFFFFu;

struct Params {
    int M = 30;    // params.rs:40  (also M_MAX, params.rs:37)
    int M0 = 60;   // params.rs:34
    int efC = 100; // params.rs:43
    int ef = 30;   // params.rs:46
};
static inline int prune_m(int m) { return m * 95 / 100; }  // params.rs:29-31
static inline int stride0_for(int M0) { return (M0 + 31) / 32 * 32; }
static inline int strideU_for(int M) { return (M + 15) / 16 * 16; }

// ---- level RNG (build.rs:40, 97-101) ------------------------------------------------------
struct SmallRng {  // xoshiro256++, SplitMix64 seeding [recalled]
    uint64_t s[4];
    explicit SmallRng(uint64_t state) {
        for (int i = 0; i < 4; ++i) {
            state += 0x9e3779b97f4a7c15ull;
            uint64_t z = state;
            z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
            z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
            s[i] = z ^ (z >> 31);
        }
    }
    static uint64_t rotl(uint64_t x, int k) { return (x << k) | (x >> (64 - k)); }
    uint64_t next_u64() {
        uint64_t r = rotl(s[0] + s[3], 23) + s[0];
        uint64_t t = s[1] << 17;
        s[2] ^= s[0]; s[3] ^= s[1]; s[1] ^= s[2]; s[0] ^= s[3];
        s[2] ^= t;
        s[3] = rotl(s[3], 45);
        return r;
    }
    double uniform01() { return (double)(next_u64() >> 12) * (1.0 / 4503599627370496.0); }  // 2^-52
};
static inline void assign_levels(uint32_t n, int M, uint64_t seed, uint8_t* level) {
    SmallRng rng(seed);
    double level_factor = 1.0 / std::log((double)M);  // params.rs:20-22
    for (uint32_t i = 0; i < n; ++i) {
        double u = rng.uniform01();
        double picked = -std::log(u) * level_factor;
        double r = std::round(picked);  // Rust f64::round: half away from zero
        if (!(r < 250.0)) r = 250.0;    // u == 0 -> inf; `as usize` saturates, we clamp
        level[i] = (uint8_t)r;
    }
}

// ---- flat graph view ----------------------------------------------------------------------
struct GraphView {
    uint32_t n = 0;
    int M = 0, M0 = 0, s0 = 0, su = 0;
    const uint8_t* level = nullptr;
    uint32_t entry_node = 0, entry_layer = 0;
    uint32_t* adj0 = nullptr; float* w0 = nullptr;
    const uint64_t* upper_off = nullptr;
    uint32_t* adjU = nullptr; float* wU = nullptr;

    uint32_t* row(uint32_t node, int layer) const {
        return layer == 0 ? adj0 + (size_t)node * s0 : adjU + (upper_off[node] + (uint64_t)(layer - 1)) * su;
    }
    float* wrow(uint32_t node, int layer) const {
        return layer == 0 ? w0 + (size_t)node * s0 : wU + (upper_off[node] + (uint64_t)(layer - 1)) * su;
    }
    int stride(int layer) const { return layer == 0 ? s0 : su; }
    int mmax(int layer) const { return layer == 0 ? M0 : M; }  // params.rs:24-26
};

struct Data {
    const float* vecs = nullptr;   // [n][ld]
    const float* norms = nullptr;  // [n] norm_ordered, read for cosine and L2
    uint32_t n = 0;
    int d = 0, ld = 0, sim = SIM_DOT;
    const float* vec(uint32_t i) const { return vecs + (size_t)i * ld; }
    float nrm(uint32_t i) const { return sim != SIM_DOT ? norms[i] : 0.0f; }
};

struct Scored {
    uint32_t id;
    float score;
};
static inline bool better(const Scored& a, const Scored& b) { return rank_key(a.score, a.id) > rank_key(b.score, b.id); }
// search.rs:381 `filtered_result.sort_by(|a, b| b.1.total_cmp(&a.1))`: a STABLE sort on the score alone, so equal scores keep the
// order closest_up_nodes accepted them in (a late-found neighbour can tie with an earlier result and carry a lower id).
static inline void sort_by_score(std::vector<Scored>& r) {
    std::stable_sort(r.begin(), r.end(), [](const Scored& a, const Scored& b) { return ordered_bits(a.score) > ordered_bits(b.score); });
}

struct alignas(64) Counters {  // one cache line per thread: these are bumped on every similarity
    uint64_t n_dist = 0, n_expand = 0, n_edges_read = 0;
};

// Per-thread scratch: exact visited set as an epoch array (same semantics as the FxHashSet).
struct Scratch {
    std::vector<uint32_t> stamp;
    uint32_t epoch = 0;
    void reset(uint32_t n) {
        if (stamp.size() != n) { stamp.assign(n, 0); epoch = 0; }
        if (++epoch == 0) { std::fill(stamp.begin(), stamp.end(), 0); epoch = 1; }
    }
    bool test_and_set(uint32_t i) { if (stamp[i] == epoch) return true; stamp[i] = epoch; return false; }
    bool test(uint32_t i) const { return stamp[i] == epoch; }
};

struct Query {
    const float* q;
    float qnorm;
};
static inline float sim_to(const Data& D, const Query& q, uint32_t x, Counters* c) {
    if (c) c->n_dist++;
    return similarity(D.sim, D.vec(x), D.nrm(x), q.q, q.qnorm, D.d);
}

// hnsw/search.rs:242-304.  Returns results sorted descending.  `score(x)` is Retriever::similarity_upper_bound(x, query).score:
// the exact similarity for a dense query, the RaBitQ estimate for a quantised one (segment.rs:339-348).
// `will_need(y)` is the reference's preload pass (search.rs:276-281: Retriever::will_need_vector on every unvisited neighbour
// before the first similarity; an madvise(MADV_WILLNEED) there, vector_store.rs:91-110).  The restatement issues software
// prefetches instead, so that the CPU baseline overlaps the neighbours' memory latencies as the reference's page-cache
// read-ahead does; it cannot change a result.
struct NoPreload { void operator()(uint32_t) const {} };
template <class ScoreFn, class PreloadFn = NoPreload>
static inline std::vector<Scored> layer_search_with(uint32_t n, const GraphView& G, ScoreFn score, int layer, size_t k,
                                                    const std::vector<uint32_t>& entry_points, Scratch& sc, Counters* cnt,
                                                    PreloadFn will_need = PreloadFn()) {
    auto worse_first = [](const Scored& a, const Scored& b) { return better(a, b); };   // min-heap on rank
    auto better_first = [](const Scored& a, const Scored& b) { return better(b, a); };  // max-heap on rank
    std::priority_queue<Scored, std::vector<Scored>, decltype(better_first)> candidates(better_first);
    std::priority_queue<Scored, std::vector<Scored>, decltype(worse_first)> ms(worse_first);
    sc.reset(n);
    for (uint32_t ep : entry_points) {  // 256-261: pushed to both heaps, no k bound
        sc.test_and_set(ep);
        Scored s{ep, score(ep)};
        candidates.push(s);
        ms.push(s);
    }
    while (!candidates.empty()) {
        Scored c = candidates.top();
        candidates.pop();
        float ws = ms.top().score;
        if (c.score < ws) break;  // 268-273, strict
        if (cnt) cnt->n_expand++;
        const uint32_t* edges = G.row(c.id, layer);
        int stride = G.stride(layer);
        for (int e = 0; e < stride; ++e) {  // 276-281: preload pass over the unvisited neighbours
            uint32_t y = edges[e];
            if (y == NIL) break;
            if (!sc.test(y)) will_need(y);
        }
        for (int e = 0; e < stride; ++e) {
            uint32_t y = edges[e];
            if (y == NIL) break;
            if (cnt) cnt->n_edges_read++;
            if (sc.test_and_set(y)) continue;
            float s = score(y);
            if (s > ws || ms.size() < k) {  // 286
                candidates.push({y, s});
                ms.push({y, s});
                if (ms.size() > k) ms.pop();
                ws = ms.top().score;
            }
        }
    }
    std::vector<Scored> out;
    out.reserve(ms.size());
    while (!ms.empty()) { out.push_back(ms.top()); ms.pop(); }
    std::reverse(out.begin(), out.end());  // into_sorted_vec of Reverse => descending
    return out;
}
static inline std::vector<Scored> layer_search(const Data& D, const GraphView& G, const Query& q, int layer, size_t k,
                                               const std::vector<uint32_t>& entry_points, Scratch& sc, Counters* cnt) {
    // HnswSearcher::new(&retriever, true) on the query path (segment.rs:540); the builder passes false (build.rs:41), where the
    // prefetches are harmless.  One prefetch per 64-byte line of the row, into L2 (32 rows of 3 KB exceed L1).
    auto preload = [&](uint32_t y) {
        const char* p = reinterpret_cast<const char*>(D.vec(y));
        for (size_t off = 0; off < (size_t)D.d * 4; off += 64) __builtin_prefetch(p + off, 0, 2);
    };
    return layer_search_with(D.n, G, [&](uint32_t x) { return sim_to(D, q, x, cnt); }, layer, k, entry_points, sc, cnt, preload);
}

// hnsw/search.rs:135-171 NodeFilter + 388-412 RepCounter.
struct NodeFilter {
    const uint64_t* filter_bits = nullptr;  // bit per paragraph; nullptr = all pass
    const uint32_t* paragraph_of = nullptr; // [n] paragraph address of each vector; nullptr = identity
    bool with_duplicates = true;
    bool multi_vector = false;
    std::vector<uint32_t> accepted;             // accepted vector addrs (for byte-equality dedup)
    std::vector<uint32_t> accepted_paragraphs;
    bool passes(const Data& D, uint32_t v) {
        uint32_t p = paragraph_of ? paragraph_of[v] : v;
        if (filter_bits && !((filter_bits[p >> 6] >> (p & 63)) & 1)) return false;
        if (!with_duplicates)
            for (uint32_t a : accepted)
                if (std::memcmp(D.vec(a), D.vec(v), sizeof(float) * D.d) == 0) return false;
        if (multi_vector) {
            for (uint32_t ap : accepted_paragraphs) if (ap == p) return false;
            accepted_paragraphs.push_back(p);
        }
        if (!with_duplicates) accepted.push_back(v);
        return true;
    }
};

// hnsw/search.rs:188-240.
static inline std::vector<Scored> closest_up_nodes(const Data& D, const GraphView& G, const Query& q, std::vector<Scored> entry_points,
                                                   size_t number_of_results, float min_score, NodeFilter& filter, Scratch& sc,
                                                   Counters* cnt) {
    std::vector<Scored> results;
    sc.reset(D.n);
    for (auto& e : entry_points) sc.test_and_set(e.id);
    std::vector<Scored> candidates = std::move(entry_points);
    auto asc = [](const Scored& a, const Scored& b) { return better(b, a); };
    std::sort(candidates.begin(), candidates.end(), asc);
    while (!candidates.empty()) {
        Scored c = candidates.back();
        candidates.pop_back();
        if (c.score < min_score) break;                                    // 206
        if (!(c.score != c.score) && filter.passes(D, c.id)) results.push_back(c);  // 210
        if (results.size() == number_of_results) break;                    // 214
        if (cnt) cnt->n_expand++;
        const uint32_t* edges = G.row(c.id, 0);
        for (int e = 0; e < G.s0; ++e) {
            uint32_t y = edges[e];
            if (y == NIL) break;
            if (cnt) cnt->n_edges_read++;
            if (sc.test_and_set(y)) continue;
            float s = sim_to(D, q, y, cnt);
            if (s >= min_score) candidates.push_back({y, s});              // 231
        }
        std::sort(candidates.begin(), candidates.end(), asc);              // 236
    }
    return results;
}

// hnsw/search.rs:306-383 (dense f32 path; the RaBitQ branch is a "next" row, SURVEY 8f).
static inline std::vector<Scored> hnsw_search(const Data& D, const GraphView& G, const Query& q, size_t k_neighbours, int ef,
                                              float min_score, NodeFilter& filter, Scratch& sc, Counters* cnt) {
    if (k_neighbours == 0 || D.n == 0) return {};
    std::vector<uint32_t> eps{G.entry_node};
    for (int layer = (int)G.entry_layer; layer > 0; --layer) {
        auto r = layer_search(D, G, q, layer, 1, eps, sc, cnt);
        eps.clear();
        for (auto& s : r) eps.push_back(s.id);
    }
    size_t last_k = std::max(k_neighbours, (size_t)ef);  // 338-345
    auto neighbours = layer_search(D, G, q, 0, last_k, eps, sc, cnt);
    auto filtered = closest_up_nodes(D, G, q, neighbours, k_neighbours, min_score, filter, sc, cnt);
    sort_by_score(filtered);  // 381
    return filtered;
}

// ---- build --------------------------------------------------------------------------------
// build.rs:57-95.  cand: (id, sim-to-the-new-node) in the given order.
static inline std::vector<Scored> select_neighbours_heuristic(const Data& D, size_t k, const std::vector<Scored>& cand, Counters* cnt) {
    std::vector<Scored> results;
    auto better_first = [](const Scored& a, const Scored& b) { return better(b, a); };
    std::priority_queue<Scored, std::vector<Scored>, decltype(better_first)> discarded(better_first);
    for (const Scored& x : cand) {
        if (results.size() == k) break;
        bool check = true;
        for (const Scored& y : results) {
            if (cnt) cnt->n_dist++;
            float inter = similarity(D.sim, D.vec(x.id), D.nrm(x.id), D.vec(y.id), D.nrm(y.id), D.d);
            if (!(x.score > inter)) { check = false; break; }  // .all(|inter_sim| sim > inter_sim), short-circuit
        }
        if (check) results.push_back(x); else discarded.push(x);
    }
    if (results.size() < k) {
        while (results.size() < k && !discarded.empty()) { results.push_back(discarded.top()); discarded.pop(); }
        std::sort(results.begin(), results.end(), better);
    }
    return results;
}

static inline int row_len(const uint32_t* row, int stride) {
    int c = 0;
    while (c < stride && row[c] != NIL) ++c;
    return c;
}
static inline void write_row(uint32_t* row, float* w, int stride, const std::vector<Scored>& v) {
    for (int i = 0; i < stride; ++i) {
        row[i] = i < (int)v.size() ? v[i].id : NIL;
        w[i] = i < (int)v.size() ? v[i].score : 0.0f;
    }
}

// Search half of build.rs:123-150 for one node on the frozen graph: neighbours per layer, layer 0 first.
static inline std::vector<std::vector<Scored>> insert_search(const Data& D, const GraphView& G, const Params& p, uint32_t node, Scratch& sc,
                                                             Counters* cnt) {
    Query q{D.vec(node), D.nrm(node)};
    std::vector<uint32_t> ep{G.entry_node};
    int top = G.level[node];
    std::vector<std::vector<Scored>> per_layer(top + 1);
    for (int l = (int)G.entry_layer; l >= 0; --l) {
        bool in_layer = l <= top;
        size_t k = in_layer ? (size_t)p.efC : 1;
        auto res = layer_search(D, G, q, l, k, ep, sc, cnt);
        ep.clear();
        for (auto& s : res) ep.push_back(s.id);
        if (in_layer) per_layer[l] = std::move(res);
    }
    return per_layer;
}

// build.rs:104-119 for one (node, layer).
static inline void layer_insert(const Data& D, const GraphView& G, const Params& p, uint32_t x, int layer, const std::vector<Scored>& found,
                                Counters* cnt) {
    int mmax = G.mmax(layer), stride = G.stride(layer);
    auto neighbours = select_neighbours_heuristic(D, (size_t)p.M, found, cnt);
    write_row(G.row(x, layer), G.wrow(x, layer), stride, neighbours);
    for (const Scored& y : neighbours) {
        uint32_t* row = G.row(y.id, layer);
        float* w = G.wrow(y.id, layer);
        int len = row_len(row, stride);
        std::vector<Scored> edges(len + 1);
        for (int i = 0; i < len; ++i) edges[i] = {row[i], w[i]};
        edges[len] = {x, y.score};
        if ((int)edges.size() > mmax) edges = select_neighbours_heuristic(D, (size_t)prune_m(mmax), edges, cnt);
        write_row(row, w, stride, edges);
    }
}

}  // namespace nidx_oracle
