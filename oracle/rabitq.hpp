// ORACLE — TEST INFRASTRUCTURE ONLY (see distance.hpp).
//
// CPU restatement of nidx_vector's RaBitQ 1-bit quantisation (SURVEY §8f rank 1, a9):
//   nidx/nidx_vector/src/vector_types/rabitq.rs:70-106    EncodedVector::encode  -> [f32 dot_quant_original][u32 sum_bits][dim/8 sign bits]
//   rabitq.rs:124-157                                     QueryVector::from_vector (4-bit scalar quantisation as 4 bit planes)
//   rabitq.rs:166-200                                     QueryVector::dot (AND + popcount per plane, weights 1, 2, 4, 8)
//   rabitq.rs:202-218                                     QueryVector::similarity -> (estimate, error bound), EPSILON = 1.9
//   rabitq.rs:222-244                                     rerank_top (exact re-scoring with upper-bound pruning)
//   nidx/nidx_vector/src/hnsw/search.rs:306-383           HnswSearcher::search with a SearchVector::RabitQ query: the walk ranks by
//                                                         the estimate, layer 0 asks for min(k * 100, 2000) nodes, rerank_top
//                                                         re-scores them exactly, closest_up_nodes runs on exact similarities
// Only valid for Dot similarity and dim % 64 == 0 (config.rs:170-173 quantizable_vectors).
// `f32::dot(v, v_repr)` in encode is simsimd's dot: restated with the lane-blocked order of distance.hpp.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <queue>
#include <vector>

#include "distance.hpp"
#include "hnsw.hpp"

namespace nidx_oracle {

static const float RABITQ_EPSILON = 1.9f;         // rabitq.rs:30
static const size_t RERANKING_FACTOR = 100;       // rabitq.rs:34
static const size_t RERANKING_LIMIT = 2000;       // rabitq.rs:36

static inline size_t rabitq_encoded_len(int d) { return (size_t)d / 8 + 8; }  // rabitq.rs:70-73

// rabitq.rs:75-106.  out: rabitq_encoded_len(d) bytes.
static inline void rabitq_encode(const float* v, int d, unsigned char* out) {
    float root_dim = std::sqrt((float)d);
    std::vector<uint64_t> q(d / 64, 0);
    std::vector<float> repr(d);
    uint32_t sum_bits = 0;
    float pos = 1.0f / root_dim, neg = -1.0f / root_dim;
    for (int i = 0; i < d; ++i) {
        if (v[i] > 0.0f) { q[i / 64] += (uint64_t)1 << (i % 64); sum_bits++; repr[i] = pos; }
        else repr[i] = neg;
    }
    float dqo = dot_ordered(v, repr.data(), d);
    std::memcpy(out, &dqo, 4);
    std::memcpy(out + 4, &sum_bits, 4);
    std::memcpy(out + 8, q.data(), (size_t)d / 8);
}

struct RabitqQuery {  // rabitq.rs:108-157
    std::vector<uint64_t> plane[4];
    float low = 0, delta = 0, root_dim = 0;
    uint32_t sum_quantized = 0;
    int d = 0;
    static RabitqQuery from_vector(const float* q, int d) {
        RabitqQuery r;
        r.d = d;
        float low = q[0], hi = q[0];
        for (int i = 0; i < d; ++i) { if (q[i] < low) low = q[i]; if (q[i] > hi) hi = q[i]; }
        hi = hi + 0.00001f;
        float delta = (hi - low) / 16.0f;
        for (auto& p : r.plane) p.assign(d / 64, 0);
        uint64_t sum = 0;
        for (int i = 0; i < d; ++i) {
            float f = (q[i] - low) / delta;
            uint64_t wq = f >= 0.0f ? (uint64_t)f : 0;  // `as u64`: truncation, saturating at 0
            sum += wq;
            r.plane[0][i / 64] += (wq % 2) << (i % 64);
            r.plane[1][i / 64] += ((wq / 2) % 2) << (i % 64);
            r.plane[2][i / 64] += ((wq / 4) % 2) << (i % 64);
            r.plane[3][i / 64] += ((wq / 8) % 2) << (i % 64);
        }
        r.low = low; r.delta = delta; r.sum_quantized = (uint32_t)sum; r.root_dim = std::sqrt((float)d);
        return r;
    }
    uint32_t dot(const unsigned char* enc) const {  // rabitq.rs:166-200
        const uint64_t* stored = reinterpret_cast<const uint64_t*>(enc + 8);
        uint32_t dd[4] = {0, 0, 0, 0};
        for (int p = 0; p < 4; ++p)
            for (int w = 0; w < d / 64; ++w) { uint64_t s; std::memcpy(&s, stored + w, 8); dd[p] += (uint32_t)__builtin_popcountll(plane[p][w] & s); }
        return dd[0] + dd[1] * 2 + dd[2] * 4 + dd[3] * 8;
    }
    void similarity(const unsigned char* enc, float* estimate, float* error) const {  // rabitq.rs:202-218
        float dotf = (float)dot(enc);
        float dqo; uint32_t sum_bits;
        std::memcpy(&dqo, enc, 4);
        std::memcpy(&sum_bits, enc + 4, 4);
        float dot_quant_query = 2.0f * delta / root_dim * dotf + 2.0f * low * (float)sum_bits / root_dim - delta * (float)sum_quantized / root_dim - low * root_dim;
        *estimate = dot_quant_query / dqo;
        float d2 = dqo * dqo;
        *error = std::sqrt((1.0f - d2) / d2) * RABITQ_EPSILON / root_dim;
    }
};

// rabitq.rs:222-244.  candidates in the given order: (addr, upper_bound).  Returns ascending by exact score
// (BinaryHeap<Reverse<Cnx>>::into_sorted_vec of Reverse => descending inner ... the callers re-sort anyway).
template <class ExactSim>
static inline std::vector<Scored> rerank_top(const std::vector<std::pair<uint32_t, float>>& candidates, size_t top_k, float min_score, ExactSim exact) {
    auto worse_first = [](const Scored& a, const Scored& b) { return better(a, b); };
    std::priority_queue<Scored, std::vector<Scored>, decltype(worse_first)> best(worse_first);
    float best_k = 0.0f;
    for (auto& c : candidates) {
        if (best.size() < top_k || best_k < c.second) {
            float real = exact(c.first);
            if (real >= min_score && (best.size() < top_k || best_k < real)) {
                best.push({c.first, real});
                if (best.size() > top_k) best.pop();
                best_k = best.top().score;
            }
        }
    }
    std::vector<Scored> out;
    while (!best.empty()) { out.push_back(best.top()); best.pop(); }
    std::reverse(out.begin(), out.end());
    return out;
}

// hnsw/search.rs:306-383 for a quantised query (segment.rs:506-513: data store has vectors.quant and RaBitQ search is not
// disabled).  enc: rabitq_encoded_len(d) bytes per vector.  cnt->n_dist counts EXACT similarities only; n_quant the estimates.
static inline std::vector<Scored> hnsw_search_rabitq(const Data& D, const GraphView& G, const unsigned char* enc, const Query& q,
                                                     size_t k_neighbours, float min_score, NodeFilter& filter, Scratch& sc, Counters* cnt,
                                                     uint64_t* n_quant) {
    if (k_neighbours == 0 || D.n == 0) return {};
    RabitqQuery rq = RabitqQuery::from_vector(q.q, D.d);
    size_t len = rabitq_encoded_len(D.d);
    auto estimate = [&](uint32_t x) {
        float est, err;
        rq.similarity(enc + (size_t)x * len, &est, &err);
        if (n_quant) ++*n_quant;
        return est;
    };
    std::vector<uint32_t> eps{G.entry_node};
    for (int layer = (int)G.entry_layer; layer > 0; --layer) {   // 321-327
        auto r = layer_search_with(D.n, G, estimate, layer, 1, eps, sc, cnt);
        eps.clear();
        for (auto& s : r) eps.push_back(s.id);
    }
    size_t last_k = std::min(k_neighbours * RERANKING_FACTOR, RERANKING_LIMIT);   // 335-337
    auto neighbours = layer_search_with(D.n, G, estimate, 0, last_k, eps, sc, cnt);
    std::vector<std::pair<uint32_t, float>> cand;   // (addr, upper_bound = estimate + error), best estimate first
    cand.reserve(neighbours.size());
    for (auto& s : neighbours) {
        float est, err;
        rq.similarity(enc + (size_t)s.id * len, &est, &err);
        cand.push_back({s.id, est + err});
    }
    auto reranked = rerank_top(cand, k_neighbours, min_score, [&](uint32_t v) { return sim_to(D, q, v, cnt); });   // 355-361
    auto filtered = closest_up_nodes(D, G, q, reranked, k_neighbours, min_score, filter, sc, cnt);                  // 369-375, exact
    sort_by_score(filtered);   // 381
    return filtered;
}

}  // namespace nidx_oracle
