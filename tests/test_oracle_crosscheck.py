"""Second opinions on the oracle: small, independent pure-Python / float64 restatements of the same published formulas, written
without looking at oracle/*.hpp's structure.  They cannot pin the oracle to the reference (test_oracle_golden.py does what the
reference's own tests allow), but a slip in the C++ restatement would have to be repeated here to go unnoticed."""
import math

import numpy as np

import oracle as O
from conftest import make_queries, make_vectors


def naive_bm25(docs, n_terms, query, mode, use_tf, k1=1.2, b=0.75, weights=None, norm=None):
    """tantivy's Bm25Weight from its published formula, float64, document at a time.  docs: list of token-id lists.
    weights[term] and norm[fieldnorm id], when given, replace idf * (1 + k1) and k1 * (1 - b + b * dl / avg): fed the f32 values a
    scorer starts from (taken as exact), the float64 sum measures only that scorer's arithmetic after them."""
    n = len(docs)
    avg = sum(len(d) for d in docs) / n
    df = [sum(1 for d in docs if t in d) for t in range(n_terms)] if weights is None else None
    out = []
    for i, d in enumerate(docs):
        fid = O.fieldnorm_to_id(len(d))
        dl = O.fieldnorm_id_to_value(fid)                                # the 1-byte quantised length is what tantivy scores with
        hits = [t for t in query if t < n_terms and t in d]
        if not hits or (mode == O.BM25_AND and len(hits) < len(query)):
            continue
        s = 0.0
        for t in hits:
            tf = d.count(t) if use_tf else 1
            w = math.log(1.0 + (n - df[t] + 0.5) / (df[t] + 0.5)) * (1.0 + k1) if weights is None else float(weights[t])
            nrm = k1 * (1.0 - b + b * dl / avg) if norm is None else float(norm[fid])
            s += w * tf / (tf + nrm)
        out.append((s, i))
    out.sort(key=lambda x: (-x[0], x[1]))
    return out


def test_bm25_oracle_equals_a_naive_restatement():
    rng = np.random.default_rng(31)
    n_terms = 40
    docs = [list(rng.integers(0, n_terms, int(rng.integers(1, 60)))) for _ in range(300)]
    doc_off = np.concatenate([[0], np.cumsum([len(d) for d in docs])])
    P = O.Postings(doc_off, np.concatenate(docs).astype(np.uint32), n_terms)
    for mode, use_tf, nt in ((O.BM25_OR, True, 4), (O.BM25_OR, False, 4), (O.BM25_AND, True, 2)):
        for _ in range(6):
            query = [int(t) for t in rng.choice(n_terms, nt, replace=False)]
            want = naive_bm25(docs, n_terms, query, mode, use_tf)
            got_docs, got_sc, got_cnt, got_total = O.bm25_search(P, [query], 25, mode=mode, use_tf=use_tf)
            assert got_total[0] == len(want) and got_cnt[0] == min(25, len(want))
            c = int(got_cnt[0])
            assert np.allclose(got_sc[0, :c], [s for s, _ in want[:c]], rtol=2e-6, atol=1e-6)
            for j in range(c):                                    # same document wherever the naive scores are clearly apart
                apart = (j == 0 or want[j - 1][0] - want[j][0] > 1e-5) and (j + 1 >= len(want) or want[j][0] - want[j + 1][0] > 1e-5)
                if apart:
                    assert got_docs[0, j] == want[j][1]


def test_brute_force_oracle_equals_float64_argsort():
    v = make_vectors(800, 96, seed=33)
    v[7] = 0.0                                                    # simsimd: both norms 0 -> distance 0 only if the query is 0 too
    q = make_queries(v, 12, seed=34)
    for sim in (O.SIM_DOT, O.SIM_COSINE):
        exact = q.astype(np.float64) @ v.astype(np.float64).T
        if sim == O.SIM_COSINE:
            exact /= np.maximum(np.linalg.norm(q.astype(np.float64), axis=1)[:, None] * np.linalg.norm(v.astype(np.float64), axis=1)[None, :], 1e-300)
        ids, sc, cnt = O.brute_force(v, q, 10, sim=sim, min_score=-1.0)
        order = np.argsort(-exact, axis=1, kind="stable")[:, :10]
        assert (cnt == 10).all()
        assert np.abs(sc - np.take_along_axis(exact, order, axis=1)).max() < 2e-6
        gaps = np.abs(np.diff(np.take_along_axis(exact, np.argsort(-exact, axis=1)[:, :11], axis=1), axis=1)) > 1e-5
        clear = np.concatenate([np.ones((len(q), 1), bool), gaps[:, :9]], axis=1) & gaps[:, :10]
        assert (ids[clear] == order[clear]).all()


def test_built_graph_invariants():
    """hnsw/params.rs:24-31 and build.rs:104-119: degree caps per layer, links stay inside their layer, rows are left packed,
    weights are the similarities, no duplicates and no self links -- except on the entry point: `insert` starts every search at
    the entry point, so the entry point finds ITSELF (similarity 1), links to itself and gets the reverse link too
    (build.rs:104-119 has no self check).  The reference does the same; the visited set makes it harmless."""
    v = make_vectors(1500, 48, seed=35)
    g = O.hnsw_build(v, M=6, M0=12, efC=30, max_batch=16, nthreads=4)
    assert (g.level == O.assign_levels(len(v), 6, 2)).all() and g.level[g.entry_node] == g.entry_layer == g.level.max()
    for node in range(len(v)):
        for layer in range(int(g.level[node]) + 1):
            row = g.adj0[node] if layer == 0 else g.adjU[int(g.upper_off[node]) + layer - 1]
            w = g.w0[node] if layer == 0 else g.wU[int(g.upper_off[node]) + layer - 1]
            k = int((row != O.NIL).sum())
            assert (row[:k] != O.NIL).all() and (row[k:] == O.NIL).all()
            assert k <= (12 if layer == 0 else 6)
            if node == g.entry_node:
                assert row[:k].tolist().count(node) == 2 and len(set(row[:k].tolist())) == k - 1
            else:
                assert node not in row[:k] and len(set(row[:k].tolist())) == k
            assert (g.level[row[:k]] >= layer).all()
            for t, wt in zip(row[:k], w[:k]):
                assert abs(float(wt) - O.cosine(v[node], v[int(t)])) < 1e-6
    deg0 = (g.adj0 != O.NIL).sum(1)
    assert deg0.min() >= 1                                                          # nobody is left without a link


# ---- a literal Python transcription of hnsw/search.rs (heapq, sets) against the oracle's C++ walk ---------------------------------
import heapq


class _Key:
    """Ordering of Cnx / CnxWithBound (search.rs:87-123: f32 total_cmp on the score) with the oracle's documented tie rule: of two
    equal scores the lower id ranks higher (the reference leaves ties to BinaryHeap / sort_unstable)."""
    __slots__ = ("id", "score")

    def __init__(self, id, score):
        self.id, self.score = int(id), float(score)

    def rank(self):
        return (self.score, -self.id)

    def __lt__(self, other):
        return self.rank() < other.rank()


class _Max(_Key):                      # heapq is a min-heap: invert for BinaryHeap<Cnx>
    def __lt__(self, other):
        return self.rank() > other.rank()


def py_layer_search(sim, edges, k, entry_points):
    """search.rs:242-304."""
    visited = set()
    candidates, ms = [], []            # BinaryHeap<CnxWithBound> (max), BinaryHeap<Reverse<CnxWithBound>> (min)
    for ep in entry_points:
        visited.add(ep)
        s = sim(ep)
        heapq.heappush(candidates, _Max(ep, s))
        heapq.heappush(ms, _Key(ep, s))
    while candidates:
        c = heapq.heappop(candidates)
        ws = ms[0].score
        if c.score < ws:
            break
        for y in edges(c.id):
            if y not in visited:
                visited.add(y)
                s = sim(y)
                if s > ws or len(ms) < k:
                    heapq.heappush(candidates, _Max(y, s))
                    heapq.heappush(ms, _Key(y, s))
                    if len(ms) > k:
                        heapq.heappop(ms)
                    ws = ms[0].score
    return sorted(ms, key=lambda x: x.rank(), reverse=True)


def py_search(sim, g, vecs, k, ef, min_score, filter_bits, with_duplicates):
    """search.rs:306-383 (dense query) + closest_up_nodes 188-240 + NodeFilter::passes 147-170."""
    eps = [g.entry_node]
    for layer in range(g.entry_layer, 0, -1):
        eps = [x.id for x in py_layer_search(sim, lambda n, l=layer: g.edges(n, l), 1, eps)]
    neighbours = py_layer_search(sim, lambda n: g.edges(n, 0), max(k, ef), eps)
    results, accepted = [], []
    visited = {x.id for x in neighbours}
    candidates = sorted(neighbours, key=lambda x: x.rank())          # ascending; pop() takes the best
    while candidates:
        c = candidates.pop()
        if c.score < min_score:
            break
        passes = not np.isnan(c.score)
        if passes and filter_bits is not None:
            passes = bool((int(filter_bits[c.id >> 6]) >> (c.id & 63)) & 1)
        if passes and not with_duplicates:
            passes = not any(vecs[a].tobytes() == vecs[c.id].tobytes() for a in accepted)
            if passes:
                accepted.append(c.id)
        if passes:
            results.append(c)
        if len(results) == k:
            break
        for y in g.edges(c.id, 0):
            if y not in visited:
                visited.add(y)
                s = sim(y)
                if s >= min_score:
                    candidates.append(_Key(y, s))
        candidates.sort(key=lambda x: x.rank())
    return sorted(results, key=lambda x: x.rank(), reverse=True)


def test_oracle_walk_equals_the_python_transcription():
    v = make_vectors(1500, 32, seed=36)
    v[900:904] = v[20:24]                                            # exact duplicates
    g = O.hnsw_build(v, M=6, M0=12, efC=30, max_batch=8, nthreads=4)
    q = np.concatenate([make_queries(v, 12, seed=37), v[20:22]])
    keep = np.random.default_rng(5).random(len(v)) < 0.5
    words = np.zeros((len(v) + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(keep, bitorder="little")
    words[: len(pb)] = pb
    bits = words.view(np.uint64)
    for filter_bits, with_duplicates, min_score, ef in ((None, True, -1.0, 20), (bits, False, 0.0, 20), (bits, True, 0.2, 5)):
        ids, sc, cnt, _ = O.hnsw_search(v, g, q, 7, ef, min_score=min_score, with_duplicates=with_duplicates, filter_bits=filter_bits)
        for qi in range(len(q)):
            want = py_search(lambda x: O.cosine(v[x], q[qi]), g, v, 7, ef, min_score, filter_bits, with_duplicates)
            assert cnt[qi] == len(want)
            assert ids[qi, : cnt[qi]].tolist() == [x.id for x in want]
            assert sc[qi, : cnt[qi]].tolist() == [np.float32(x.score) for x in want]


def py_select_neighbours(pair_sim, k, candidates):
    """build.rs:57-95.  candidates: [(id, similarity to the new node)] in the given order."""
    results, discarded = [], []
    for x, s in candidates:
        if len(results) == k:
            break
        if all(s > pair_sim(x, y) for y, _ in results):
            results.append((x, s))
        else:
            heapq.heappush(discarded, _Max(x, s))
    if len(results) < k:
        while len(results) < k and discarded:
            d = heapq.heappop(discarded)
            results.append((d.id, d.score))
        results.sort(key=lambda t: (-t[1], t[0]))
    return results


def test_oracle_build_equals_the_python_transcription():
    """build.rs:104-166 one node at a time (the reference with a single rayon thread, in the oracle's insertion order: entry point
    first, then ascending id) against hnsw_build(max_batch = 1), edge for edge."""
    n, M, M0, efC = 260, 4, 8, 12
    v = make_vectors(n, 24, seed=38)
    g = O.hnsw_build(v, M=M, M0=M0, efC=efC, max_batch=1)
    level = O.assign_levels(n, M, 2)
    top = int(level.max())
    entry = int(np.nonzero(level == top)[0][0])
    out = [{int(i): [] for i in np.nonzero(level >= l)[0]} for l in range(top + 1)]      # RAMLayer.out per layer
    pair = lambda a, b: O.cosine(v[a], v[b])
    prune_m = lambda m: m * 95 // 100                                                     # params.rs:29-31
    for x in [entry] + [i for i in range(n) if i != entry]:
        eps, found = [entry], {}
        for l in range(top, -1, -1):                                                       # insert(): top-down search
            in_layer = l <= level[x]
            res = py_layer_search(lambda y: pair(y, x), lambda node, l=l: [t for t, _ in out[l][node]], efC if in_layer else 1, eps)
            eps = [r.id for r in res]
            if in_layer:
                found[l] = [(r.id, r.score) for r in res]
        for l in range(0, int(level[x]) + 1):                                              # then link bottom-up (layer_insert)
            mmax = M0 if l == 0 else M
            neighbours = py_select_neighbours(pair, M, found[l])
            out[l][x] = list(neighbours)
            for y, s in neighbours:
                out[l][y].append((x, s))
                if len(out[l][y]) > mmax:
                    out[l][y] = py_select_neighbours(pair, prune_m(mmax), out[l][y])
    assert g.entry_node == entry and g.entry_layer == top
    for l in range(top + 1):
        for node, edges in out[l].items():
            assert g.edges(node, l).tolist() == [t for t, _ in edges], (l, node)


def test_rabitq_oracle_equals_a_numpy_transcription():
    """rabitq.rs:75-106 (encode), 124-157 (query planes), 166-218 (dot, similarity) in numpy float32, operation by operation."""
    f32 = np.float32
    d = 192
    rng = np.random.default_rng(39)
    v = rng.standard_normal((50, d)).astype(f32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    v[3, :5] = 0.0
    q = rng.standard_normal((4, d)).astype(f32)
    enc = O.rabitq_encode(v)
    assert enc.shape == (50, d // 8 + 8)
    bits = np.unpackbits(enc[:, 8:], axis=1, bitorder="little")[:, :d].astype(bool)          # u64 LE words, bit i % 64 of word i / 64
    assert (bits == (v > 0)).all()                                                            # `> 0.0`: zero goes to the negative side
    assert (enc[:, 4:8].copy().view(np.uint32)[:, 0] == (v > 0).sum(1)).all()                 # sum_bits
    dqo = enc[:, 0:4].copy().view(f32)[:, 0]                                                  # dot(v, sign(v) / sqrt(d))
    assert np.abs(dqo - np.abs(v).sum(1, dtype=np.float64) / np.sqrt(d)).max() < 1e-6
    for qi in range(len(q)):
        low, hi = q[qi].min(), f32(q[qi].max() + f32(0.00001))
        delta = f32(f32(hi - low) / f32(16.0))
        wq = (f32(q[qi] - low) / delta).astype(np.uint64)
        planes, olow, odelta, osum = O.rabitq_query(q[qi])
        assert olow == low and odelta == delta and osum == int(wq.sum())
        for b in range(4):
            want = np.packbits(((wq >> np.uint64(b)) & np.uint64(1)).astype(np.uint8), bitorder="little").view(np.uint64)
            assert (planes[b] == want).all()
        est, err = O.rabitq_estimate(enc, d, q[qi : qi + 1])
        root_dim = f32(np.sqrt(f32(d)))
        for i in range(len(v)):
            dot = f32(int((wq * bits[i]).sum()))                                              # d0 + 2 d1 + 4 d2 + 8 d3
            sum_bits = f32(int(bits[i].sum()))
            dqq = f32(f32(f32(f32(f32(2.0) * delta) / root_dim) * dot) + f32(f32(f32(f32(2.0) * low) * sum_bits) / root_dim))
            dqq = f32(f32(dqq - f32(f32(delta * f32(int(wq.sum()))) / root_dim)) - f32(low * root_dim))
            assert est[0, i] == f32(dqq / dqo[i])
            d2 = f32(dqo[i] * dqo[i])
            assert err[0, i] == f32(f32(f32(np.sqrt(f32(f32(f32(1.0) - d2) / d2))) * f32(1.9)) / root_dim)


def test_rabitq_scan_and_rerank_equal_a_python_transcription():
    """segment.rs:581-608 + rabitq.rs:222-244: estimate every vector, keep upper_bound >= min_score, then rerank_top in address
    order (exact similarity only when the bound could still beat the k-th best)."""
    d, k = 128, 5
    v = make_vectors(400, d, seed=40)
    q = make_queries(v, 6, seed=41)
    enc = O.rabitq_encode(v)
    for min_score in (0.0, 0.4):
        ids, sc, cnt, evals = O.rabitq_brute_force(v, enc, q, k, min_score=min_score)
        est, err = O.rabitq_estimate(enc, d, q)
        for qi in range(len(q)):
            best, best_k, n_exact = [], 0.0, 0                       # BinaryHeap<Reverse<Cnx>> as a min-heap of (score, -id)
            for addr in range(len(v)):
                upper = np.float32(est[qi, addr] + err[qi, addr])
                if not upper >= np.float32(min_score):
                    continue
                if len(best) < k or best_k < upper:
                    real = O.dot(v[addr], q[qi])
                    n_exact += 1
                    if real >= min_score and (len(best) < k or best_k < real):
                        heapq.heappush(best, _Key(addr, real))
                        if len(best) > k:
                            heapq.heappop(best)
                        best_k = best[0].score
            want = sorted(best, key=lambda x: x.rank(), reverse=True)
            assert cnt[qi] == len(want) and evals[qi] == n_exact
            assert ids[qi, : cnt[qi]].tolist() == [x.id for x in want] and sc[qi, : cnt[qi]].tolist() == [np.float32(x.score) for x in want]
