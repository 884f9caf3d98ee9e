"""GPU tests for the BM25 kernel (through the C ABI).  Two pins:
  * bit for bit against tests/bm25_model.py, the host restatement of the kernel's fixed-point arithmetic: ids, scores, counts and
    totals are equal, everywhere;
  * within a stated tolerance against the oracle's restatement of tantivy (a float32 sum).  Parity with tantivy itself is unpinned
    (SURVEY F9)."""
import numpy as np
import pytest

import bm25_model as M
import oracle as O
from nucliadb_b200 import _lib
from nucliadb_b200.segment import TextSegment

pytestmark = pytest.mark.gpu


def corpus(n_docs, n_terms, seed, mean_len=40):
    rng = np.random.default_rng(seed)
    lens = np.maximum(1, rng.lognormal(np.log(mean_len), 0.6, n_docs).astype(np.int64))
    doc_off = np.concatenate([[0], np.cumsum(lens)])
    tokens = (rng.zipf(1.2, int(doc_off[-1])) - 1) % n_terms
    return O.Postings(doc_off, tokens.astype(np.uint32), n_terms)


def alive_words(alive):
    words = np.zeros((len(alive) + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(alive, bitorder="little")
    words[: len(pb)] = pb
    return words.view(np.uint64)


def pack(queries):
    qoff = np.concatenate([[0], np.cumsum([len(x) for x in queries])]).astype(np.uint32)
    qt = np.concatenate([np.asarray(x, dtype=np.uint32) for x in queries]) if qoff[-1] else np.zeros(0, np.uint32)
    return qt, qoff


def default_stats(P, stats):
    """stats = (total_docs, total_tokens, doc_freq); default: the segment's own exact ones (an empty segment keeps what
    nidx_txt_create sets: None)."""
    return (P.n_docs, P.total_tokens, P.doc_freq) if stats is None and P.n_docs else stats


def model_for(P, alive=None, stats=None):
    stats = default_stats(P, stats)
    if stats is None:
        return M.Bm25Model(P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id, alive_bits=alive)
    return M.Bm25Model.of(P, total_docs=stats[0], total_tokens=stats[1], doc_freq=stats[2], alive_bits=alive)


def segment(P, alive=None, stats=None):
    """The segment and its model."""
    ts = TextSegment.create(P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id)
    stats = default_stats(P, stats)
    if stats is not None:
        ts.set_stats(*stats)
    if alive is not None:
        ts.set_alive(alive)
    return ts, model_for(P, alive, stats)


def search(ts, queries, k, mode, use_tf, device=False, **kw):
    qt, qoff = pack(queries)
    if not device:
        return ts.search(qt, qoff, k, mode=mode, use_tf=use_tf, **kw)
    import torch

    out = ts.search(torch.tensor(qt.astype(np.int64), dtype=torch.int32, device="cuda"), torch.tensor(qoff.astype(np.int64), dtype=torch.int32, device="cuda"),
                    k, mode=mode, use_tf=use_tf, **kw)
    torch.cuda.synchronize()
    d, s, c, t = (x.cpu().numpy() for x in out)
    return d.view(np.uint32), s, c, t.view(np.uint64)


def assert_equal_to_model(got, want):
    docs, sc, cnt, total = got
    wd, ws, wc, wt = want
    assert np.array_equal(total, wt), "Count differs from the model"
    assert np.array_equal(cnt, wc), "result counts differ from the model"
    assert np.array_equal(docs, wd), "ids differ from the model"
    assert np.array_equal(sc.view(np.uint32), ws.view(np.uint32)), "scores differ from the model"


def run(P, queries, k, mode, use_tf, min_score=0.0, alive=None, stats=None, after=None, docaddr_base=0, device=False):
    """The kernel's top-k, asserted equal to the model's bit for bit."""
    ts, model = segment(P, alive, stats)
    got = search(ts, queries, k, mode, use_tf, device=device, min_score=min_score, after=after, docaddr_base=docaddr_base)
    assert_equal_to_model(got, model.search(queries, k, mode, use_tf, min_score=min_score, after=after, docaddr_base=docaddr_base))
    ts.close()
    return got


def oracle_agrees(P, queries, k, mode, use_tf, got, alive=None, stats=None):
    """The tantivy-side pin: Count exact; scores within 1e-5 (relative and absolute), widened only where the model's error bound
    plus the oracle's own f32 error is larger (shifts well below 24); ids wherever the oracle's neighbours are further apart than
    that; a document only one side returns must tie the k-th score within that tolerance."""
    docs, sc, cnt, total = got
    model = model_for(P, alive, stats)
    kw = {} if stats is None else dict(total_docs=stats[0], total_tokens=stats[1], doc_freq=stats[2])
    od, osc, oc, otot = O.bm25_search(P, queries, k + 1, mode=mode, use_tf=use_tf, alive_bits=alive, nthreads=4, **kw)
    assert (total == otot).all() and (cnt == np.minimum(oc, k)).all()
    for q, query in enumerate(queries):
        c = int(cnt[q])
        if c == 0:
            continue
        md, msc, _, csum, npost, s = model.ranked(query, mode, use_tf)
        tol_of = dict(zip(md.tolist(), np.maximum(1e-5 * np.maximum(1.0, msc), M.error_bound(msc, csum, npost, s) + 3.03 * npost * M.U * csum)))
        tol = np.array([tol_of[int(d)] for d in docs[q, :c]])
        assert (np.abs(sc[q, :c].astype(np.float64) - osc[q, :c]) <= tol).all()
        n_o = int(min(oc[q], k + 1))
        otol = np.array([tol_of[int(d)] for d in od[q, :n_o]])
        gaps = np.diff(osc[q, :n_o].astype(np.float64)) < -(otol[:-1] + otol[1:])
        strict = (np.concatenate([[True], gaps]) & np.concatenate([gaps, [True]]))[:c]
        assert (docs[q, :c][strict] == od[q, :c][strict]).all()
        mine, theirs = set(docs[q, :c].tolist()), set(od[q, :c].tolist())
        if oc[q] <= k:
            assert mine == theirs
        for d in mine - theirs:
            assert abs(float(sc[q, docs[q, :c].tolist().index(d)]) - float(osc[q, c - 1])) <= 2 * tol_of[d]
        for d in theirs - mine:
            assert abs(float(osc[q, od[q, :c].tolist().index(d)]) - float(sc[q, c - 1])) <= 2 * tol_of[d]


def check_against_oracle(P, queries, k, mode, use_tf, alive=None, stats=None, device=False):
    got = run(P, queries, k, mode, use_tf, alive=alive, stats=stats, device=device)
    oracle_agrees(P, queries, k, mode, use_tf, got, alive=alive, stats=stats)
    return got


@pytest.mark.parametrize("mode,use_tf", [(_lib.NIDX_BM25_OR, False), (_lib.NIDX_BM25_OR, True), (_lib.NIDX_BM25_AND, True)])
def test_bm25_matches_oracle(mode, use_tf):
    P = corpus(60000, 5000, seed=7)
    rng = np.random.default_rng(1)
    nterms = 3 if mode == _lib.NIDX_BM25_AND else 12
    queries = [list(rng.choice(400, nterms, replace=False) + (0 if mode == _lib.NIDX_BM25_AND else 20)) for _ in range(40)]
    host = check_against_oracle(P, queries, 100, mode, use_tf)
    dev = run(P, queries, 100, mode, use_tf, device=True)   # device buffers: the same bytes
    for a, b in zip(host, dev):
        assert np.array_equal(a, b)


def test_bm25_ties_keep_doc_order():
    # tf == 1 and equal lengths => exactly equal scores: TopDocs orders by doc id ascending; the k-th place falls inside runs of
    # ties, and k = 1000 / 1024 lie above the match count of [10]
    n_docs, n_terms = 5000, 50
    doc_off = np.arange(0, (n_docs + 1) * 8, 8)
    rng = np.random.default_rng(3)
    tokens = np.concatenate([rng.choice(n_terms, 8, replace=False) for _ in range(n_docs)]).astype(np.uint32)
    P = O.Postings(doc_off, tokens, n_terms)
    queries = [[1, 2, 3], [10], [4, 40]]
    for k in (1, 7, 50, 1000, 1024):
        docs, sc, cnt, total = check_against_oracle(P, queries, k, _lib.NIDX_BM25_OR, False)
        od, osc, oc, otot = O.bm25_search(P, queries, k, mode=O.BM25_OR, use_tf=False)
        assert (docs == od).all() and (cnt == oc).all() and (total == otot).all()


def test_bm25_min_score_alive_and_missing_terms():
    P = corpus(20000, 2000, seed=9)
    alive = np.ones(P.n_docs, dtype=bool)
    alive[::2] = False
    bits = alive_words(alive)
    queries = [[5, 6, 7], [1999999], [], [3, 1999999]]
    docs, sc, cnt, total = check_against_oracle(P, queries, 20, _lib.NIDX_BM25_OR, True, alive=bits)
    assert all(alive[d] for d in docs[docs != 0xFFFFFFFF])
    # AND with an unknown term matches nothing (tantivy: empty term => empty intersection)
    d2, s2, c2, t2 = run(P, [[3, 1999999]], 20, _lib.NIDX_BM25_AND, True)
    assert c2[0] == 0 and t2[0] == 0
    # min_score cut after top-k (nidx_text/src/reader.rs:302-305), at a returned score: the document holding it stays
    d0, s0, c0, _ = run(P, [[5, 6, 7]], 20, _lib.NIDX_BM25_OR, True)
    thr = float(s0[0, 7])
    d3, s3, c3, _ = run(P, [[5, 6, 7]], 20, _lib.NIDX_BM25_OR, True, min_score=thr)
    assert c3[0] == int((s0[0, : c0[0]] >= thr).sum()) and (s3[0, : c3[0]] >= thr).all() and c3[0] >= 8
    assert (d3[0, : c3[0]] == d0[0, : c3[0]]).all()


def test_bm25_dense_tiles_fall_back_to_fine_tiles():
    """Few documents, long documents, frequent terms: a fine tile (4096 docs) holds far more postings than a round has slots,
    so the tile span drops to one fine tile processed in several rounds (postings re-read in phase C, runs located by binary
    search instead of the octet map)."""
    P = corpus(30000, 60, seed=21, mean_len=120)
    rng = np.random.default_rng(4)
    queries = [list(rng.choice(60, 40, replace=False)) for _ in range(6)]
    check_against_oracle(P, queries, 100, _lib.NIDX_BM25_OR, True)
    check_against_oracle(P, queries, 100, _lib.NIDX_BM25_OR, False)
    check_against_oracle(P, [q[:3] for q in queries], 100, _lib.NIDX_BM25_AND, True)


def test_bm25_sparse_query_spans_many_fine_tiles_per_tile():
    """Rare terms over many documents: one tile covers the maximum span of fine tiles (terms without a skip row are walked
    linearly), and the threshold-crossing candidate list carries the top-k from tile to tile."""
    P = corpus(300000, 40000, seed=23, mean_len=30)
    df = np.diff(P.term_off.astype(np.int64))
    rng = np.random.default_rng(5)
    rare = np.nonzero((df >= 3) & (df < 200))[0]
    mid = np.nonzero(df >= 300)[0]
    queries = [list(rng.choice(rare, 30, replace=False)) for _ in range(8)] + [list(rng.choice(mid, 20, replace=False)) for _ in range(8)]
    queries += [list(rng.choice(rare, 10, replace=False)) + list(rng.choice(mid, 10, replace=False)) for _ in range(8)]
    check_against_oracle(P, queries, 100, _lib.NIDX_BM25_OR, False)
    check_against_oracle(P, queries, 10, _lib.NIDX_BM25_OR, True)
    check_against_oracle(P, [[int(q[-1]), int(q[-2])] for q in queries[8:]], 50, _lib.NIDX_BM25_AND, True)


EDGE_DOCS = (0, 31, 32, 4095, 4096, 131071, 131072)
UNKNOWN = 999_999


def edge_corpus(n_docs):
    """Postings at the document-space edges.  Term 0 is in every document (tf 1..3); term 1 only on the edge documents (no skip
    row: df < 256), one of them with tf = 10^6 and one above the 24-bit clamp; term 2 on the edge documents and every 97th (a skip
    row once df >= 256); term 3 only in the first fine tile and term 4 only from document 131 072 on (an AND of them has no tile in
    common); terms 5..204 are Zipf background.  Fieldnorm ids 0 and 255 on the first and last documents."""
    rng = np.random.default_rng(n_docs)
    edges = sorted({d for d in EDGE_DOCS if d < n_docs} | ({n_docs - 1} if n_docs else set()))
    per_doc = [[0] * int(rng.integers(1, 4)) for _ in range(n_docs)]
    for d in edges:
        per_doc[d] += [1, 2]
    for d in range(0, n_docs, 97):
        per_doc[d].append(2)
    for d in range(0, min(n_docs, 4096), 7):
        per_doc[d].append(3)
    for d in range(131072, n_docs, 5):
        per_doc[d].append(4)
    bg = (rng.zipf(1.3, 4 * n_docs) - 1) % 200 + 5
    nb = rng.integers(0, 7, n_docs)
    pos = np.concatenate([[0], np.cumsum(nb)])
    for d in range(n_docs):
        per_doc[d] += bg[pos[d]:pos[d + 1]].tolist()
    doc_off = np.concatenate([[0], np.cumsum([len(x) for x in per_doc])]).astype(np.int64)
    tokens = np.array([t for x in per_doc for t in x], dtype=np.uint32)
    P = O.Postings(doc_off, tokens, 205)
    if n_docs:
        P.fieldnorm_id[0] = 0
        P.fieldnorm_id[-1] = 255
        b = int(P.term_off[1])
        P.post_tf[b] = 10 ** 6                        # term 1 on document 0
        if int(P.term_off[2]) - b > 1:
            P.post_tf[b + 1] = (1 << 24) + 5          # term 1 on the second edge document: stored as 0xFFFFFF
    return P, edges


@pytest.mark.parametrize("n_docs", [0, 1, 33, 4097, 131073, 262145])
def test_bm25_document_space_and_query_edges(n_docs):
    OR, AND = _lib.NIDX_BM25_OR, _lib.NIDX_BM25_AND
    P, edges = edge_corpus(n_docs)
    queries = [[0], [1], [2], [1, 2], [0, 1, 2, 7], list(range(127)), list(range(128)), [1, 1, 2], [1, UNKNOWN, 2], [UNKNOWN], [],
               [2] * 128, [9, 5]]
    and_queries = [[3, 4], [0, 1], [0, 2], [2, 2], [1, UNKNOWN], [UNKNOWN], [], [0, 3], [0, 4]]
    for k in (1, 7, 100, 1000, 1024):
        check_against_oracle(P, queries, k, OR, True)
    check_against_oracle(P, queries, 100, OR, False)
    check_against_oracle(P, queries, 1000, OR, False, device=True)
    for k in (7, 1000):
        check_against_oracle(P, and_queries, k, AND, True)
    docs = run(P, [[1], [2]], 1024, OR, True)[0]
    assert set(docs[0][docs[0] != M.NIL].tolist()) == set(edges)
    if n_docs:
        # weights inflated through the statistics: the 128-term query's shift drops to 18
        stats = (1 << 58, (P.total_tokens // n_docs) << 58, P.doc_freq)
        assert model_for(P, stats=stats).shift(list(range(128))) == 18
        check_against_oracle(P, queries, 100, OR, True, stats=stats)
        check_against_oracle(P, and_queries, 100, AND, True, stats=stats)
    if n_docs >= 33:
        every_other = np.arange(n_docs) % 2 == 1
        boundary_dead = np.ones(n_docs, dtype=bool)
        boundary_dead[edges] = False
        for alive in (every_other, np.zeros(n_docs, dtype=bool), boundary_dead):
            check_against_oracle(P, queries, 100, OR, True, alive=alive_words(alive))
            check_against_oracle(P, and_queries, 100, AND, True, alive=alive_words(alive))
        # search-after (nidx_paragraph reader.rs:379-392) at a tied score, with a non-zero docaddr_base; min_score at a returned score
        d0, s0, c0, _ = run(P, [[0]], 1024, OR, False)
        j = min(int(c0[0]) - 1, 40)
        tied = np.nonzero(s0[0, : c0[0]] == s0[0, j])[0]
        assert n_docs < 4097 or len(tied) > 1
        base = 1 << 33
        for mode in (1, 2, 3):
            run(P, [[0], [0, 2], [0, 1, 2, 7]], 100, OR, False, after=(float(s0[0, j]), mode, base + int(d0[0, j])), docaddr_base=base)
        run(P, [[0], [0, 2]], 100, OR, False, min_score=float(s0[0, j]))


def test_bm25_results_do_not_depend_on_the_batch():
    """Each query alone, all of them in one call, the call shuffled and the call with a 128-term query added give byte-identical rows
    (every query has its own fixed-point scale); the faceted search returns the same rows."""
    P = corpus(60000, 5000, seed=7)
    rng = np.random.default_rng(1)
    queries = [list(rng.choice(400, 12, replace=False) + 20) for _ in range(40)]
    long_query = list(rng.choice(P.n_terms, 128, replace=False))
    ts, model = segment(P)
    ts.set_facets([b"l\0a", b"l\0b"], np.arange(P.n_docs + 1, dtype=np.uint64), (np.arange(P.n_docs) % 2).astype(np.uint32))
    for mode, use_tf in ((_lib.NIDX_BM25_OR, True), (_lib.NIDX_BM25_OR, False), (_lib.NIDX_BM25_AND, True)):
        qs = [q[:3] for q in queries] if mode == _lib.NIDX_BM25_AND else queries
        batch = search(ts, qs, 100, mode, use_tf)
        alone = [search(ts, [q], 100, mode, use_tf) for q in qs]
        for i in range(len(qs)):
            for a, b in zip(batch, alone[i]):
                assert a[i].tobytes() == b[0].tobytes()
        perm = rng.permutation(len(qs))
        shuffled = search(ts, [qs[i] for i in perm], 100, mode, use_tf)
        with_long = search(ts, qs + [long_query], 100, mode, use_tf)
        for a, b, c in zip(batch, shuffled, with_long):
            assert a[perm].tobytes() == b.tobytes()
            assert a.tobytes() == c[: len(qs)].tobytes()
        qt, qoff = pack(qs)
        faceted = ts.search_faceted(qt, qoff, 100, [b"l"], mode=mode, use_tf=use_tf)
        for a, b in zip(batch, faceted[:4]):
            assert a.tobytes() == b.tobytes()
        assert_equal_to_model(with_long, model.search(qs + [long_query], 100, mode, use_tf))
    ts.close()
