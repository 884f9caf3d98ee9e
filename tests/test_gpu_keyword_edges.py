"""The BM25 kernel's facet, order and phrase variants and the catalogue kernels at the edges, exactly:
  * bm25_facet_kernel on the BM25 edge corpora of test_gpu_text.py (0 .. 262 145 documents, dense tiles that fall back to fine
    tiles, sparse queries over many fine tiles): counts against tests/facet_oracle.py with 1, 4 096 (the last size with shared
    counters) and 4 097 buckets, ids / scores / counts / Count equal to nidx_txt_search's;
  * bm25_order_kernel and bm25_order_facet_kernel on the same corpora: ids, dates, counts and Count against tests/order_oracle.py
    on tie- and extreme-heavy date columns with the tile-boundary documents undated;
  * phrase virtual lists over two coarse tiles (skip rows built for and read from the compacted lists) and drivers with 70 .. 100
    start positions (three or four 32-start windows) against tests/phrase_model.py: plain, faceted and ordered;
  * date_topk_all_kernel and facet_count_all_kernel over three grid-stride rounds, at n % 8 != 0 and on an empty segment, with
    alive bitsets whose padding bits past n_docs are set.
tests/test_keyword_edge_models.py checks the references on the same corpora without a GPU."""
import functools

import numpy as np
import pytest

import facet_oracle as FO
import order_oracle as OO
import phrase_model as PM
from nucliadb_b200 import _lib
from test_gpu_phrase import index, make_corpus
from test_gpu_text import UNKNOWN, alive_words, corpus, edge_corpus, pack

pytestmark = pytest.mark.gpu

OR, AND = _lib.NIDX_BM25_OR, _lib.NIDX_BM25_AND
KS = (1, 7, 100, 1000, 1024)
FIELDS = (_lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_MODIFIED)

# ---- facets and dates shared by every corpus ------------------------------------------------------------------------------------
WIDE = 4096
# /z has one child, /m has 4 096 (some with a grandchild that collapses into it), /l three levels, /k three children
KEYS = sorted({b"k", b"l", b"m", b"z", b"z\0only"} | {f"k\0{c}".encode() for c in range(3)} | {f"l\0s{a}".encode() for a in range(8)}
              | {f"l\0s{a}\0x{b}".encode() for a in range(8) for b in range(6)} | {f"m\0{i:05d}".encode() for i in range(WIDE)}
              | {f"m\0{i:05d}\0g".encode() for i in range(0, WIDE, 64)})
REQUESTS = ([b"z"], [b"m"], [b"m", b"z"], [b"l", b"k"])   # 1, 4 096 (shared counters), 4 097 (global counters) and 11 buckets
EXTREMES = [(1 << 63) - 1, -(1 << 63) + 1, -1, 0, 1, 1 << 62, -(1 << 62)]


def facets_for(n_docs, seed, long_docs=()):
    """(doc_off, ords) over KEYS: 0 .. 5 labels per document, 40 on every 61st document and on `long_docs` (ords ascending, repeats
    dropped: up to 40 ords); half of them uniform over the dictionary (mostly /m), half Zipf over its first ords (/k, /l and the
    facets themselves, which count nothing).  Every 7th document also carries /z/only, every 5th /m/00064 and /m/00064/g (two
    ords under one child)."""
    rng = np.random.default_rng(seed)
    n_lab = rng.integers(0, 6, n_docs)
    n_lab[::61] = 40
    n_lab[list(long_docs)] = 40
    t = int(n_lab.sum())
    ords = np.where(rng.random(t) < 0.5, rng.integers(0, len(KEYS), t), (rng.zipf(1.3, t) - 1) % len(KEYS))
    doc = np.repeat(np.arange(n_docs, dtype=np.int64), n_lab)
    every7, every5 = np.arange(0, n_docs, 7), np.arange(0, n_docs, 5)
    doc = np.concatenate([doc, every7, every5, every5])
    ords = np.concatenate([ords, np.full(len(every7), KEYS.index(b"z\0only")), np.full(len(every5), KEYS.index(b"m\x0000064")),
                           np.full(len(every5), KEYS.index(b"m\x0000064\0g"))])
    key = np.unique(doc * len(KEYS) + ords)
    doc_off = np.zeros(n_docs + 1, np.uint64)
    doc_off[1:] = np.cumsum(np.bincount(key // len(KEYS), minlength=n_docs))
    return doc_off, (key % len(KEYS)).astype(np.uint32)


def dates_for(n_docs, seed, undated=(), extremes=()):
    """(created, modified): created on 7 distinct dates (heavy ties), modified on ~n/3 minutes; 5 % undated, the `undated`
    documents without either date and the ends of the i64 range on the `extremes` documents."""
    rng = np.random.default_rng(seed)
    created = 1_400_000_000 + rng.integers(0, 7, n_docs).astype(np.int64) * 86_400
    modified = 1_500_000_000 + rng.integers(0, max(n_docs // 3, 1), n_docs).astype(np.int64) * 60
    created[rng.random(n_docs) < 0.05] = OO.NONE
    modified[rng.random(n_docs) < 0.05] = OO.NONE
    for i, d in enumerate(extremes):
        modified[d] = EXTREMES[i % len(EXTREMES)]
    created[list(undated)] = OO.NONE
    modified[list(undated)] = OO.NONE
    return created, modified


def padded_alive(alive):
    """The alive bitset with every padding bit past n_docs SET: no kernel may count a document that does not exist."""
    words = alive_words(alive)
    if len(alive) % 64:
        words[-1] |= np.uint64(((1 << 64) - 1) ^ ((1 << (len(alive) % 64)) - 1))
    return words


# ---- the BM25 edge corpora ------------------------------------------------------------------------------------------------------
EDGE_QUERIES = [[0], [1], [2], [1, 2], [0, 1, 2, 7], list(range(127)), list(range(128)), [1, 1, 2], [1, UNKNOWN, 2], [UNKNOWN], [],
                [2] * 128, [9, 5]]
EDGE_AND = [[3, 4], [0, 1], [0, 2], [2, 2], [1, UNKNOWN], [UNKNOWN], [], [0, 3], [0, 4]]
CORPORA = ("0", "1", "33", "4097", "131073", "262145", "dense", "sparse")


@functools.lru_cache(maxsize=None)
def edge_case(name):
    """-> dict(P, edges, queries, and_queries, doc_off, ords, created, modified, alive patterns)."""
    if name == "dense":     # test_bm25_dense_tiles_fall_back_to_fine_tiles: fine tiles of more postings than a round has slots
        P = corpus(30000, 60, seed=21, mean_len=120)
        rng = np.random.default_rng(4)
        own = [list(rng.choice(60, 40, replace=False)) for _ in range(6)]
        edges = [0, 4095, 4096, 8191, 8192, P.n_docs - 1]
        own_and = [q[:3] for q in own] + [[0, 1, 2], [0, 1], [1, 0, 3, 2]]
    elif name == "sparse":  # test_bm25_sparse_query_spans_many_fine_tiles_per_tile: rare terms over 300 000 documents
        P = corpus(300000, 40000, seed=23, mean_len=30)
        df = np.diff(P.term_off.astype(np.int64))
        rng = np.random.default_rng(5)
        rare, mid = np.nonzero((df >= 3) & (df < 200))[0], np.nonzero(df >= 300)[0]
        own = [list(rng.choice(rare, 30, replace=False)) for _ in range(4)] + [list(rng.choice(mid, 20, replace=False)) for _ in range(4)]
        own += [list(rng.choice(rare, 10, replace=False)) + list(rng.choice(mid, 10, replace=False)) for _ in range(4)]
        edges = [0, 4095, 4096, 131071, 131072, 262143, 262144, P.n_docs - 1]
        own_and = [[int(q[-1]), int(q[-2])] for q in own[4:]]
    else:
        P, edges = edge_corpus(int(name))
        own, own_and = [], []
    n = P.n_docs
    doc_off, ords = facets_for(n, n + 1, edges)
    created, modified = dates_for(n, n + 2, undated=edges[::2], extremes=edges[1::2])
    alive = [None]
    if n >= 33:
        every_other = np.arange(n) % 2 == 1
        boundary_dead = np.ones(n, dtype=bool)
        boundary_dead[edges] = False
        alive += [padded_alive(a) for a in (every_other, np.zeros(n, dtype=bool), boundary_dead)]
    return dict(P=P, edges=edges, queries=EDGE_QUERIES + own, and_queries=EDGE_AND + own_and, doc_off=doc_off, ords=ords, created=created,
                modified=modified, alive=alive)


def edge_segment(c):
    from nucliadb_b200.segment import TextSegment

    P = c["P"]
    ts = TextSegment.create(P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id)
    if P.n_docs:
        ts.set_stats(P.n_docs, P.total_tokens, P.doc_freq)
    ts.set_facets(KEYS, c["doc_off"], c["ords"])
    ts.set_dates(c["created"], c["modified"])
    return ts


def matched(c, queries, conj, alive):
    P = c["P"]
    return [FO.matched(P.n_docs, P.term_off, P.post_doc, q, conj, alive) for q in queries]


def expected_counts(c, masks, request):
    bucket, b_req, _ = FO.plan(KEYS, request)
    return np.stack([FO.count(c["doc_off"], c["ords"], bucket, len(b_req), m) for m in masks])


def assert_same_rows(got, want):
    """(docs, scores, counts, total) equal bit for bit."""
    for g, w, name in zip(got, want, ("docs", "scores", "counts", "total")):
        assert g.dtype == w.dtype and np.array_equal(g.view(np.uint32) if g.dtype == np.float32 else g,
                                                     w.view(np.uint32) if w.dtype == np.float32 else w), name


@pytest.mark.parametrize("name", CORPORA)
def test_faceted_search_at_the_bm25_edges(name):
    """bm25_facet_kernel<CONJ, TF>: every request's counts equal the oracle's; ids, scores, counts and Count equal the plain
    kernel's, at every k, under every alive pattern."""
    c = edge_case(name)
    ts = edge_segment(c)
    assert [len(FO.plan(KEYS, r)[1]) for r in REQUESTS] == [1, 4096, 4097, 11]
    try:
        for alive in c["alive"]:
            ts.set_alive(alive)
            for mode, queries in ((OR, c["queries"]), (AND, c["and_queries"])):
                qt, qoff = pack(queries)
                masks = matched(c, queries, mode == AND, alive)
                want = {tuple(r): expected_counts(c, masks, r) for r in REQUESTS}
                if alive is None and mode == OR and c["P"].n_docs:   # every request counts something, /z/only included
                    assert all(w.any() for w in want.values()) and want[(b"m", b"z")][:, WIDE].any()
                for use_tf in (False, True):
                    for k in KS:
                        plain = ts.search(qt, qoff, k, mode=mode, use_tf=use_tf)
                        assert np.array_equal(plain[3], [int(m.sum()) for m in masks])
                        for r in REQUESTS:
                            got = ts.search_faceted(qt, qoff, k, r, mode=mode, use_tf=use_tf)
                            assert_same_rows(got[:4], plain)
                            assert np.array_equal(got[4].astype(np.int64), want[tuple(r)]), (r, mode, use_tf, k)
    finally:
        ts.close()


def ordered_top(masks, secs, order_type):
    """Per mask the oracle's top 1 024 (a top k is its first k)."""
    return [OO.order_topk(m, secs, 1024, order_type) for m in masks]


def check_ordered(got, masks, top, k, plain_total):
    docs, dates, counts, total = got
    assert np.array_equal(total, plain_total)
    for i, m in enumerate(masks):
        d, s = top[i][0][:k], top[i][1][:k]
        assert int(total[i]) == int(m.sum()) and int(counts[i]) == len(d), (i, k)
        assert np.array_equal(docs[i, : len(d)].astype(np.int64), d) and np.array_equal(dates[i, : len(d)], s), (i, k)
        assert (docs[i, len(d):] == _lib.NIL).all() and (dates[i, len(d):] == OO.NONE).all()


@pytest.mark.parametrize("name", CORPORA)
def test_ordered_search_at_the_bm25_edges(name):
    """bm25_order_kernel<CONJ> for both fields and directions at every k, and bm25_order_facet_kernel with 4 096 and 4 097
    buckets: the ordered rows of the plain search and the faceted search's counts."""
    c = edge_case(name)
    ts = edge_segment(c)
    try:
        for alive in c["alive"]:
            ts.set_alive(alive)
            for mode, queries in ((OR, c["queries"]), (AND, c["and_queries"])):
                qt, qoff = pack(queries)
                masks = matched(c, queries, mode == AND, alive)
                plain_total = ts.search(qt, qoff, 1, mode=mode)[3]
                for field, secs in zip(FIELDS, (c["created"], c["modified"])):
                    for typ in (OO.DESC, OO.ASC):
                        top = ordered_top(masks, secs, typ)
                        for k in KS:
                            check_ordered(ts.search_ordered(qt, qoff, k, field, typ, mode), masks, top, k, plain_total)
                for r in ([b"m"], [b"m", b"z"]):
                    for k in (7, 1024):
                        rows = ts.search_ordered(qt, qoff, k, _lib.NIDX_ORDER_MODIFIED, OO.ASC, mode)
                        both = ts.search_ordered(qt, qoff, k, _lib.NIDX_ORDER_MODIFIED, OO.ASC, mode, facets=r)
                        assert all(np.array_equal(a, b) for a, b in zip(rows, both[:4]))
                        assert np.array_equal(both[4].astype(np.int64), expected_counts(c, masks, r)), (r, mode, k)
    finally:
        ts.close()


# ---- phrases over two coarse tiles and several start windows --------------------------------------------------------------------
N_PH = 262_145                 # two coarse tiles of 32 fine tiles and one document of a third
VOCAB = 300
R, R2 = VOCAB, VOCAB + 1       # planted terms: R rare with tf 70 .. 100, R2 on 400 documents of the second coarse tile
N_PH_TERMS = VOCAB + 2
X, A, B, C = 40, 61, 83, 120   # background terms of df ~ 10 000 .. 2 000 (the model walks a phrase's first term in Python)
R_DOCS = (0, 5, 4095, 4096, 131071, 131072, 131073, 200_000, 262_143, 262_144)
LONG_DOCS_EVERY = 6151


def plant(docs, seed):
    """Rewrite documents of make_corpus in place.  "A B" on every 131st document (a phrase of ~2 000 matches in every tile);
    R: ~40 documents (R_DOCS and every LONG_DOCS_EVERY-th) of 150 .. 200 tokens, 70 .. 100 of them R, the rest X or background,
    some starting with R, some with a dropped token; R2: 400 documents from 131 072 on, each once, followed by X on half of them.
    -> (R documents, R2 documents)."""
    rng = np.random.default_rng(seed)
    for d in range(17, N_PH, 131):   # "A B" in every fine tile
        toks = docs[d]
        j = int(rng.integers(0, len(toks) - 1))
        toks[j], toks[j + 1] = (toks[j][0], A), (toks[j + 1][0], B)
    r_docs = sorted(set(R_DOCS) | set(range(LONG_DOCS_EVERY, N_PH, LONG_DOCS_EVERY)))
    for i, d in enumerate(r_docs):
        while True:
            n = int(rng.integers(150, 201))
            kind = rng.random(n)
            ids = np.where(kind < 0.5, R, np.where(kind < 0.75, X, (rng.zipf(1.3, n) - 1) % VOCAB))
            if i % 3 == 0:
                ids[0] = R          # a start below the driver's index in "X R"
            if 70 <= int((ids == R).sum()) <= 100:
                break
        pos = np.arange(n)
        if i % 2:
            pos[n // 2:] += 1       # a token RemoveLongFilter dropped
        docs[d] = [(int(p), int(t)) for p, t in zip(pos, ids)]
    r2_docs = sorted(rng.choice(np.arange(131_072, N_PH), 400, replace=False).tolist())
    for i, d in enumerate(r2_docs):
        toks = docs[d]
        j = int(rng.integers(0, len(toks) - 1))
        toks[j] = (toks[j][0], R2)
        if i % 2:
            toks[j + 1] = (toks[j + 1][0], X)
    return r_docs, r2_docs


@functools.lru_cache(maxsize=None)
def phrase_corpus():
    """-> (docs, term_off, post_doc, post_tf, fieldnorm, pos, flat positions, R documents, R2 documents)."""
    docs = make_corpus(5, N_PH, VOCAB)
    r_docs, r2_docs = plant(docs, 6)
    return (docs, *index(docs, N_PH_TERMS), r_docs, r2_docs)


PHRASES = [[R, R], [R, X], [X, R], [R, X, R], [R, R, R], [R2, X], [X, R2], [A, B], [B, A, C], [C, B]]


def phrase_queries():
    qs = [([], [p]) for p in PHRASES]
    qs += [([X], [[R, R]]), ([A], [[R, X], [B, A]]), ([R2], [[A, B]]), ([R, X], [[R, X]]), ([C, UNKNOWN], [[X, R2], [R, R]]),
           ([], [[R, UNKNOWN]]), ([B], [])]
    return qs


@pytest.fixture(scope="module")
def phrase_seg():
    from nucliadb_b200.segment import TextSegment

    docs, term_off, post_doc, post_tf, fn, pos, flat, r_docs, r2_docs = phrase_corpus()
    df = np.diff(term_off.astype(np.int64))
    assert 70 <= post_tf[term_off[R]:term_off[R + 1]].min() and post_tf[term_off[R]:term_off[R + 1]].max() <= 100
    assert df[R2] >= 256 and post_doc[term_off[R2]] >= 131_072 and min(df[X], df[A], df[B], df[C]) >= 256
    s = TextSegment.create(N_PH, N_PH_TERMS, term_off, post_doc, post_tf, fn)
    s.set_positions(flat)
    doc_off, ords = facets_for(N_PH, 7, r_docs)
    s.set_facets(KEYS, doc_off, ords)
    created, modified = dates_for(N_PH, 8, undated=r_docs[::2], extremes=r_docs[1::2])
    s.set_dates(created, modified)
    model = PM.PhraseModel(N_PH, N_PH_TERMS, term_off, post_doc, post_tf, fn, pos=pos)
    yield s, model, doc_off, ords, created, modified
    s.close()


def run_phrases(s, qs, k, **kw):
    qt, qoff = pack([q[0] for q in qs])
    return s.search_phrases(qt, qoff, [(i, p) for i, q in enumerate(qs) for p in q[1]], k, **kw)


@pytest.mark.parametrize("mode", [OR, AND])
@pytest.mark.parametrize("use_tf", [False, True])
def test_phrases_across_coarse_tiles_and_start_windows(phrase_seg, mode, use_tf):
    s, model, doc_off, ords, created, modified = phrase_seg
    qs = phrase_queries()
    for k in (10, 1024):
        got = run_phrases(s, qs, k, mode=mode, use_tf=use_tf)
        assert_same_rows(got, model.search(qs, k, mode=mode, use_tf=use_tf))
    masks = []
    for q in qs:
        m = np.zeros(N_PH, dtype=bool)
        m[model.ranked(q, mode, use_tf)[0]] = True
        masks.append(m)
    assert masks[0][list(R_DOCS)].any() and masks[5].any()
    assert masks[7][:131_072].any() and masks[7][131_072:].any()   # "A B" in both coarse tiles
    for r in ([b"m", b"z"], [b"l", b"k"]):
        got = run_phrases(s, qs, 100, mode=mode, use_tf=use_tf, facets=r)
        assert_same_rows(got[:4], model.search(qs, 100, mode=mode, use_tf=use_tf))
        bucket, b_req, _ = FO.plan(KEYS, r)
        assert np.array_equal(got[4].astype(np.int64), np.stack([FO.count(doc_off, ords, bucket, len(b_req), m) for m in masks])), r
    total = np.asarray([m.sum() for m in masks], np.uint64)
    for field, secs in zip(FIELDS, (created, modified)):
        for typ in (OO.DESC, OO.ASC):
            got = run_phrases(s, qs, 100, mode=mode, use_tf=use_tf, order=(field, typ))
            check_ordered(got, masks, ordered_top(masks, secs, typ), 100, total)


# ---- the catalogue kernels: the empty body over every alive document ------------------------------------------------------------
def catalogue(n, seed):
    """A segment of n documents with one posting and KEYS facets -> (segment, doc_off, ords)."""
    from nucliadb_b200.segment import TextSegment

    m = min(n, 1)
    ts = TextSegment.create(n, 1, np.asarray([0, m], np.uint64), np.zeros(m, np.uint32), np.ones(m, np.uint32), np.zeros(n, np.uint8))
    doc_off, ords = facets_for(n, seed)
    ts.set_facets(KEYS, doc_off, ords)
    return ts, doc_off, ords


def check_catalogue(ts, n, doc_off, ords, alive, columns, requests, device=False):
    import torch

    mask = FO.alive_mask(n, alive)
    for field, secs in zip(FIELDS, columns):
        for typ in (OO.DESC, OO.ASC):
            want_d, want_s = OO.order_topk(mask, secs, 1024, typ)
            for k in (1, 100, 1024):
                docs, dates, count, total = ts.list_ordered(k, field, typ)
                d, s = want_d[:k], want_s[:k]
                assert total == int(mask.sum()) and count == len(d), (n, field, typ, k)
                assert np.array_equal(docs[:count].astype(np.int64), d) and np.array_equal(dates[:count], s), (n, field, typ, k)
                assert (docs[count:] == _lib.NIL).all() and (dates[count:] == OO.NONE).all()
                if device:
                    dd = ts.list_ordered(k, field, typ, device_out=True)
                    torch.cuda.synchronize()
                    assert np.array_equal(dd[0].cpu().numpy().view(np.uint32), docs) and np.array_equal(dd[1].cpu().numpy(), dates)
                    assert int(dd[2].item()) == count and int(dd[3].item()) == total
    for r in requests:
        bucket, b_req, _ = FO.plan(KEYS, r)
        want = FO.count(doc_off, ords, bucket, len(b_req), mask)
        assert np.array_equal(ts.facet_count_all(r).astype(np.int64), want), (n, r)
        if device:
            dev = ts.facet_count_all(r, device_out=True)
            torch.cuda.synchronize()
            assert np.array_equal(dev.cpu().numpy().astype(np.int64), want), (n, r)


def first_round_cover():
    """Documents the listing and the all-documents count cover in their first grid-stride round: nidx_txt_list_ordered launches
    min(2 SMs, ...) CTAs of 512 threads x DATE_PT = 8 documents, nidx_txt_facet_count_all min(8 SMs, ...) CTAs of 256 threads
    x FACET_BATCH = 4 documents."""
    import torch

    sm = torch.cuda.get_device_properties(0).multi_processor_count
    return max(2 * sm * 512 * 8, 8 * sm * 256 * 4)


def round_dates(n, cover):
    """(created, modified) of the grid-stride test: undated documents and the i64 ends on the round boundaries and the tail."""
    ends = [0, cover - 1, cover, cover + 7, 2 * cover - 1, 2 * cover, 2 * cover + 4, n - 6, n - 2, n - 1]
    return dates_for(n, 10, undated=ends[::3], extremes=ends)


def tail_columns(n):
    """(created, modified) pairs of the tail test: all documents undated, one date for all, one dated document."""
    none = np.full(n, OO.NONE, np.int64)
    one = np.full(n, 1_700_000_000, np.int64)
    single = none.copy()
    single[n // 2:n // 2 + 1] = -5
    return (none, one), (single, none), (one, single)


def random_alive(n, seed, p):
    return padded_alive(np.random.default_rng(seed).random(n) < p)


def test_catalogue_kernels_past_the_first_grid_stride_round():
    cover = first_round_cover()
    n = 2 * cover + 13          # a third, partial round; n % 8 == 5 and n % 64 == 13
    ts, doc_off, ords = catalogue(n, 9)
    try:
        columns = round_dates(n, cover)
        ts.set_dates(*columns)
        for alive in (None, random_alive(n, 11, 0.8)):
            ts.set_alive(alive)
            check_catalogue(ts, n, doc_off, ords, alive, columns, ([b"k"], [b"m"], [b"m", b"z"]), device=True)
    finally:
        ts.close()


@pytest.mark.parametrize("n", [0, 1, 7, 9, 4095, 4097])
def test_catalogue_kernels_at_the_tail(n):
    """The listing's last partial group of 8 documents and the rank column's zero padding."""
    ts, doc_off, ords = catalogue(n, 12 + n)
    try:
        for columns in tail_columns(n):
            ts.set_dates(*columns)
            for alive in [None] + ([random_alive(n, n, 0.6)] if n else []):
                ts.set_alive(alive)
                check_catalogue(ts, n, doc_off, ords, alive, columns, ([b"k"], [b"m", b"z"]), device=alive is None)
    finally:
        ts.close()
