"""The `mem` contract of include/nidx_b200.h: every entry point with a `mem` argument gives the same results, bit for bit, with host
buffers (NIDX_MEM_HOST: copies inside the call) and with device buffers (NIDX_MEM_DEVICE) -- ids, scores as bits, counts, totals,
facet counts and dates -- for every search method and the cases that stage differently (ldq != ld, NULL outputs, host or device
filter bits, formulas, an alive set, nothing matching, an empty segment).  The C ABI is called through ctypes, so NULL outputs and
padded query rows are reachable.  The last test checks that every vector search resets the per-call counters."""
import ctypes as C

import numpy as np
import pytest
import torch

import oracle as O
from nucliadb_b200 import _lib
from nucliadb_b200._lib import FilterNode, NIL, RrfSource, ShardSearchRequest, ShardSearchResponse, TxtOrder, TxtSearchParams, VecSearchParams, check, ptr
from nucliadb_b200.segment import TextSegment, VectorSegment, _facet_request

pytestmark = pytest.mark.gpu

HOST, DEVICE = _lib.NIDX_MEM_HOST, _lib.NIDX_MEM_DEVICE
D, N = 128, 3000


def _both(fn, ins, outs):
    """Runs fn(mem, in_ptrs, out_ptrs, stream) with host buffers, then with device copies of the same inputs, and asserts that every
    output is the same bytes.  ins: numpy arrays or None (NULL); outs: (count, dtype) or None (NULL).  Returns the host outputs."""
    got = []
    for mem in (HOST, DEVICE):
        if mem == HOST:
            iv = [None if a is None else np.ascontiguousarray(a) for a in ins]
            ov = [None if o is None else np.full(o[0] * np.dtype(o[1]).itemsize, 0xA5, dtype=np.uint8) for o in outs]
            stream = None
        else:
            iv = [None if a is None else torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1).copy()).cuda() for a in ins]
            ov = [None if o is None else torch.full((o[0] * np.dtype(o[1]).itemsize,), 0xA5, dtype=torch.uint8, device="cuda") for o in outs]
            stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
        check(fn(mem, [ptr(a) for a in iv], [ptr(o) for o in ov], stream))
        torch.cuda.synchronize()
        got.append([None if o is None else (o if mem == HOST else o.cpu().numpy()) for o in ov])
    for i, (h, d) in enumerate(zip(*got)):
        assert (h is None) == (d is None)
        if h is not None:
            assert np.array_equal(h, d), f"output {i}: host and device results differ"
    return [None if (o is None or h is None) else h.view(o[1]) for o, h in zip(outs, got[0])]


def _label_nodes(key):
    keys = (C.c_void_p * 1)(C.cast(C.c_char_p(key), C.c_void_p))
    lens = (C.c_uint32 * 1)(len(key))
    return (FilterNode * 1)(FilterNode(_lib.NIDX_F_LABEL, 1, keys, lens)), (keys, key)


@pytest.fixture(scope="module")
def vec():
    rng = np.random.default_rng(5)
    v = rng.standard_normal((N, D)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    seg = VectorSegment.create(v, D, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    seg.build_hnsw(seed=2, max_batch=256)
    seg.rabitq_encode()
    # labels "/a" (every third paragraph) and "/b" (every fifth)
    post = [np.arange(0, N, 3, dtype=np.uint32), np.arange(0, N, 5, dtype=np.uint32)]
    kb = np.frombuffer(b"/a/b", dtype=np.uint8).copy()
    ko = np.array([0, 2, 4], dtype=np.uint64)
    po = np.array([0, len(post[0]), len(post[0]) + len(post[1])], dtype=np.uint64)
    pp = np.concatenate(post)
    check(_lib.load().nidx_vec_set_inverted_index(seg._h, _lib.NIDX_INV_LABELS, 2, ptr(kb), ptr(ko), ptr(po), ptr(pp)))
    alive = np.packbits(rng.random(N) < 0.9, bitorder="little")
    alive = np.concatenate([alive, np.zeros((-len(alive)) % 8, np.uint8)]).view(np.uint64)
    return seg, v, alive


def _queries(rng, v, nq, ldq):
    q = np.zeros((nq, ldq), dtype=np.float32)
    q[:, :D] = v[rng.integers(0, len(v), nq)] + 0.05 * rng.standard_normal((nq, D)).astype(np.float32)
    q[:, D:] = 7.0   # padding columns the library must ignore
    return q


def _vec_search(seg, q, k, method, fbits=None, formula=None, counts=True, ef=48, matching=0):
    nq, ldq = q.shape
    L = _lib.load()

    def fn(mem, i, o, stream):
        p = VecSearchParams(k, ef, -1.0, 1, method, i[1].value if i[1] is not None else None, matching)
        if formula is not None:
            return L.nidx_vec_search_formula(seg._h, i[0], nq, ldq, mem, C.byref(p), formula, 1, o[0], o[1], o[2], stream)
        return L.nidx_vec_search(seg._h, i[0], nq, ldq, mem, C.byref(p), o[0], o[1], o[2], stream)

    return _both(fn, [q, fbits], [(nq * k, np.uint32), (nq * k, np.float32), (nq, np.int32) if counts else None])


METHODS = [("exact", _lib.NIDX_METHOD_BRUTE, 8, 10), ("tensor_core", _lib.NIDX_METHOD_BRUTE, 128, 10), ("rabitq_scan", _lib.NIDX_METHOD_BRUTE_RABITQ, 8, 10),
           ("hnsw", _lib.NIDX_METHOD_HNSW, 8, 10), ("hnsw_rabitq", _lib.NIDX_METHOD_HNSW_RABITQ, 8, 10), ("auto", _lib.NIDX_METHOD_AUTO, 8, 10)]


@pytest.mark.parametrize("name,method,nq,k", METHODS, ids=[m[0] for m in METHODS])
@pytest.mark.parametrize("ldq", [D, D + 8], ids=["ldq_eq_ld", "ldq_padded"])
def test_vec_search_host_equals_device(vec, name, method, nq, k, ldq):
    seg, v, alive = vec
    rng = np.random.default_rng(nq + ldq + method)
    q = _queries(rng, v, nq, ldq)
    fbits = np.packbits(rng.random(N) < 0.5, bitorder="little")
    fbits = np.concatenate([fbits, np.zeros((-len(fbits)) % 8, np.uint8)]).view(np.uint64)
    nodes, _keep = _label_nodes(b"/a")
    try:
        for alive_bits in (None, alive):
            seg.set_alive(alive_bits)
            ids, _, cnt = _vec_search(seg, q, k, method)
            assert (cnt > 0).all() and (ids[:k] != NIL).any()
            _vec_search(seg, q, k, method, fbits=fbits)
            _vec_search(seg, q, k, method, fbits=fbits, matching=int(N // 2))
            ids, _, _ = _vec_search(seg, q, k, method, formula=nodes)
            assert (ids[ids != NIL] % 3 == 0).all()
            _vec_search(seg, q, k, method, counts=False)
            # nothing matches: an empty result whatever the method
            ids, sc, cnt = _vec_search(seg, q, k, method, fbits=np.zeros_like(fbits))
            assert (ids == NIL).all() and (sc == 0).all() and (cnt == 0).all()
            none, _keep2 = _label_nodes(b"/zz")
            ids, _, cnt = _vec_search(seg, q, k, method, formula=none)
            assert (ids == NIL).all() and (cnt == 0).all()
    finally:
        seg.set_alive(None)


def test_vec_search_empty_segment_host_equals_device():
    seg = VectorSegment.create(np.zeros((0, D), np.float32), D, similarity=_lib.NIDX_SIM_DOT)
    seg.build_hnsw()
    q = _queries(np.random.default_rng(1), np.ones((1, D), np.float32), 4, D + 4)
    for method in (_lib.NIDX_METHOD_BRUTE, _lib.NIDX_METHOD_HNSW, _lib.NIDX_METHOD_AUTO):
        ids, sc, cnt = _vec_search(seg, q, 5, method)
        assert (ids == NIL).all() and (sc == 0).all() and (cnt == 0).all()
        _vec_search(seg, q, 5, method, counts=False)


@pytest.mark.parametrize("with_bits", [True, False])
def test_vec_filter_host_equals_device(vec, with_bits):
    seg, _, alive = vec
    L = _lib.load()
    words = (N + 63) // 64
    for alive_bits in (None, alive):
        seg.set_alive(alive_bits)
        for key in (b"/a", b"/b", b"/zz"):
            nodes, _keep = _label_nodes(key)
            counts = []

            def fn(mem, i, o, stream):
                m = C.c_uint64(0)
                r = L.nidx_vec_filter(seg._h, nodes, 1, o[0], mem, C.byref(m), stream)
                counts.append(m.value)
                return r

            out = _both(fn, [], [(words, np.uint64) if with_bits else None])
            assert counts[0] == counts[1]
            if with_bits:
                assert counts[0] == int(np.unpackbits(out[0].view(np.uint8)).sum())
    seg.set_alive(None)


@pytest.mark.parametrize("ldq", [D, D + 8])
def test_rabitq_estimate_host_equals_device(vec, ldq):
    seg, v, _ = vec
    q = _queries(np.random.default_rng(ldq), v, 6, ldq)
    L = _lib.load()
    _both(lambda mem, i, o, stream: L.nidx_vec_rabitq_estimate(seg._h, i[0], 6, ldq, mem, o[0], o[1], stream), [q],
          [(6 * N, np.float32), (6 * N, np.float32)])


@pytest.fixture(scope="module")
def txt():
    rng = np.random.default_rng(8)
    n_docs, n_terms = 1500, 150
    lens = rng.integers(5, 40, n_docs)
    doc_off = np.concatenate([[0], np.cumsum(lens)])
    P = O.Postings(doc_off, (rng.zipf(1.3, doc_off[-1]) % n_terms).astype(np.uint32), n_terms)
    t = TextSegment.create(P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id)
    t.set_stats(P.n_docs, P.total_tokens, P.doc_freq)
    keys = [b"a", b"a\0x", b"a\0y", b"b", b"b\0z"]
    ords = [sorted(rng.choice(5, int(rng.integers(0, 3)), replace=False)) for _ in range(n_docs)]
    t.set_facets(keys, np.concatenate([[0], np.cumsum([len(o) for o in ords])]), np.array([x for o in ords for x in o], dtype=np.uint32))
    created = rng.integers(0, 400, n_docs).astype(np.int64)
    created[::7] = _lib.NIDX_DATE_NONE
    t.set_dates(created, rng.integers(0, 50, n_docs).astype(np.int64))
    alive = np.packbits(rng.random(n_docs) < 0.9, bitorder="little")
    t.set_alive(np.concatenate([alive, np.zeros((-len(alive)) % 8, np.uint8)]).view(np.uint64))
    queries = [list(rng.integers(0, n_terms, int(rng.integers(1, 6)))) for _ in range(20)]
    qoff = np.concatenate([[0], np.cumsum([len(x) for x in queries])]).astype(np.uint32)
    return t, np.concatenate(queries).astype(np.uint32), qoff


@pytest.mark.parametrize("mode", [_lib.NIDX_BM25_OR, _lib.NIDX_BM25_AND])
@pytest.mark.parametrize("with_total", [True, False])
def test_txt_searches_host_equal_device(txt, mode, with_total):
    t, qt, qoff = txt
    L = _lib.load()
    nq, k = len(qoff) - 1, 12
    p = TxtSearchParams(k, mode, 1, 0.0, 0, 0.0, 0, 0)
    req, _keep = _facet_request([b"a", b"b"])
    nb = len(t.facet_buckets([b"a", b"b"])[0])
    total = (nq, np.uint64) if with_total else None
    _both(lambda mem, i, o, s: L.nidx_txt_search(t._h, i[0], i[1], nq, mem, C.byref(p), o[0], o[1], o[2], o[3], s), [qt, qoff],
          [(nq * k, np.uint32), (nq * k, np.float32), (nq, np.int32), total])
    _both(lambda mem, i, o, s: L.nidx_txt_search_faceted(t._h, i[0], i[1], nq, mem, C.byref(p), C.byref(req), o[0], o[1], o[2], o[3], o[4], s), [qt, qoff],
          [(nq * k, np.uint32), (nq * k, np.float32), (nq, np.int32), total, (nq * nb, np.uint32)])
    for field in (_lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_MODIFIED):
        for typ in (_lib.NIDX_ORDER_DESC, _lib.NIDX_ORDER_ASC):
            o_ = TxtOrder(field, typ)
            _both(lambda mem, i, o, s: L.nidx_txt_search_ordered(t._h, i[0], i[1], nq, mem, C.byref(p), C.byref(o_), None, o[0], o[1], o[2], o[3], None, s),
                  [qt, qoff], [(nq * k, np.uint32), (nq * k, np.int64), (nq, np.int32), total])
            _both(lambda mem, i, o, s: L.nidx_txt_search_ordered(t._h, i[0], i[1], nq, mem, C.byref(p), C.byref(o_), C.byref(req), o[0], o[1], o[2], o[3], o[4],
                                                                 s),
                  [qt, qoff], [(nq * k, np.uint32), (nq * k, np.int64), (nq, np.int32), total, (nq * nb, np.uint32)])
            out = _both(lambda mem, i, o, s: L.nidx_txt_list_ordered(t._h, C.byref(o_), k, mem, o[0], o[1], o[2], o[3], s), [],
                        [(k, np.uint32), (k, np.int64), (1, np.int32), (1, np.uint64) if with_total else None])
            assert out[2][0] > 0
    out = _both(lambda mem, i, o, s: L.nidx_txt_facet_count_all(t._h, C.byref(req), mem, o[0], s), [], [(nb, np.uint32)])
    assert out[0].sum() > 0


def _records(seg, v, nq, k, n_parts, dedup):
    """n_parts exchange records of one segment searched with different queries (device memory)."""
    rng = np.random.default_rng(n_parts + dedup)
    words = nq * k * (6 if dedup else 2)
    rec = torch.empty(n_parts * words, dtype=torch.int32, device="cuda")
    for part in range(n_parts):
        q = torch.from_numpy(_queries(rng, v, nq, D)).cuda()
        p = VecSearchParams(k, 48, -1.0, 1, _lib.NIDX_METHOD_HNSW, None, 0)
        check(_lib.load().nidx_vec_shard_record(seg._h, ptr(q), nq, D, DEVICE, C.byref(p), part, dedup, C.c_void_p(rec.data_ptr() + part * words * 4),
                                                C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return rec


@pytest.mark.parametrize("dedup", [0, 1])
def test_shard_merge_host_equals_device(vec, dedup):
    seg, v, _ = vec
    nq, k, n_parts = 9, 10, 3
    rec = _records(seg, v, nq, k, n_parts, dedup)
    L = _lib.load()
    for with_opt in (True, False):
        outs = [(nq * k, np.uint32), (nq * k, np.float32), (nq * k, np.int32) if with_opt else None, (nq, np.int32) if with_opt else None]
        _both(lambda mem, i, o, s: L.nidx_shard_merge(0, ptr(rec), n_parts, nq, k, dedup, 1, mem, o[0], o[1], o[2], o[3], s), [], outs)


@pytest.mark.parametrize("with_counts", [True, False])
def test_rank_fusion_host_equals_device(with_counts):
    rng = np.random.default_rng(4)
    nq, ks = 17, [12, 5]
    keys = [rng.integers(0, 40, (nq, k)).astype(np.uint64) for k in ks]
    scores = [-np.sort(-rng.random((nq, k)).astype(np.float32), axis=1) for k in ks]
    counts = [rng.integers(0, k + 1, nq).astype(np.int32) for k in ks]
    cap = sum(ks)
    L = _lib.load()

    def fn(mem, i, o, s):
        src = (RrfSource * 2)(*[RrfSource(i[3 * j].value, i[3 * j + 1].value, i[3 * j + 2].value if with_counts else None, ks[j], 1.0 + j) for j in range(2)])
        return L.nidx_rank_fusion_rrf(0, src, 2, nq, C.c_double(30.0), mem, o[0], o[1], o[2], o[3], s)

    ins = [a for j in range(2) for a in (keys[j], scores[j], counts[j])]
    _both(fn, ins, [(nq * cap, np.uint64), (nq * cap, np.float64), (nq * cap, np.uint32), (nq, np.int32)])


def _text_corpus(rng, n_docs, n_terms):
    lens = rng.integers(5, 40, n_docs)
    doc_off = np.concatenate([[0], np.cumsum(lens)])
    return O.Postings(doc_off, (rng.zipf(1.3, doc_off[-1]) % n_terms).astype(np.uint32), n_terms)


def test_shard_search_host_equals_device(vec):
    """The request shapes test_gpu_rank_fusion uses: vector + paragraph + document with fusion (both orders), paragraph only,
    vector + document without fusion."""
    seg, v, _ = vec
    rng = np.random.default_rng(12)
    nq, kv, kp, kd = 21, 10, 15, 5
    seg.set_paragraph_keys(rng.permutation(N).astype(np.uint64) + 1000)
    P = _text_corpus(rng, N, 200)
    par = TextSegment.create(P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id)
    par.set_stats(P.n_docs, P.total_tokens, P.doc_freq)
    Dc = _text_corpus(rng, 500, 120)
    doc = TextSegment.create(Dc.n_docs, Dc.n_terms, Dc.term_off, Dc.post_doc, Dc.post_tf, Dc.fieldnorm_id)
    doc.set_stats(Dc.n_docs, Dc.total_tokens, Dc.doc_freq)
    pq = [list(rng.integers(0, 200, 4)) for _ in range(nq)]
    dq = [list(rng.integers(0, 120, 2)) for _ in range(nq)]
    poff = np.concatenate([[0], np.cumsum([len(x) for x in pq])]).astype(np.uint32)
    doff = np.concatenate([[0], np.cumsum([len(x) for x in dq])]).astype(np.uint32)
    pterms, dterms = np.concatenate(pq).astype(np.uint32), np.concatenate(dq).astype(np.uint32)
    q = _queries(rng, v, nq, D + 4)
    vp = VecSearchParams(kv, 48, -1.0, 1, _lib.NIDX_METHOD_HNSW, None, 0)
    pp = TxtSearchParams(kp, _lib.NIDX_BM25_OR, 0, 0.0, 0, 0.0, 0, 0)
    dp = TxtSearchParams(kd, _lib.NIDX_BM25_AND, 1, 0.0, 0, 0.0, 0, 0)
    L = _lib.load()
    names = ["vec_ids", "vec_scores", "vec_counts", "par_docs", "par_scores", "par_counts", "par_total", "doc_docs", "doc_scores", "doc_counts", "doc_total",
             "fused_keys", "fused_scores", "fused_refs", "fused_counts"]
    for use_vec, use_par, use_doc, rrf_k, semantic_first in [(1, 1, 1, 60.0, 0), (1, 1, 1, 60.0, 1), (0, 1, 0, 0.0, 0), (1, 0, 1, 0.0, 0)]:
        fuse = rrf_k > 0 and use_vec and use_par
        sizes = dict(vec_ids=(nq * kv, np.uint32), vec_scores=(nq * kv, np.float32), vec_counts=(nq, np.int32), par_docs=(nq * kp, np.uint32),
                     par_scores=(nq * kp, np.float32), par_counts=(nq, np.int32), par_total=(nq, np.uint64), doc_docs=(nq * kd, np.uint32),
                     doc_scores=(nq * kd, np.float32), doc_counts=(nq, np.int32), doc_total=(nq, np.uint64), fused_keys=(nq * (kv + kp), np.uint64),
                     fused_scores=(nq * (kv + kp), np.float64), fused_refs=(nq * (kv + kp), np.uint32), fused_counts=(nq, np.int32))
        on = dict(vec=use_vec, par=use_par, doc=use_doc, fused=fuse)
        outs = [sizes[n] if on[n.split("_")[0]] else None for n in names]

        def fn(mem, i, o, s):
            rq, rs = ShardSearchRequest(), ShardSearchResponse()
            rq.nq = nq
            if use_vec:
                rq.vec, rq.queries, rq.ldq, rq.vec_params = seg._h.value, i[0].value, D + 4, C.pointer(vp)
            if use_par:
                rq.par, rq.par_terms, rq.par_off, rq.par_params = par._h.value, i[1].value, i[2].value, C.pointer(pp)
            if use_doc:
                rq.doc, rq.doc_terms, rq.doc_off, rq.doc_params = doc._h.value, i[3].value, i[4].value, C.pointer(dp)
            rq.rrf_k, rq.weight_keyword, rq.weight_semantic, rq.semantic_first = rrf_k, 1.0, 2.0, semantic_first
            for n, x in zip(names, o):
                setattr(rs, n, None if x is None else x.value)
            return L.nidx_shard_search(C.byref(rq), C.byref(rs), mem, s)

        _both(fn, [q, pterms, poff, dterms, doff], outs)
    seg.set_paragraph_keys(None)


def test_every_search_resets_the_counters(vec):
    """nidx_vec_counters / _ex / exact_rows / scan_counters describe the last search call: a search that does not walk the graph
    (a RaBitQ scan, a search where nothing matches, a search on an empty segment) leaves them all 0."""
    seg, v, _ = vec
    q = _queries(np.random.default_rng(3), v, 8, D)

    def counters(s):
        return [s.counters(), s.counters_ex(), s.exact_rows(), s.scan_counters()]

    def zero(c):
        return all(x == 0 for x in list(c[0].values()) + list(c[1].values()) + [c[2]] + list(c[3].values()))

    seg.search(q, 10, ef=48, method=_lib.NIDX_METHOD_HNSW)
    assert counters(seg)[0]["similarities"] > 0
    seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE_RABITQ)
    assert zero(counters(seg))
    seg.search(q, 10, ef=48, method=_lib.NIDX_METHOD_HNSW)
    seg.search(q, 10, ef=48, method=_lib.NIDX_METHOD_HNSW, filter_bits=np.zeros((N + 63) // 64, np.uint64))
    assert zero(counters(seg))
    # a segment whose rows are all deleted: until a search, the getters report its build's counters
    gone = VectorSegment.create(v[:500], D, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    gone.build_hnsw(seed=2, max_batch=64)
    assert counters(gone)[0]["similarities"] > 0
    gone.set_alive(np.zeros((500 + 63) // 64, np.uint64))
    gone.search(q, 10, ef=48, method=_lib.NIDX_METHOD_HNSW)
    assert zero(counters(gone))
    # smoke check only: an empty segment never holds stale counters (its build counts nothing, and neither can any search)
    empty = VectorSegment.create(np.zeros((0, D), np.float32), D, similarity=_lib.NIDX_SIM_DOT)
    empty.build_hnsw()
    empty.search(q, 10, method=_lib.NIDX_METHOD_HNSW)
    assert zero(counters(empty))
