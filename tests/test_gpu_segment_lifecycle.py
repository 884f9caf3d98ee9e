"""Segments own their device memory: a rejected or failed setter leaves the previous data in place, setting the same data again
changes no result, a create that fails after its upload raises and leaves the library usable, and segments with every optional
array set give the same results over many create / close cycles."""
import numpy as np
import pytest

from conftest import make_queries
from nucliadb_b200 import _lib
from nucliadb_b200 import vector as V
from nucliadb_b200.dist import shard_record
from nucliadb_b200.segment import VectorSegment
from test_gpu_facets import _alive, _corpus, _queries
from test_gpu_facets import _segment as _text_segment
from test_gpu_filter import _segment

pytestmark = pytest.mark.gpu

METHODS = (_lib.NIDX_METHOD_BRUTE, _lib.NIDX_METHOD_HNSW, _lib.NIDX_METHOD_BRUTE_RABITQ, _lib.NIDX_METHOD_HNSW_RABITQ)


def _formulas(pool, rids):
    return ([[V.Literal(l)] for l in pool + ["/l", "/e/PERSON", "/none"]]
            + [[V._KeyPrefixSet(frozenset(f"{r}/a/title" for r in rids[:9]))],
               [V.Operation("or", (V.Literal("/k/c"), V.Literal("/e/PERSON"))), V.Not(V.Literal("/l/b"))]])


def _set_indexes(seg):
    """What OpenSegment's constructor gives the library, given once more."""
    for which, index in ((_lib.NIDX_INV_LABELS, {k.encode(): v for k, v in seg._label_index.items()}), (_lib.NIDX_INV_FIELDS, seg._field_index)):
        keys = sorted(index)
        seg.segment.set_inverted_index(which, keys, [sorted(index[k]) for k in keys])


def _vector_results(seg, pool, rids, q):
    out = []
    for clauses in _formulas(pool, rids):
        got, matching = seg.device_filter(clauses)
        out += [got, np.int64(matching)]
        for method in (_lib.NIDX_METHOD_BRUTE, _lib.NIDX_METHOD_HNSW):
            out += list(seg.search_batch(q, 10, min_score=-1.0, with_duplicates=True, clauses=clauses, method=method))
    return out


def _text_results(seg, c, qt, qo):
    out = list(seg.search_faceted(qt, qo, 20, [b"l", b"k"]))
    out.append(seg.facet_count_all([b"l\0s3", b"k"]))
    for field in (_lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_MODIFIED):
        out += list(seg.search_ordered(qt, qo, 20, field, _lib.NIDX_ORDER_ASC, facets=[b"l"]))
        docs, dates, count, total = seg.list_ordered(50, field, _lib.NIDX_ORDER_DESC)
        out += [docs, dates, np.int64(count), np.int64(total)]
    return out


def _same(a, b):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.asarray(x).dtype == np.asarray(y).dtype and np.array_equal(np.asarray(x), np.asarray(y)), i


def _dates(c, seed):
    rng = np.random.default_rng(seed)
    created = (1_400_000_000 + rng.integers(0, 300, c["n_docs"]) * 3_600).astype(np.int64)
    created[rng.random(c["n_docs"]) < 0.1] = _lib.NIDX_DATE_NONE
    return created, created[::-1].copy()


def test_a_rejected_inverted_index_keeps_the_previous_one():
    seg, rids, pool = _segment()
    vs = seg.segment
    for which in (_lib.NIDX_INV_LABELS, _lib.NIDX_INV_FIELDS):
        with pytest.raises(_lib.NidxError):
            vs.set_inverted_index(which, [b"/l/b", b"/l/a"], [[0], [1]])        # keys out of order
        with pytest.raises(_lib.NidxError):
            vs.set_inverted_index(which, [b"/l/a", b"/l/b"], [[0], [seg.records]])   # a posting >= paragraphs
    for clauses in _formulas(pool, rids):
        got, matching = seg.device_filter(clauses)
        want = seg.filter_bitset(clauses)
        assert np.array_equal(got, want) and matching == int(want.sum()), clauses
    seg.close()


def test_setting_the_same_data_again_changes_nothing():
    seg, rids, pool = _segment(n=3000, dim=64, seed=6)
    q = make_queries(seg.host_vectors, 12, seed=3)
    once = _vector_results(seg, pool, rids, q)
    _set_indexes(seg)
    _set_indexes(seg)
    _same(once, _vector_results(seg, pool, rids, q))
    seg.close()

    c = _corpus(7, 40_000)
    created, modified = _dates(c, 8)
    ts = _text_segment(c, _alive(c["n_docs"], 9))
    ts.set_dates(created, modified)
    _, qt, qo = _queries(c, 10, 8, False)
    once = _text_results(ts, c, qt, qo)
    ts.set_facets(c["keys"], c["doc_off"], c["ords"])
    ts.set_dates(created, modified)
    _same(once, _text_results(ts, c, qt, qo))
    ts.close()


def test_a_failed_setter_keeps_the_previous_facets():
    c = _corpus(7, 5_000)
    ts = _text_segment(c)
    _, qt, qo = _queries(c, 10, 8, False)
    once = list(ts.search_faceted(qt, qo, 20, [b"l", b"k"])) + [ts.facet_count_all([b"l", b"k"])]
    bad = c["ords"].copy()
    bad[0] = len(c["keys"])                       # an ord >= n_facets
    with pytest.raises(_lib.NidxError):
        ts.set_facets(c["keys"], c["doc_off"], bad)
    _same(once, list(ts.search_faceted(qt, qo, 20, [b"l", b"k"])) + [ts.facet_count_all([b"l", b"k"])])
    ts.close()


def test_a_create_that_fails_after_the_upload_leaves_the_library_usable():
    rng = np.random.default_rng(1)
    v = rng.standard_normal((500, 64)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    par = np.repeat(np.arange(250, dtype=np.uint32), 2)
    par[300:302] = 7                              # paragraph 7 again after 149: not contiguous
    with pytest.raises(_lib.NidxError):
        VectorSegment.create(v, 64, similarity=_lib.NIDX_SIM_DOT, paragraph_of=par)
    seg = VectorSegment.create(v, 64, similarity=_lib.NIDX_SIM_DOT, paragraph_of=np.repeat(np.arange(250, dtype=np.uint32), 2))
    ids, scores, counts = seg.search(v[:8], 5, method=_lib.NIDX_METHOD_BRUTE, with_duplicates=True)
    assert (counts == 5).all() and (ids < len(v)).all() and np.allclose(scores[:, 0], 1.0, atol=1e-5)   # each query finds itself
    seg.close()


def test_create_close_cycles_with_every_optional_array_give_the_same_results():
    c = _corpus(3, 20_000)
    created, modified = _dates(c, 4)
    _, qt, qo = _queries(c, 5, 8, False)
    first_vec = first_txt = None
    for cycle in range(24):
        seg, rids, pool = _segment(n=1500, dim=64, seed=6)   # graph and fp16 copy (the build's walk makes it), label and field indexes
        vs = seg.segment
        vs.rabitq_encode()
        seg.apply_deletions([f"{rids[2]}/a/title", rids[5]])   # alive bits
        vs.set_paragraph_keys(np.arange(seg.records, dtype=np.uint64) * 7919 + 11)
        q = make_queries(seg.host_vectors, 16, seed=5)
        got = [vs.rabitq_codes(), *vs.get_graph().values()]
        for method in METHODS:
            got += list(vs.search(q, 10, ef=40, method=method))
        got += _vector_results(seg, pool, rids, q)
        got.append(shard_record(vs, q, 10, dedup=True).cpu().numpy())
        seg.close()

        ts = _text_segment(c, _alive(c["n_docs"], 6))
        ts.set_dates(created, modified)
        ts.set_doc_keys(np.arange(c["n_docs"], dtype=np.uint64) * 3 + 1)
        txt = _text_results(ts, c, qt, qo)
        ts.close()
        if cycle == 0:
            first_vec, first_txt = got, txt
        else:
            _same(first_vec, got)
            _same(first_txt, txt)
