"""closest_up_nodes on the kept layer-0 visited set: when every pop is accepted and the list's k-th entry scores above its last, a
neighbour the layer-0 walk already visited is settled without its f32 row (hs_can_defer).  Ids, scores and counts must stay
bit-identical to the f32-only walk (NIDX_B200_HS_F16=0, which scores every neighbour) and to the oracle, with the oracle's
similarity and expansion counters and no overflow; the walks that cannot defer must stay as they were."""
import numpy as np
import pytest

import oracle as O
from conftest import make_queries, make_vectors
from nucliadb_b200 import _lib
from nucliadb_b200.segment import VectorSegment

pytestmark = pytest.mark.gpu


def _oracle_graph(seg, n):
    g = seg.get_graph()
    og = O.Graph(n, 16, 32, g["level"])
    og.adj0[:], og.adjU[:] = g["adj0"], g["adjU"][: og.adjU.shape[0]]
    og.entry_node, og.entry_layer = g["entry_node"], g["entry_layer"]
    return og


def _bits(n, frac, seed):
    keep = np.random.default_rng(seed).random(n) < frac
    words = np.zeros((n + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(keep, bitorder="little")
    words[: len(pb)] = pb
    return words.view(np.uint64)


def _search(seg, q, k, ef, monkeypatch, f32, **kw):
    if f32:
        monkeypatch.setenv("NIDX_B200_HS_F16", "0")
    else:
        monkeypatch.delenv("NIDX_B200_HS_F16", raising=False)
    r = seg.search(q, k, ef=ef, method=_lib.NIDX_METHOD_HNSW, **kw)
    return r, seg.counters(), seg.exact_rows()


def _check(seg, v, og, q, k, ef, monkeypatch, sim, filter_bits=None, min_score=-1.0, with_duplicates=True):
    """The screened walk against the f32-only walk and the oracle; returns the screened walk's exact_rows.  Without duplicates the
    counters are compared with the f32-only walk's only: the kernel and the oracle count a rejected duplicate differently (the
    f32-only walk of the parent commit counts the same as this one)."""
    kw = dict(min_score=min_score, with_duplicates=with_duplicates, filter_bits=filter_bits)
    (i32, s32, c32), k32, e32 = _search(seg, q, k, ef, monkeypatch, True, **kw)
    (i16, s16, c16), k16, e16 = _search(seg, q, k, ef, monkeypatch, False, **kw)
    assert (c16 == c32).all() and (i16 == i32).all() and np.array_equal(s16.view(np.uint32), s32.view(np.uint32))
    assert k16 == k32 and k16["overflows"] == 0
    oi, os_, oc, counters = O.hnsw_search(v, og, q, k, ef, sim=sim, min_score=min_score, with_duplicates=with_duplicates,
                                          filter_bits=filter_bits, nthreads=8)
    assert (c16 == oc).all() and (i16 == oi).all() and np.array_equal(s16.view(np.uint32), os_.view(np.uint32))
    if with_duplicates:
        assert k16["similarities"] == counters[0] - len(q) * og.entry_layer and k16["expansions"] == counters[1]
    assert e32 == k32["similarities"] and e16 < e32
    return e16


@pytest.fixture(scope="module")
def latent():
    v = make_vectors(30000, 128, seed=41)
    seg = VectorSegment.create(v, 128, similarity=_lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=1024)
    yield v, seg, _oracle_graph(seg, len(v))
    seg.close()


def test_unfiltered_top_k_reads_no_row_after_the_walk(latent, monkeypatch):
    """Every neighbour of the final layer-0 list was visited by the walk: k = 10 and k = 100 read the rows k = 1 reads, no more.
    At ef = 30, k = 100 makes ef0 = k, so the k-th entry is the last one and the walk scores every neighbour, as before."""
    v, seg, og = latent
    q = make_queries(v, 64, seed=42)
    for ef, deferring, scoring in ((30, (10,), (100,)), (128, (10, 100), ())):
        e1 = _check(seg, v, og, q, 1, ef, monkeypatch, O.SIM_COSINE)
        for k in deferring:
            assert _check(seg, v, og, q, k, ef, monkeypatch, O.SIM_COSINE) == e1
        for k in scoring:
            assert _check(seg, v, og, q, k, ef, monkeypatch, O.SIM_COSINE) > e1


def _check_each(seg, v, og, q, k, ef, monkeypatch, sim, min_scores=None, **kw):
    """_check query by query (min_scores: one per query), every query: one whose first walk outgrows a capacity (closest_up_nodes'
    cu_cap entries or the visited set) is walked again on capacities that cannot overflow, and must still equal the oracle with no
    overflow counted; returns how many were checked."""
    checked = 0
    for i in range(len(q)):
        qi = q[i : i + 1]
        if min_scores is not None:
            kw["min_score"] = float(min_scores[i])
        _check(seg, v, og, qi, k, ef, monkeypatch, sim, **kw)
        checked += 1
    return checked


@pytest.mark.parametrize("col", [10, 30, 79])
def test_min_score_break(latent, monkeypatch, col):
    """k = 40, ef = 64 and a min_score at a query's 11th, 31st or 80th best score: the walk defers and stops at min_score."""
    v, seg, og = latent
    q = make_queries(v, 32, seed=43)
    _, sc, _ = O.brute_force(v, q, 80, sim=O.SIM_COSINE, nthreads=8)
    assert _check_each(seg, v, og, q, 40, 64, monkeypatch, O.SIM_COSINE, min_scores=sc[:, col]) == len(q)


@pytest.mark.parametrize("frac", [0.3, 0.9])
def test_filtered_walk_scores_every_neighbour(latent, monkeypatch, frac):
    """A filter can reject pops, so these walks run the kernel that scores every neighbour.  At 30 % most queries outgrow cu_cap
    in their first walk and are walked again."""
    v, seg, og = latent
    q = make_queries(v, 32, seed=44)
    assert _check_each(seg, v, og, q, 10, 64, monkeypatch, O.SIM_COSINE, filter_bits=_bits(len(v), frac, seed=45)) == len(q)


def test_duplicates_walk_scores_every_neighbour(monkeypatch):
    """with_duplicates=False on exact duplicate rows can reject pops, so these walks take the path that scores every neighbour;
    with min_scores around the layer-0 list's last score."""
    v = make_vectors(20000, 96, seed=45)
    v[10000:10600] = v[0:600]
    seg = VectorSegment.create(v, 96, similarity=_lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=1024)
    og = _oracle_graph(seg, len(v))
    q = np.concatenate([v[:16] + 0.0, make_queries(v, 16, seed=46)])
    _, sc, _ = O.brute_force(v, q, 80, sim=O.SIM_COSINE, nthreads=8)
    for col in (40, 79):
        assert _check_each(seg, v, og, q, 64, 64, monkeypatch, O.SIM_COSINE, min_scores=sc[:, col], with_duplicates=False) == len(q)


def test_signed_zero_rows_at_the_bound(monkeypatch):
    """Dot rows of +0.0 and of -0.0 both score +0.  Only 40 rows score above zero, so the ef = 64 list ends among the zero rows:
    s_w = +0, and the zero rows the walk visited tie with the bound.  k = 10 defers them; k = 64 (the k-th entry is the last)
    and with_duplicates=False score every neighbour."""
    n, d = 12000, 64
    v = make_vectors(n, d, seed=49)
    v[:, 0] = -np.abs(v[:, 0]) - 0.5
    v[:40, 0] *= -1.0
    v[2000:5000] = 0.0
    v[5000:8000] = -0.0
    v = np.ascontiguousarray(v, dtype=np.float32)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    seg.build_hnsw(seed=2, max_batch=512)
    og = _oracle_graph(seg, n)
    q = 0.02 * make_queries(v, 16, seed=50)
    q[:, 0] = 1.0
    q = np.ascontiguousarray(q, dtype=np.float32)
    checked = 0
    for k, ms, dup in ((10, -1e30, True), (10, 0.0, True), (64, 0.0, True), (64, 0.0, False)):
        checked += _check_each(seg, v, og, q, k, 64, monkeypatch, O.SIM_DOT, min_scores=np.full(len(q), ms), with_duplicates=dup)
    assert checked == 4 * len(q)
