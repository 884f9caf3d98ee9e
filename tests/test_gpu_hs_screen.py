"""The HNSW walk's fp16 screen: a neighbour whose fp16 similarity plus a proven error bound cannot enter the list is rejected
without reading its f32 row.  The walk must stay bit-identical to the f32-only walk (NIDX_B200_HS_F16=0) and to the oracle:
same ids, scores, counts, similarity / expansion / overflow counters, and the same graph from the GPU build."""
import numpy as np
import pytest

import oracle as O
from conftest import make_queries, make_vectors
from nucliadb_b200 import _lib
from nucliadb_b200.segment import VectorSegment

pytestmark = pytest.mark.gpu

SIMS = [_lib.NIDX_SIM_COSINE, _lib.NIDX_SIM_DOT, _lib.NIDX_SIM_L2]


def _data(sim, n, d, seed):
    v = make_vectors(n, d, seed=seed)
    if sim != _lib.NIDX_SIM_COSINE:   # Dot and L2 see the row norms: make them differ
        v = v * np.random.default_rng(seed).uniform(0.5, 2.0, (n, 1)).astype(np.float32)
    return np.ascontiguousarray(v, dtype=np.float32), make_queries(v, 48, seed=seed + 1)


def _oracle_graph(seg, n):
    g = seg.get_graph()
    og = O.Graph(n, 16, 32, g["level"])
    og.adj0[:], og.adjU[:] = g["adj0"], g["adjU"][: og.adjU.shape[0]]
    og.entry_node, og.entry_layer = g["entry_node"], g["entry_layer"]
    return og


def _search_both(seg, q, ef, monkeypatch):
    monkeypatch.setenv("NIDX_B200_HS_F16", "0")
    f32 = seg.search(q, 10, ef=ef, method=_lib.NIDX_METHOD_HNSW)
    c32, e32 = seg.counters(), seg.exact_rows()
    monkeypatch.delenv("NIDX_B200_HS_F16")
    f16 = seg.search(q, 10, ef=ef, method=_lib.NIDX_METHOD_HNSW)
    c16, e16 = seg.counters(), seg.exact_rows()
    return f32, c32, e32, f16, c16, e16


def _same(a, b):
    assert (a[2] == b[2]).all() and (a[0] == b[0]).all()
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))   # bitwise


@pytest.mark.parametrize("sim", SIMS)
@pytest.mark.parametrize("d", [128, 100, 512, 1024, 1536, 4096])
def test_screened_walk_is_the_f32_walk_and_the_oracle(sim, d, monkeypatch):
    v, q = _data(sim, 8000, d, seed=21 + d + sim)
    seg = VectorSegment.create(v, d, similarity=sim, m=16, m0=32, ef_construction=64)
    monkeypatch.setenv("NIDX_B200_HS_F16", "0")
    seg.build_hnsw(seed=2, max_batch=512)
    og = _oracle_graph(seg, len(v))
    for ef in (30, 128):
        f32, c32, e32, f16, c16, e16 = _search_both(seg, q, ef, monkeypatch)
        _same(f32, f16)
        assert c32 == c16 and c16["overflows"] == 0
        assert e32 == c32["similarities"]            # the f32-only walk reads a row per similarity
        assert e16 < c16["similarities"]             # the lists fill: the screen settles some neighbours
        oi, os_, oc, counters = O.hnsw_search(v, og, q, 10, ef, sim=sim, nthreads=8)
        assert (f16[2] == oc).all() and (f16[0] == oi).all() and np.array_equal(f16[1], os_)
        assert c16["similarities"] == counters[0] - len(q) * og.entry_layer and c16["expansions"] == counters[1]


@pytest.mark.parametrize("sim", SIMS)
def test_screened_walk_on_near_ties(sim, monkeypatch):
    """Exact and near-duplicate rows put many candidates within ~1e-6 of the list's worst key."""
    rng = np.random.default_rng(7)
    base, _ = _data(sim, 2000, 96, seed=3)
    v = np.concatenate([base] + [base + rng.normal(0, s, base.shape).astype(np.float32) for s in (0.0, 1e-7, 1e-6)])
    v = np.ascontiguousarray(v, dtype=np.float32)
    q = np.concatenate([v[rng.integers(0, len(v), 24)], make_queries(v, 24, seed=5)])
    seg = VectorSegment.create(v, 96, similarity=sim, m=16, m0=32, ef_construction=64)
    monkeypatch.setenv("NIDX_B200_HS_F16", "0")
    seg.build_hnsw(seed=2, max_batch=256)
    og = _oracle_graph(seg, len(v))
    f32, c32, e32, f16, c16, e16 = _search_both(seg, q, 64, monkeypatch)
    _same(f32, f16)
    assert c32 == c16 and e16 < c16["similarities"]
    oi, os_, oc, _ = O.hnsw_search(v, og, q, 10, 64, sim=sim, nthreads=8)
    assert (f16[0] == oi).all() and np.array_equal(f16[1], os_)


@pytest.mark.parametrize("sim", [_lib.NIDX_SIM_COSINE, _lib.NIDX_SIM_L2])
def test_gpu_build_graph_is_the_f32_builds(sim, monkeypatch):
    v, _ = _data(sim, 30000, 96, seed=11)
    graphs, counters = [], []
    for force_f32 in (True, False):
        if force_f32:
            monkeypatch.setenv("NIDX_B200_HS_F16", "0")
        else:
            monkeypatch.delenv("NIDX_B200_HS_F16")
        seg = VectorSegment.create(v, 96, similarity=sim, m=16, m0=32, ef_construction=100)
        seg.build_hnsw(seed=2, max_batch=1024)
        graphs.append(seg.get_graph())
        counters.append((seg.counters(), seg.exact_rows()))
        seg.close()
    for key in ("level", "adj0", "w0", "adjU"):
        assert np.array_equal(np.asarray(graphs[0][key]), np.asarray(graphs[1][key])), key
    assert graphs[0]["entry_node"] == graphs[1]["entry_node"] and graphs[0]["entry_layer"] == graphs[1]["entry_layer"]
    (c32, e32), (c16, e16) = counters
    assert c32 == c16 and e32 == c32["similarities"] and e16 < c16["similarities"]


def test_nonfinite_and_extreme_rows_take_the_exact_path(monkeypatch):
    """Rows with NaN / Inf, zero rows, and rows spanning 1e-20 .. 1e20: the screened walk still equals the f32 walk."""
    rng = np.random.default_rng(9)
    v, q = _data(_lib.NIDX_SIM_DOT, 4000, 128, seed=13)
    v = v.copy()
    v[10:20] = 0.0
    v[20:30, 5] = np.nan
    v[30:40, 7] = np.inf
    v[40:200] *= np.float32(1e-20)
    v[200:400] *= np.float32(1e18)
    v[400:600] *= 10.0 ** rng.uniform(-20, 20, (200, 1)).astype(np.float32)
    for sim in SIMS:
        seg = VectorSegment.create(v, 128, similarity=sim, m=16, m0=32, ef_construction=64)
        monkeypatch.setenv("NIDX_B200_HS_F16", "0")
        seg.build_hnsw(seed=2, max_batch=256)
        f32, c32, e32, f16, c16, e16 = _search_both(seg, q, 64, monkeypatch)
        _same(f32, f16)
        assert c32 == c16
        seg.close()
