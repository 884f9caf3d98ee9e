"""Embedding widths of real embedders (1 536 - 4 096) on the paths that branch on the row length: the GPU HNSW build re-reading
kept rows from global memory once they no longer fit its shared-memory cache, and RaBitQ's wide-code branches up to its
4 096-dimension limit."""
import numpy as np
import pytest

import oracle as O
from conftest import make_queries, make_vectors
from nucliadb_b200 import _lib
from nucliadb_b200.segment import VectorSegment

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("m,m0", [(16, 32), (30, 60)])
@pytest.mark.parametrize("d", [1536, 3072])
def test_gpu_build_equals_oracle_batch_build_at_wide_rows(d, m, m0):
    """The select / reverse-link kernels cache 96 KB of kept rows: 16 rows at d = 1536, 8 at 3072, so both M0 = 32 and 60 spill.
    Same levels, same batch schedule, same arithmetic order => the same graph, edge for edge."""
    v = make_vectors(2500, d, seed=71)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_COSINE, m=m, m0=m0, ef_construction=40)
    seg.build_hnsw(seed=2, max_batch=128)
    g = seg.get_graph()
    og = O.hnsw_build(v, M=m, M0=m0, efC=40, seed=2, max_batch=128, nthreads=8)
    assert (g["level"] == og.level).all() and g["entry_node"] == og.entry_node
    assert (g["adj0"] == og.adj0).all() and np.array_equal(g["w0"], og.w0)
    assert (g["adjU"][: og.adjU.shape[0]] == og.adjU).all()


@pytest.mark.parametrize("d", [1984, 2048, 4096])
def test_rabitq_scan_at_wide_rows(d):
    v = make_vectors(4000, d, seed=72)
    q = make_queries(v, 24, seed=73)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT)
    seg.rabitq_encode()
    assert (seg.rabitq_codes() == O.rabitq_encode(v, nthreads=8)).all()
    for k, ms in ((10, 0.0), (1, 0.3)):
        ids, sc, cnt = seg.search(q, k, min_score=ms, method=_lib.NIDX_METHOD_BRUTE_RABITQ)
        oi, os_, oc, _ = O.rabitq_brute_force(v, O.rabitq_encode(v, nthreads=8), q, k, min_score=ms, nthreads=8)
        assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)


def test_rabitq_refuses_dimensions_above_4096():
    seg = VectorSegment.create(make_vectors(200, 4160, seed=74), 4160, similarity=_lib.NIDX_SIM_DOT)
    with pytest.raises(_lib.NidxError):
        seg.rabitq_encode()
    with pytest.raises(_lib.NidxError):
        seg.search(make_queries(make_vectors(20, 4160, seed=75), 2), 5, method=_lib.NIDX_METHOD_BRUTE_RABITQ)
