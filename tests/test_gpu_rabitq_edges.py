"""The RaBitQ kernels against the oracle where they can go wrong without the rest of the suite noticing (vector_types/rabitq.rs,
segment.rs:581-608, hnsw/search.rs:306-383):

* the quantised walk's global visited table on a 500 000-node segment with the reference's constants (M = 30, M0 = 60) at
  top_k >= 20, where layer 0 visits more nodes than a 2^16-slot table admits;
* the quantised scan's query groups (more than 4 GiB of estimates: several groups, the last one ragged);
* the rerank chunk edges of the scan (RR_CHUNK = 4096) and of the walk (RQ_RC = 64, lists shorter than last_k);
* the walk's NG instances (d = 64, 256, 384, 512, 1024) in both CTA shapes;
* the estimator's numeric edges (rabitq_edge_inputs.py; test_rabitq_edge_models.py pins the oracle to the reference on them).

Codes are compared byte for byte, estimates and errors bitwise (a NaN equal to any NaN), ids, scores and counts exactly, and the
walk's expansion and estimate counters equal the oracle's with no visited-set overflow.  Run time on one H100 80GB HBM3 with
8 host cores: about 20 seconds, a third of it the 500 000-node graph build."""
import ctypes as C

import numpy as np
import pytest

import oracle as O
from conftest import make_queries, make_vectors
from nucliadb_b200 import _lib
from nucliadb_b200.segment import VectorSegment
from rabitq_edge_inputs import edge_queries, edge_rows, f32, same_bits, same_codes

pytestmark = pytest.mark.gpu

NT = 8
RQ = _lib.NIDX_METHOD_HNSW_RABITQ
SCAN = _lib.NIDX_METHOD_BRUTE_RABITQ


def _oracle_graph(seg, n, m, m0):
    g = seg.get_graph()
    og = O.Graph(n, m, m0, g["level"])
    og.adj0[:], og.adjU[:] = g["adj0"], g["adjU"][: og.adjU.shape[0]]
    og.entry_node, og.entry_layer = g["entry_node"], g["entry_layer"]
    return og


def _words(alive):
    words = np.zeros((len(alive) + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(alive, bitorder="little")
    words[: len(pb)] = pb
    return words.view(np.uint64)


def _oracle_scan(v, enc, q, k, ms, alive=None):
    """oracle.rabitq_brute_force over the alive rows only (the scan's candidates are the alive rows in address order, so the
    oracle on the subset, ids mapped back, is the filtered scan)."""
    idx = np.arange(len(v)) if alive is None else np.nonzero(alive)[0]
    if len(idx) == 0:
        nq = len(q)
        return np.full((nq, k), O.NIL, np.uint32), np.zeros((nq, k), f32), np.zeros(nq, np.int32)
    oi, os_, oc, _ = O.rabitq_brute_force(v[idx], enc[idx], q, k, min_score=ms, nthreads=NT)
    ids = np.where(oi == O.NIL, O.NIL, idx[np.minimum(oi, len(idx) - 1)]).astype(np.uint32)
    return ids, os_, oc


def _check_scan(seg, v, enc, q, k, ms, alive=None, what=""):
    ids, sc, cnt = seg.search(q, k, min_score=ms, method=SCAN, filter_bits=None if alive is None else _words(alive))
    oi, os_, oc = _oracle_scan(v, enc, q, k, ms, alive)
    assert (cnt == oc).all(), (what, k, ms, np.nonzero(cnt != oc)[0][:8])
    assert (ids == oi).all() and same_bits(sc, os_), (what, k, ms, np.nonzero((ids != oi).any(1))[0][:8])


def _check_walk(seg, v, enc, og, q, k, ms=-1.0, dup=True, bits=None, what="", estimates=True):
    """The quantised walk equals the oracle's: results, and the estimate / expansion counters with no overflow.  The kernel carries
    the entry point's estimate from layer to layer, the reference re-evaluates it in every layer_search (search.rs:256-261)."""
    ids, sc, cnt = seg.search(q, k, min_score=ms, with_duplicates=dup, method=RQ, filter_bits=bits)
    c = seg.counters_ex()
    raw = (C.c_uint64 * 6)()
    _lib.load().nidx_vec_counters_ex(seg._h, raw)
    c["visited_overflows"], c["cu_overflows"] = raw[2], raw[3]
    oi, os_, oc, ocnt = O.hnsw_search_rabitq(v, enc, og, q, k, min_score=ms, with_duplicates=dup, filter_bits=bits, nthreads=NT)
    assert (cnt == oc).all() and (ids == oi).all() and same_bits(sc, os_), (what, k, ms, dup, np.nonzero((ids != oi).any(1))[0][:8])
    assert c["expansions"] == int(ocnt[1]), (what, k, c, ocnt)
    assert not estimates or c["estimates"] == int(ocnt[3]) - len(q) * og.entry_layer, (what, k, c, ocnt)
    assert c["overflows"] == 0, (what, k, c)
    return ids, cnt


# ---- 1. the walk's global visited table -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def big_graph():
    n, d = 500_000, 64
    v = make_vectors(n, d, seed=5, latent=64, noise=1.0)
    rng = np.random.default_rng(8)
    q = np.concatenate([make_queries(v, 48, seed=9), rng.standard_normal((16, d)).astype(f32)])
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT, m=30, m0=60, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=4096)
    seg.rabitq_encode()
    enc = O.rabitq_encode(v, nthreads=NT)
    assert np.array_equal(seg.rabitq_codes(), enc)
    yield seg, v, q, enc, _oracle_graph(seg, n, 30, 60)
    seg.close()


@pytest.mark.parametrize("shape", ["8", "4"])
@pytest.mark.parametrize("k", [20, 100])
def test_walk_past_the_visited_table_limit_of_a_64k_table(big_graph, k, shape, monkeypatch):
    """top_k >= 20 asks layer 0 for 2 000 nodes; with adjacency rows of 64 slots the walk estimates 50 000 - 75 000 nodes per
    query on this segment, more than the 61 376 inserts a 2^16-slot table admits.  Every node the reference scores must be scored:
    the same results and counters as the oracle, no overflow."""
    monkeypatch.setenv("NIDX_B200_RQ_W", shape)
    seg, v, q, enc, og = big_graph
    if k == 20 and shape == "8":   # the case keeps testing the limit: the oracle's own count per query passes it
        per_q = [int(O.hnsw_search_rabitq(v, enc, og, q[i : i + 1], k, min_score=-1.0, nthreads=1)[3][3]) for i in range(len(q))]
        assert max(per_q) > 61_376, max(per_q)
    L = _lib.load()
    n0 = L.nidx_launch_count()
    seg.search(q, 10, method=RQ)                   # 37 000 estimates at most: no table of this walk fills
    base = L.nidx_launch_count() - n0
    n0 = L.nidx_launch_count()
    _check_walk(seg, v, enc, og, q, k, what=f"n=500000 k={k} W={shape}")
    # as many launches as at k = 10: the table is sized for the walk, so no query overflowed and the batch did not run again
    assert L.nidx_launch_count() - n0 == base


def test_filtered_walk_past_the_visited_table_limit(big_graph):
    """Every third node dead: closest_up_nodes walks on from the reranked list until it has k alive results, and its list of
    cu_cap = k + k * s0 entries fills and drops its worst ones -- which no pop reaches, so the results are the reference's."""
    seg, v, q, enc, og = big_graph
    alive = np.ones(len(v), dtype=bool)
    alive[::3] = False
    bits = _words(alive)
    ids, cnt = _check_walk(seg, v, enc, og, q, 20, bits=bits, what="filtered")
    assert all(alive[i] for i in ids[ids != O.NIL])


def test_walk_runs_again_when_the_layer0_table_overflows(big_graph, monkeypatch):
    """A 2^16-slot table (NIDX_B200_RQ_GV_BITS) cannot hold this walk: the queries overflow it, the call runs the batch again on
    the table that holds every node -- one more walk launch -- and returns the oracle's results with no overflow counted."""
    seg, v, q, enc, og = big_graph
    L = _lib.load()
    n0 = L.nidx_launch_count()
    seg.search(q, 20, method=RQ)
    base = L.nidx_launch_count() - n0
    monkeypatch.setenv("NIDX_B200_RQ_GV_BITS", "16")
    n0 = L.nidx_launch_count()
    _check_walk(seg, v, enc, og, q, 20, what="re-run")
    assert L.nidx_launch_count() - n0 == base + 1


# ---- 2. query groups of the scan -------------------------------------------------------------------------------------------
def test_scan_query_groups():
    """4 GiB of estimates per group: n = 600 000 gives groups of 894 queries, so 1 000 queries run as 894 + 106.  Every query of
    both groups equals the oracle."""
    n, d, nq = 600_000, 64, 1000
    assert (4 << 30) // (n * 8) == 894
    v = make_vectors(n, d, seed=21)
    q = make_queries(v, nq, seed=22)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT)
    seg.rabitq_encode()
    enc = O.rabitq_encode(v, nthreads=NT)
    assert np.array_equal(seg.rabitq_codes(), enc)
    _check_scan(seg, v, enc, q, 10, -1.0, what="groups")
    seg.close()


# ---- 3. rerank chunk edges -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 63, 64, 4095, 4096, 4097, 8193])
def test_scan_rerank_chunk_edges(n):
    """RR_CHUNK = 4096 candidates are filtered against the heap at the start of their chunk: segments just below, at and above a
    chunk, k from 1 to past the number of rows, filters that leave fewer than k rows or none, and min_score above every score."""
    d = 64
    v = make_vectors(n, d, seed=30 + n)               # unit rows: every error bound is finite, every row a candidate
    names, q = edge_queries(v, d, seed=31)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT)
    seg.rabitq_encode()
    enc = O.rabitq_encode(v, nthreads=NT)
    assert same_codes(seg.rabitq_codes(), enc)
    for k in sorted({1, 10, n, n + 3, 1024}):
        if k > 1024:
            continue
        _check_scan(seg, v, enc, q, k, -1.0, what=f"n={n}")
        _check_scan(seg, v, enc, q, k, -np.inf, what=f"n={n}")
    rng = np.random.default_rng(n)
    few = np.zeros(n, dtype=bool)
    few[rng.choice(n, min(n, 5), replace=False)] = True
    _check_scan(seg, v, enc, q, 10, -1.0, alive=few, what=f"n={n} five alive")
    # no alive row: the call returns before the scan (segment.rs:532-534), so this checks that early exit
    _check_scan(seg, v, enc, q, 10, -1.0, alive=np.zeros(n, dtype=bool), what=f"n={n} none alive")
    # rows alive but no upper bound or score reaches min_score: the scan's rerank runs with no candidate
    _check_scan(seg, v, enc, q, 10, 1e30, what=f"n={n} min_score above every score")
    _check_scan(seg, v, enc, q, 10, 1e30, alive=few, what=f"n={n} five alive, min_score above every score")
    seg.close()


@pytest.mark.parametrize("shape", ["8", "4"])
@pytest.mark.parametrize("n", [1, 2, 65, 1999])
def test_walk_on_small_segments(n, shape, monkeypatch):
    """Lists shorter than last_k: the walk's rerank (chunks of RQ_RC = 64) ends on a partial chunk, or runs on one entry."""
    monkeypatch.setenv("NIDX_B200_RQ_W", shape)
    d = 128
    v = make_vectors(n, d, seed=40 + n)
    q = make_queries(make_vectors(64, d, seed=40 + n), 12, seed=41)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    seg.build_hnsw(seed=2, max_batch=256)
    seg.rabitq_encode()
    enc = O.rabitq_encode(v, nthreads=NT)
    og = _oracle_graph(seg, n, 16, 32)
    for k in (1, 10, 20):
        _check_walk(seg, v, enc, og, q, k, what=f"n={n}")
    _check_walk(seg, v, enc, og, q, 10, ms=0.3, what=f"n={n} min_score")
    seg.close()


# ---- 4. NG instances of the walk -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", ["8", "4"])
@pytest.mark.parametrize("d", [64, 256, 384, 512, 1024])
def test_walk_ng_instances(d, shape, monkeypatch):
    """hnsw_rabitq_kernel<NG> for NG = 2, 3, 4, 8 and the run-time loop at d = 64, whose whole code is one 16-byte chunk (header and
    both sign words), with test_quantised_walk_matches_oracle's k / min_score / duplicates loop and a filter."""
    monkeypatch.setenv("NIDX_B200_RQ_W", shape)
    n = 6000
    v = make_vectors(n, d, seed=61)
    v[100:110] = v[90:100]                                   # byte-identical vectors for with_duplicates=False
    q = make_queries(v, 24)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    seg.build_hnsw(seed=2, max_batch=512)
    seg.rabitq_encode()
    enc = O.rabitq_encode(v, nthreads=NT)
    assert np.array_equal(seg.rabitq_codes(), enc)
    og = _oracle_graph(seg, n, 16, 32)
    for k, ms, dup in ((10, -1.0, True), (10, 0.2, True), (5, -1.0, False), (25, -1.0, True)):
        _check_walk(seg, v, enc, og, q, k, ms=ms, dup=dup, what=f"d={d}")
    alive = np.ones(n, dtype=bool)
    alive[::3] = False
    ids, _ = _check_walk(seg, v, enc, og, q, 10, bits=_words(alive), what=f"d={d} filtered")
    assert all(alive[i] for i in ids[ids != O.NIL])
    seg.close()


# ---- 5. numeric edges --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [64, 256])
def test_codes_estimates_and_scan_at_the_numeric_edges(d):
    n = 5000
    v = edge_rows(n, d, seed=70 + d)
    names, q = edge_queries(v, d, seed=71)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT)
    seg.rabitq_encode()
    enc = O.rabitq_encode(v, nthreads=NT)
    assert same_codes(seg.rabitq_codes(), enc)
    est, err = seg.rabitq_estimate(q)
    oest, oerr = O.rabitq_estimate(enc, d, q, nthreads=NT)
    for qi, name in enumerate(names):
        assert same_bits(est[qi], oest[qi]) and same_bits(err[qi], oerr[qi]), name
    for k, ms in ((1, -1.0), (10, -1.0), (100, 0.0), (1024, -np.inf)):
        _check_scan(seg, v, enc, q, k, ms, what=f"edges d={d}")
    seg.close()


@pytest.mark.parametrize("shape", ["8", "4"])
def test_walk_at_the_numeric_edges(shape, monkeypatch):
    """The walk over edge rows on a graph built from finite unit rows (set_graph), for every edge query.  What the walk does there:
    * a NaN-first query has low = delta = NaN: every estimate is NaN, no neighbour ranks above a full list's worst, every exact
      similarity is NaN and fails `>= min_score`, so the result is empty;
    * a +-inf query has delta = inf and every estimate NaN: the walk admits nodes in graph order by id until the list is full and
      reranks them exactly;
    * a constant query has estimates that depend on sum_bits alone, so the walk follows ties broken by id;
    * a +-inf query makes every exact similarity +-inf: the results tie, and the final sort keeps them in the order
      closest_up_nodes accepted them (search.rs:381 is a stable sort on the score alone), not in id order;
    * rows with dot_quant_original > 1 have a NaN error bound and a NaN upper bound, which rerank_top evaluates only while it holds
      fewer than k results; rows with a NaN estimate rank above every finite one.
    Only equality with the oracle is asserted, not recall.  The estimate counter is compared for the queries whose estimates are
    numbers; where every estimate is NaN (the +-inf and NaN-first queries) the kernel counted 11 more estimates per query (k = 10) than the
    oracle with the same expansions and results (DESIGN.md §4).  Exact similarities must not be a NaN made by arithmetic, whose sign
    differs between x86 and CUDA (DESIGN.md §4) and would rank it at the other end of closest_up_nodes' candidates: so the rows
    hold no +-inf (inf - inf against an inf query), and the +-inf queries run on the rows without the zero row (0 * inf)."""
    monkeypatch.setenv("NIDX_B200_RQ_W", shape)
    n, d = 6000, 64
    base = VectorSegment.create(make_vectors(n, d, seed=80), d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    base.build_hnsw(seed=2, max_batch=512)
    g = base.get_graph()
    base.close()
    v = edge_rows(n, d, seed=81, nonfinite=False)
    v[n // 2, 5] = np.nan
    names, q = edge_queries(v, d, seed=82)
    inf_q = np.array(["inf" in x for x in names])
    no_zero = v.copy()
    no_zero[0] = make_vectors(1, d, seed=83)[0]                     # edge_rows puts the zero row at 0
    assert not v[0].any() and no_zero[0].all()
    for rows, sel in ((v, ~inf_q), (no_zero, inf_q)):
        seg = VectorSegment.create(rows, d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
        seg.set_graph(g["level"], g["adj0"], g["adjU"], g["w0"], g["wU"])
        seg.rabitq_encode()
        enc = O.rabitq_encode(rows, nthreads=NT)
        assert same_codes(seg.rabitq_codes(), enc)
        og = _oracle_graph(seg, n, 16, 32)
        for k, ms in ((10, -1.0), (20, -np.inf), (5, 0.0)):
            ids, cnt = _check_walk(seg, rows, enc, og, q[sel], k, ms=ms, what="edges", estimates=False)
            sub = [x for x, s in zip(names, sel) if s]
            if "nan_first" in sub:
                assert cnt[sub.index("nan_first")] == 0
            finite = np.array([x not in ("plus_inf", "minus_inf", "nan_first") for x in sub])
            if finite.any():
                _check_walk(seg, rows, enc, og, q[sel][finite], k, ms=ms, what="edges, finite estimates")
        seg.close()
