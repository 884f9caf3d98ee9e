"""The dense HNSW walk (hnsw_search_kernel) against the oracle where its fixed capacities run out: the shared-memory visited set
(max(4096, 1.5 * ef0 * s0) slots) and closest_up_nodes' candidate list (cu_cap = min(max(ef0 + k * s0, 2 * ef0), 4096) entries),
where the reference's BitSet and heap are unbounded (search.rs:188-240).  A filter that rejects most pops makes closest_up_nodes
score thousands of nodes, more than either holds.  The walk flags a query that lost a neighbour or a candidate to them and walks it
again on capacities that cannot overflow, so every query is compared here, none skipped:

* ids, counts and scores (bitwise) equal O.hnsw_search on the graph the GPU built;
* the similarity and expansion counters equal the oracle's (the f32-only walk's where with_duplicates=False), with no overflow;
* the fp16-screened walk and the f32-only walk (NIDX_B200_HS_F16=0) both.

Cases: the reference's default constants (M = 30, M0 = 60, ef_search = 30) on 200 000 x 64 Cosine rows with uniform filters of
30 - 2 %, a filter that keeps only rows far from every query, pops rejected without a filter (duplicates, multi-vector
paragraphs), min_score, Dot and L2, a visited table capped to a few hundred slots (NIDX_B200_HS_BITS), the AUTO choice, and the
benchmark's shape, where the re-run must cost one launch that finds nothing and no host synchronisation."""
import time

import numpy as np
import pytest

import oracle as O
from conftest import make_queries, make_vectors
from nucliadb_b200 import _lib
from nucliadb_b200.segment import VectorSegment

pytestmark = pytest.mark.gpu

NT = 8
HNSW = _lib.NIDX_METHOD_HNSW


def _oracle_graph(seg, n, m, m0):
    g = seg.get_graph()
    og = O.Graph(n, m, m0, g["level"])
    og.adj0[:], og.adjU[:] = g["adj0"], g["adjU"][: og.adjU.shape[0]]
    og.entry_node, og.entry_layer = g["entry_node"], g["entry_layer"]
    return og


def _words(keep):
    words = np.zeros((len(keep) + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(keep, bitorder="little")
    words[: len(pb)] = pb
    return words.view(np.uint64)


def _uniform(n, frac, seed):
    return np.random.default_rng(seed).random(n) < frac


def _search(seg, q, k, ef, monkeypatch, f32, **kw):
    if f32:
        monkeypatch.setenv("NIDX_B200_HS_F16", "0")
    else:
        monkeypatch.delenv("NIDX_B200_HS_F16", raising=False)
    r = seg.search(q, k, ef=ef, method=HNSW, **kw)
    return r, seg.counters(), seg.exact_rows(), seg.walk_reruns()


def _check(seg, v, og, q, k, ef, monkeypatch, sim, what="", filter_bits=None, min_score=-1.0, with_duplicates=True,
           multi_vector=False, paragraph_of=None):
    """Both walks against each other and the oracle, every query; returns the queries each walk's first pass flagged
    (fp16-screened, f32-only)."""
    kw = dict(min_score=min_score, with_duplicates=with_duplicates, filter_bits=filter_bits)
    (i32, s32, c32), k32, e32, r32 = _search(seg, q, k, ef, monkeypatch, True, **kw)
    (i16, s16, c16), k16, e16, r16 = _search(seg, q, k, ef, monkeypatch, False, **kw)
    oi, os_, oc, counters = O.hnsw_search(v, og, q, k, ef if ef > 0 else 30, sim=sim, min_score=min_score, with_duplicates=with_duplicates,
                                          multi_vector=multi_vector, filter_bits=filter_bits, paragraph_of=paragraph_of, nthreads=NT)
    for name, ids, sc, cnt in (("f16", i16, s16, c16), ("f32", i32, s32, c32)):
        bad = np.nonzero((ids != oi).any(1) | (cnt != oc) | (sc.view(np.uint32) != os_.view(np.uint32)).any(1))[0]
        assert len(bad) == 0, (what, name, k, ef, bad[:8], len(bad))
    assert k16["overflows"] == 0 and k32["overflows"] == 0, (what, k16, k32)
    assert k16 == k32, (what, k16, k32)
    if with_duplicates:
        assert k16["similarities"] == counters[0] - len(q) * og.entry_layer, (what, k, ef, k16, counters)
        assert k16["expansions"] == counters[1], (what, k, ef, k16, counters)
    assert e32 == k32["similarities"] and e16 <= e32
    return r16, r32


# ---- the reference's default constants --------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def default_graph():
    n, d = 200_000, 64
    v = make_vectors(n, d, seed=61)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_COSINE, m=30, m0=60, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=4096)
    assert seg.counters()["overflows"] == 0, seg.counters()   # the build's own walk kept within its capacities
    rng = np.random.default_rng(62)
    r = rng.standard_normal((16, d)).astype(np.float32)
    q = np.concatenate([make_queries(v, 48, seed=63), r / np.linalg.norm(r, axis=1, keepdims=True)])
    yield seg, v, q, _oracle_graph(seg, n, 30, 60)
    seg.close()


@pytest.mark.parametrize("frac", [0.3, 0.1, 0.05, 0.02])
def test_uniform_filters(default_graph, monkeypatch, frac):
    """A uniform filter passing 30 - 2 % of the rows, k = 10, 20, 100 and ef = 30 (the default) or 128.  Most queries at 10 % and
    below outgrow the first pass's capacities; the line printed per shape gives how many the first pass flagged."""
    seg, v, q, og = default_graph
    bits = _words(_uniform(len(v), frac, seed=64))
    flagged = 0
    for k in (10, 20, 100):
        for ef in (0, 128):
            r16, r32 = _check(seg, v, og, q, k, ef, monkeypatch, O.SIM_COSINE, what=f"filter {frac}", filter_bits=bits)
            print(f"walk_capacity filter={frac} k={k} ef={ef or 30}: first pass flagged {r16} (fp16) / {r32} (f32) of {len(q)}")
            flagged += r16 + r32
    if frac <= 0.1:
        assert flagged > 0, "the shapes no longer reach the re-run"


def test_far_filter(default_graph, monkeypatch):
    """The rows that score in the top 5 % against any of the queries are filtered out: closest_up_nodes starts from seeds the
    filter rejects and walks far from them.  (A filter that keeps only the bottom half makes it pop about half the graph, which
    the re-run's lists, merged in O(length) per hop, take minutes over.)"""
    seg, v, q, og = default_graph
    q = q[::4]
    best = np.max(q @ v.T, axis=0)
    keep = best < np.quantile(best, 0.95)
    flagged = 0
    for k in (10, 100):
        r16, r32 = _check(seg, v, og, q, k, 0, monkeypatch, O.SIM_COSINE, what="far", filter_bits=_words(keep))
        print(f"walk_capacity far filter k={k}: first pass flagged {r16} (fp16) / {r32} (f32) of {len(q)}")
        flagged += r16 + r32
    assert flagged > 0


def test_min_score(default_graph, monkeypatch):
    """min_score at a query's 11th or 101st best score among the rows a 10 % filter passes, k = 100: closest_up_nodes stops at
    min_score (search.rs:206), before or at its k-th result."""
    seg, v, q, og = default_graph
    keep = _uniform(len(v), 0.1, seed=65)
    bits = _words(keep)
    idx = np.nonzero(keep)[0]
    qs = q[::4]
    _, sc, _ = O.brute_force(v[idx], qs, 101, sim=O.SIM_COSINE, nthreads=NT)
    for col in (10, 100):
        for i in range(len(qs)):
            _check(seg, v, og, qs[i : i + 1], 100, 0, monkeypatch, O.SIM_COSINE, what=f"min_score col {col} q {i}", filter_bits=bits,
                   min_score=float(sc[i, col]))


def test_visited_table_capped(default_graph, monkeypatch):
    """A 512-slot table (NIDX_B200_HS_BITS = 9, 416 inserts) cannot hold an unfiltered walk with M0 = 60: every query overflows its
    first pass, in the deferring kernel too, and the re-run returns the oracle's results and counters."""
    seg, v, q, og = default_graph
    monkeypatch.setenv("NIDX_B200_HS_BITS", "9")
    for k, ef in ((10, 0), (10, 128), (100, 0)):
        r16, r32 = _check(seg, v, og, q, k, ef, monkeypatch, O.SIM_COSINE, what=f"capped k={k} ef={ef}")
        assert r16 == len(q) and r32 == len(q), (k, ef, r16, r32)


def test_auto_takes_the_walk_and_equals_the_oracle(default_graph, monkeypatch):
    """A 5 % filter at k = 10 with its match count, as the prefilter hand-off (vector.py search_prefiltered) passes it with
    NIDX_METHOD_AUTO: the reference's cost model picks the walk at 200 000 nodes, and the results are the oracle's."""
    seg, v, q, og = default_graph
    keep = _uniform(len(v), 0.05, seed=66)
    bits = _words(keep)
    assert O.use_hnsw(len(v), int(keep.sum()), 10, M=30)
    monkeypatch.delenv("NIDX_B200_HS_F16", raising=False)
    ids, sc, cnt = seg.search(q, 10, filter_bits=bits, filter_matching=int(keep.sum()), method=_lib.NIDX_METHOD_AUTO)
    c = seg.counters()
    assert c["expansions"] > 0 and c["overflows"] == 0, c   # the walk ran, not the scan
    oi, os_, oc, counters = O.hnsw_search(v, og, q, 10, 30, sim=O.SIM_COSINE, filter_bits=bits, nthreads=NT)
    assert (ids == oi).all() and (cnt == oc).all() and np.array_equal(sc.view(np.uint32), os_.view(np.uint32))
    assert c["similarities"] == counters[0] - len(q) * og.entry_layer and c["expansions"] == counters[1]
    print(f"walk_capacity AUTO filter=0.05 k=10: first pass flagged {seg.walk_reruns()} of {len(q)}")


# ---- pops rejected without a filter -----------------------------------------------------------------------------------------
def test_duplicates_rejected(monkeypatch):
    """with_duplicates=False where 20 % of the rows have exact copies (queries at copied rows among them): closest_up_nodes rejects
    the copies it pops and walks on."""
    n, d = 100_000, 64
    v = make_vectors(n, d, seed=67)
    v[n // 2 : n // 2 + n // 5] = v[: n // 5]
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_COSINE, m=30, m0=60, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=4096)
    og = _oracle_graph(seg, n, 30, 60)
    q = np.concatenate([v[:16] + 0.0, make_queries(v, 32, seed=68)])
    for k in (10, 100):
        _check(seg, v, og, q, k, 0, monkeypatch, O.SIM_COSINE, what="duplicates", with_duplicates=False)
    seg.close()


def test_multi_vector_paragraphs(monkeypatch):
    """8 - 32 vectors per paragraph: closest_up_nodes rejects a pop whose paragraph it has already accepted."""
    rng = np.random.default_rng(69)
    sizes = rng.integers(8, 33, 6000)
    par = np.repeat(np.arange(len(sizes), dtype=np.uint32), sizes)
    n, d = len(par), 64
    v = make_vectors(n, d, seed=70)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_COSINE, m=30, m0=60, ef_construction=100, multi_vector=True, paragraph_of=par)
    seg.build_hnsw(seed=2, max_batch=4096)
    og = _oracle_graph(seg, n, 30, 60)
    q = make_queries(v, 48, seed=71)
    for k in (10, 100):
        r16, r32 = _check(seg, v, og, q, k, 0, monkeypatch, O.SIM_COSINE, what="multi-vector", multi_vector=True, paragraph_of=par)
        print(f"walk_capacity multi-vector k={k}: first pass flagged {r16} (fp16) / {r32} (f32) of {len(q)}")
    seg.close()


# ---- Dot and L2 -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("sim", ["dot", "l2"])
def test_dot_and_l2(monkeypatch, sim):
    """50 000 x 128 rows of norms 0.5 - 2, the 5 % and 10 % filters, k = 10 and 100."""
    n, d = 50_000, 128
    v = make_vectors(n, d, seed=72) * np.random.default_rng(73).uniform(0.5, 2.0, (n, 1)).astype(np.float32)
    v = np.ascontiguousarray(v, dtype=np.float32)
    lib_sim, o_sim = (_lib.NIDX_SIM_DOT, O.SIM_DOT) if sim == "dot" else (_lib.NIDX_SIM_L2, O.SIM_L2)
    seg = VectorSegment.create(v, d, similarity=lib_sim, m=30, m0=60, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=4096)
    og = _oracle_graph(seg, n, 30, 60)
    q = make_queries(v, 48, seed=74)
    for frac in (0.05, 0.1):
        bits = _words(_uniform(n, frac, seed=75))
        for k in (10, 100):
            r16, r32 = _check(seg, v, og, q, k, 0, monkeypatch, o_sim, what=f"{sim} {frac}", filter_bits=bits)
            print(f"walk_capacity {sim} filter={frac} k={k}: first pass flagged {r16} (fp16) / {r32} (f32) of {len(q)}")
    seg.close()


# ---- the benchmark's shape --------------------------------------------------------------------------------------------------
def test_benchmark_shape_costs_one_empty_launch_and_no_sync(monkeypatch):
    """M0 = 32, k = 10, ef = 128, unfiltered, torch tensors in and out: the call launches the query norms, the walk and the re-run
    (which finds no flagged query), nothing else, and returns before a long kernel queued ahead of it on the stream has ended
    (it does not wait on the device).  The results are the oracle's with no overflow."""
    import torch

    n, d = 30_000, 128
    v = make_vectors(n, d, seed=76)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=1024)
    og = _oracle_graph(seg, n, 16, 32)
    q = make_queries(v, 256, seed=77)
    monkeypatch.delenv("NIDX_B200_HS_F16", raising=False)
    dq = torch.as_tensor(q).cuda()
    seg.search(dq, 10, ef=128, method=HNSW)    # the workspace is allocated by the first call
    torch.cuda.synchronize()
    L = _lib.load()
    n0 = L.nidx_launch_count()
    torch.cuda._sleep(1_000_000_000)           # about half a second of one SM on the current stream
    t0 = time.perf_counter()
    ids, sc, cnt = seg.search(dq, 10, ef=128, method=HNSW)
    host_s = time.perf_counter() - t0
    launches = L.nidx_launch_count() - n0
    torch.cuda.synchronize()
    assert launches == 3, launches             # row norms, walk, re-run
    assert host_s < 0.1, host_s
    assert seg.walk_reruns() == 0 and seg.counters()["overflows"] == 0
    oi, os_, oc, counters = O.hnsw_search(v, og, q, 10, 128, sim=O.SIM_COSINE, nthreads=NT)
    assert (ids.cpu().numpy() == oi).all() and (cnt.cpu().numpy() == oc).all()
    assert np.array_equal(sc.cpu().numpy().view(np.uint32), os_.view(np.uint32))
    seg.close()
