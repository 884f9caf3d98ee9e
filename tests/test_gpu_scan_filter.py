"""The exhaustive scan's tensor-core filter (scan_tc2.cuh) against the CUDA-core scan and the oracle, bit for bit (ids, scores as
bits, counts), on the inputs where a TF32 filter goes wrong: non-finite and extreme rows and queries, rankings that TF32
inverts, every filter schedule, and the edges of the path's selection.  Each case also asserts, through
VectorSegment.scan_counters(), whether the filter ran or the segment / query fell back to the exact scan as it should."""
import numpy as np
import pytest
import torch

import oracle as O
from conftest import make_queries, make_vectors
from nucliadb_b200 import _lib
from nucliadb_b200.segment import VectorSegment
from test_scan_filter_bound import absorption, approx_scores, exact_scores, low_bits_set, tf32

pytestmark = pytest.mark.gpu
BRUTE = _lib.NIDX_METHOD_BRUTE


def same(a, b):
    ids, sc, cnt = a
    oi, os_, oc = b
    assert (cnt == oc).all(), np.nonzero(cnt != oc)[0][:8]
    assert (ids == oi).all(), np.nonzero((ids != oi).any(1))[0][:8]
    assert np.array_equal(np.asarray(sc, np.float32).view(np.uint32), np.asarray(os_, np.float32).view(np.uint32))


def three_way(seg, v, q, k, sim, monkeypatch, min_score=-1.0, mode="tensor"):
    """tensor (or the default choice when mode is None) vs exact vs the oracle; returns the filter's counters of the first."""
    want = O.brute_force(v, q, k, sim=sim, min_score=min_score, nthreads=8)
    if mode is None:
        monkeypatch.delenv("NIDX_B200_SCAN", raising=False)
    else:
        monkeypatch.setenv("NIDX_B200_SCAN", mode)
    got = seg.search(q, k, min_score=min_score, method=BRUTE)
    same(got, want)
    counters = seg.scan_counters()
    monkeypatch.setenv("NIDX_B200_SCAN", "exact")
    same(seg.search(q, k, min_score=min_score, method=BRUTE), want)
    assert seg.scan_counters() == dict(survivors=0, full_scans=0)
    return counters


def ran(c, nq):
    """The filter ran and served queries from its survivors (a query whose list may have overflowed is scanned in full)."""
    return c["survivors"] > 0 and c["full_scans"] < nq


FELL_BACK = dict(survivors=0, full_scans=0)
SIMS = [_lib.NIDX_SIM_COSINE, _lib.NIDX_SIM_DOT]


def base(n=4096 + 37, d=128, nq=96, seed=21):
    v = make_vectors(n, d, seed=seed)
    return v, make_queries(v, nq, seed=seed)


# ---- non-finite and extreme rows ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [1, 10, 16])
@pytest.mark.parametrize("kind", ["nan", "inf", "nan_low_payload"])
@pytest.mark.parametrize("sim", SIMS)
def test_a_non_finite_row_keeps_the_segment_on_the_exact_scan(sim, kind, k, monkeypatch):
    """Cosine scores a NaN row 1.0 for every query (the distance clamps to 0); a +inf element under Dot gives +inf where q_i > 0;
    a NaN whose payload is only in the 13 low bits is +inf to a tf32 operand.  The filter cannot rank such rows, so the segment
    takes the exact scan -- and returns what the small-batch kernel and the oracle return."""
    v, q = base()
    q[:, 0] = np.abs(q[:, 0]) + np.float32(0.01)
    bad = {"nan": np.float32(np.nan), "inf": np.float32(np.inf), "nan_low_payload": np.uint32(0x7F800001).view(np.float32)}[kind]
    v[1234, 0] = bad
    v[3000:3003, 5] = bad
    c = three_way(VectorSegment.create(v, 128, similarity=sim), v, q, k, sim, monkeypatch)
    assert c == FELL_BACK


@pytest.mark.parametrize("sim", SIMS)
def test_extreme_rows(sim, monkeypatch):
    """The fp16 screen's mix: zero rows, rows at 1e-20 and 1e18.  Under cosine a 1e-20 row's |v|^2 is not a normal f32, so its
    stored norm is outside the bound: the segment falls back.  Dot has no norms in its approximation and keeps the filter: its
    margin scales with max |v| = 1e18, and so do the winning scores (the 1e18 rows), so the selection serves the queries."""
    v, q = base(nq=80)
    v[10:20] = 0.0
    v[100:140] *= np.float32(1e-20)
    v[200:240] *= np.float32(1e18)
    q[:8] = v[100:108] * np.float32(1e20)
    q[8:16] = v[200:208] / np.float32(1e18)
    for k in (1, 10, 16):
        c = three_way(VectorSegment.create(v, 128, similarity=sim), v, q, k, sim, monkeypatch)
        if sim == _lib.NIDX_SIM_COSINE:
            assert c == FELL_BACK
        else:
            # the 40 large rows share one list, which may overflow for a few queries; every other query keeps at least its k
            # best approximations as survivors
            assert c["full_scans"] <= len(q) // 10 and c["survivors"] >= k * (len(q) - c["full_scans"])


@pytest.mark.parametrize("sim", SIMS)
def test_rows_whose_norm_underflows_or_overflows(sim, monkeypatch):
    """Rows at 1e-25 (|v|^2 underflows: stored norm 0, yet cosine scores them 1.0 or -inf through ab / 0) and rows whose elements
    span 1e-20 .. 1e20 (|v|^2 overflows: norm +inf)."""
    rng = np.random.default_rng(4)
    v, q = base(nq=72)
    v[50:60] *= np.float32(1e-25)
    q[:4] = v[50:54] * np.float32(1e25)
    c = three_way(VectorSegment.create(v, 128, similarity=sim), v, q, 10, sim, monkeypatch)
    assert c == FELL_BACK if sim == _lib.NIDX_SIM_COSINE else c["survivors"] > 0
    w = v.copy()
    w[300:310] = rng.standard_normal((10, 128)).astype(np.float32) * (10.0 ** rng.uniform(-20, 20, (10, 128))).astype(np.float32)
    c = three_way(VectorSegment.create(w, 128, similarity=sim), w, q, 10, sim, monkeypatch)
    assert c == FELL_BACK


# ---- non-finite queries -----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("k", [1, 10, 16])
@pytest.mark.parametrize("sim", SIMS)
def test_non_finite_and_zero_queries_are_scanned_exactly(sim, k, monkeypatch):
    v, q = base(nq=128)
    bad = [0, 5, 17, 64, 100, 127]
    q[0, 3] = np.nan
    q[5, 0] = np.inf
    q[17, 7] = -np.inf
    q[64] = np.inf
    q[100] = 0.0
    q[127] = np.uint32(0x7F800001).view(np.float32)
    c = three_way(VectorSegment.create(v, 128, similarity=sim), v, q, k, sim, monkeypatch)
    assert c["survivors"] > 0 and len(bad) <= c["full_scans"] < len(q)


# ---- rankings TF32 inverts ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("sim", SIMS)
def test_rankings_inverted_by_tf32(sim, monkeypatch):
    """A query and a row whose elements lose the most to tf32 truncation (13 low mantissa bits set, so the row equal to the query
    wins exactly) against tf32-exact rows: tf32(q) with some elements one tf32 step up.  Those rank below the winner exactly and
    above it in the filter's model.  The refine must still return the exact ranking."""
    rng = np.random.default_rng(8)
    d, n, nq = 384, 6000, 96
    v = make_vectors(n, d, seed=30)
    q = low_bits_set(np.abs(make_queries(v, nq, seed=31)))
    for i in range(nq):
        a = 40 * i + 7
        v[a] = q[i]
        near = np.repeat(tf32(q[i])[None, :], 30, 0).view(np.uint32)
        for j in range(30):
            near[j, rng.choice(d, 10 + 10 * j, replace=False)] += np.uint32(0x2000)
        v[a + 1: a + 31] = near.view(np.float32)
    ex = exact_scores(q[0], v[7:38], sim)
    ap = approx_scores(q[0], v[7:38], sim)
    assert ex[0] == ex.max() and (ap[1:] > ap[0]).sum() >= 10            # the model inverts the ranking of query 0
    for k in (1, 10, 16):
        c = three_way(VectorSegment.create(v, d, similarity=sim), v, q, k, sim, monkeypatch)
        assert c["survivors"] > 0


@pytest.mark.parametrize("sim", SIMS)
def test_absorption_input_at_4096_dimensions(sim, monkeypatch):
    """The input on which a round-toward-zero sum loses 2.4e-3 of |q||v| (above the fixed 2.2e-3 margin): the row equal to the
    query must win against tf32-exact rows a little below it."""
    d = 4096
    rng = np.random.default_rng(9)
    a = absorption(d)
    v = make_vectors(2048 + 64, d, seed=33)
    v[1000] = a
    v[1001:1061] = tf32(a[None, :] * (1 - rng.uniform(0, 2.4e-3, (60, 1))).astype(np.float32))
    q = np.concatenate([a[None, :], make_queries(v, 71, seed=34)]).astype(np.float32)
    for k in (1, 10, 16):
        c = three_way(VectorSegment.create(v, d, similarity=sim), v, q, k, sim, monkeypatch)
        assert c["survivors"] > 0


# ---- schedules --------------------------------------------------------------------------------------------------------------

def test_lists_that_persist_across_chunks(monkeypatch):
    """60 k vectors, 1 000 queries: 30 chunks, 8 query blocks, fewer CTAs per block than chunks -- a list spans several chunks."""
    v = make_vectors(60000, 384, seed=41)
    q = make_queries(v, 1000, seed=42)
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    n_chunks, n_qblocks = (60000 + 2047) // 2048, (1000 + 127) // 128
    slots = max(1, min(min(n_chunks * n_qblocks, sm) // n_qblocks, n_chunks))
    assert slots < n_chunks
    seg = VectorSegment.create(v, 384, similarity=_lib.NIDX_SIM_COSINE)
    assert ran(three_way(seg, v, q, 10, _lib.NIDX_SIM_COSINE, monkeypatch), 1000)


def test_one_slot_schedule_with_more_query_blocks_than_sms(monkeypatch):
    """More 128-query blocks than SMs: one CTA per block at a time, each CTA serving several blocks."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    nq = 128 * sm + 77
    v = make_vectors(2048 + 5, 128, seed=43)
    q = make_queries(v, nq, seed=44)
    for sim in SIMS:
        seg = VectorSegment.create(v, 128, similarity=sim)
        c = three_way(seg, v, q, 10, sim, monkeypatch)
        assert c["survivors"] > 0


def test_more_survivors_than_the_cap_without_an_overflowing_list(monkeypatch):
    """12 chunks -> 12 slots x 2 column halves = 24 lists; 23 near-copies of one row in each list: no list overflows, but 552
    survivors exceed the refine's cap of 512, so those queries are scanned in full."""
    v = make_vectors(12 * 2048, 128, seed=45)
    rng = np.random.default_rng(46)
    idx = np.arange(len(v))
    for ch in range(12):
        for half in range(2):
            members = idx[(idx // 2048 == ch) & ((idx % 128) // 64 == half)][:23]
            v[members] = v[0] * (1 + rng.uniform(-1e-5, 1e-5, (len(members), 1))).astype(np.float32)
    q = make_queries(v, 100, seed=47)
    q[:20] = v[0]
    c = three_way(VectorSegment.create(v, 128, similarity=_lib.NIDX_SIM_COSINE), v, q, 10, _lib.NIDX_SIM_COSINE, monkeypatch)
    assert c["survivors"] > 0 and c["full_scans"] >= 20


# ---- edges of the path's selection ------------------------------------------------------------------------------------------

def test_edges_of_the_filter_path(monkeypatch):
    v, q = base(nq=64)
    seg = VectorSegment.create(v, 128, similarity=_lib.NIDX_SIM_COSINE)
    sim = _lib.NIDX_SIM_COSINE
    assert ran(three_way(seg, v, q, 16, sim, monkeypatch, mode=None), 64)
    assert three_way(seg, v, q, 17, sim, monkeypatch, mode=None) == FELL_BACK           # k above 16
    assert ran(three_way(seg, v, q, 10, sim, monkeypatch, mode=None), 64)               # 64 queries: the filter
    assert three_way(seg, v, q[:63], 10, sim, monkeypatch, mode=None) == FELL_BACK       # 63: the small-batch kernels
    for n in (127, 128, 2047, 2048, 2049):
        w = v[:n]
        s = VectorSegment.create(w, 128, similarity=sim)
        c = three_way(s, w, q, 10, sim, monkeypatch)
        assert c == FELL_BACK if n < 128 else ran(c, 64)
