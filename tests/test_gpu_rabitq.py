"""GPU parity tests for the RaBitQ slice (vector_types/rabitq.rs): codes, estimator and the quantised exact scan,
against oracle/rabitq.hpp (which is pinned to the reference's own test_rabitq_estimate)."""
import numpy as np
import pytest

import oracle as O
from conftest import make_queries, make_vectors
from nucliadb_b200 import _lib
from nucliadb_b200.segment import VectorSegment

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("d", [64, 256, 768, 1984, 2048, 4096])
def test_codes_and_estimates_are_bit_identical(d):
    v = make_vectors(3000, d, seed=51)
    v[5, :7] = 0.0                      # zeros quantise to the negative side (v > 0.0 is false)
    q = make_queries(v, 9)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT)
    seg.rabitq_encode()
    codes = seg.rabitq_codes()
    want = O.rabitq_encode(v, nthreads=4)
    assert codes.shape == want.shape == (3000, d // 8 + 8)        # the reference's vectors.quant record
    assert (codes == want).all()
    est, err = seg.rabitq_estimate(q)
    oest, oerr = O.rabitq_estimate(want, d, q, nthreads=4)
    assert np.array_equal(est, oest) and np.array_equal(err, oerr)
    exact = q @ v.T
    assert np.mean(np.abs(exact - est) < err) > 0.9               # the bound is probabilistic (EPSILON = 1.9)


def test_rabitq_scan_matches_oracle_and_exact_top_k():
    v = make_vectors(30000, 256, seed=52)
    q = make_queries(v, 40)
    seg = VectorSegment.create(v, 256, similarity=_lib.NIDX_SIM_DOT)
    seg.rabitq_encode()
    alive = np.ones(len(v), dtype=bool)
    alive[::7] = False
    words = np.zeros((len(v) + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(alive, bitorder="little")
    words[: len(pb)] = pb
    for k, ms in ((10, 0.0), (50, 0.3), (1, 0.0)):
        ids, sc, cnt = seg.search(q, k, min_score=ms, method=_lib.NIDX_METHOD_BRUTE_RABITQ)
        oi, os_, oc, evals = O.rabitq_brute_force(v, O.rabitq_encode(v, nthreads=4), q, k, min_score=ms, nthreads=4)
        assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)          # the sequential rerank semantics, exactly
        bi, bs, bc = seg.search(q, k, min_score=ms, method=_lib.NIDX_METHOD_BRUTE)
        assert np.mean([len(set(a[:c]) & set(b[:c])) / max(c, 1) for a, b, c in zip(ids, bi, bc)]) >= 0.98
    seg.set_alive(words.view(np.uint64))
    ids, sc, cnt = seg.search(q, 10, min_score=0.0, method=_lib.NIDX_METHOD_BRUTE_RABITQ)
    assert all(alive[i] for i in ids[ids != 0xFFFFFFFF])


def test_rabitq_needs_dot_and_dim_multiple_of_64():
    v = make_vectors(100, 96, seed=1)
    seg = VectorSegment.create(v, 96, similarity=_lib.NIDX_SIM_DOT)
    with pytest.raises(_lib.NidxError):
        seg.rabitq_encode()
    seg = VectorSegment.create(make_vectors(100, 128, seed=1), 128, similarity=_lib.NIDX_SIM_COSINE)
    with pytest.raises(_lib.NidxError):
        seg.rabitq_encode()


def _oracle_graph(seg, n, m, m0):
    g = seg.get_graph()
    og = O.Graph(n, m, m0, g["level"])
    og.adj0[:], og.adjU[:] = g["adj0"], g["adjU"][: og.adjU.shape[0]]
    og.entry_node, og.entry_layer = g["entry_node"], g["entry_layer"]
    return og


@pytest.mark.parametrize("shape", ["8", "4"])
@pytest.mark.parametrize("d,n", [(128, 20000), (768, 6000), (1984, 3000), (2048, 3000), (4096, 3000)])
def test_quantised_walk_matches_oracle(d, n, shape, monkeypatch):
    """hnsw/search.rs:306-383 with a RaBitQ query: ids, scores and the number of estimates / expansions equal the oracle's
    restatement on the same graph (oracle.hnsw_search_rabitq), with and without deletions, duplicates suppression and min_score --
    for both CTA shapes of the kernel (8 warps per query; 4 warps, which large batches take)."""
    monkeypatch.setenv("NIDX_B200_RQ_W", shape)
    v = make_vectors(n, d, seed=61)
    v[100:110] = v[90:100]                                   # byte-identical vectors for with_duplicates=False
    q = make_queries(v, 24)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    seg.build_hnsw(seed=2, max_batch=512)
    seg.rabitq_encode()
    enc = O.rabitq_encode(v, nthreads=4)
    og = _oracle_graph(seg, n, 16, 32)
    for k, ms, dup in ((10, -1.0, True), (10, 0.2, True), (5, -1.0, False), (25, -1.0, True)):
        ids, sc, cnt = seg.search(q, k, min_score=ms, with_duplicates=dup, method=_lib.NIDX_METHOD_HNSW_RABITQ)
        c = seg.counters_ex()
        oi, os_, oc, ocnt = O.hnsw_search_rabitq(v, enc, og, q, k, min_score=ms, with_duplicates=dup, nthreads=4)
        assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)
        # the kernel carries the entry point's estimate from layer to layer, the reference re-evaluates it in every layer_search
        # (search.rs:256-261): entry_layer fewer estimates per query
        assert c["estimates"] == int(ocnt[3]) - len(q) * og.entry_layer and c["expansions"] == int(ocnt[1]) and c["overflows"] == 0
        assert c["similarities"] >= int(ocnt[0]) >= c["rerank_needed"] > 0   # exact similarities: the chunked filter may compute a few more
    # deletions + filter: closest_up_nodes walks on until k alive results are found
    alive = np.ones(n, dtype=bool)
    alive[::3] = False
    words = np.zeros((n + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(alive, bitorder="little")
    words[: len(pb)] = pb
    bits = words.view(np.uint64)
    seg.set_alive(bits)
    ids, sc, cnt = seg.search(q, 10, method=_lib.NIDX_METHOD_HNSW_RABITQ)
    oi, os_, oc, _ = O.hnsw_search_rabitq(v, enc, og, q, 10, min_score=-1.0, filter_bits=bits, nthreads=4)
    assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)
    assert all(alive[i] for i in ids[ids != 0xFFFFFFFF])


def test_auto_takes_the_quantised_walk_on_a_segment_with_codes():
    """segment.rs:506-513 + 538: a segment that carries codes is searched with a RaBitQ query; on a large unfiltered segment the cost
    model picks the graph, i.e. the quantised walk; recall against the exact scan stays high (the reference's recall test takes this
    path: segment.rs:841-912)."""
    n, d = 40000, 256
    v = make_vectors(n, d, seed=62)
    q = make_queries(v, 64)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=1024)
    seg.rabitq_encode()
    a_ids, a_sc, a_cnt = seg.search(q, 10, method=_lib.NIDX_METHOD_AUTO)
    est = seg.counters_ex()["estimates"]
    w_ids, w_sc, w_cnt = seg.search(q, 10, method=_lib.NIDX_METHOD_HNSW_RABITQ)
    assert est > 0 and (a_ids == w_ids).all() and np.array_equal(a_sc, w_sc)
    b_ids, _, _ = seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)
    recall = np.mean([len(set(a) & set(b)) / 10 for a, b in zip(w_ids, b_ids)])
    assert recall >= 0.97, recall


def test_vectors_quant_round_trip(tmp_path):
    """vectors.quant (data_store/v2/quant_vector_store.rs:29-62): written with the segment, byte for byte the reference's records
    (the oracle's encoder), and loaded as is by nidx_vec_open -- a segment written by the reference keeps its codes."""
    n, d = 2000, 128
    v = make_vectors(n, d, seed=71)
    q = make_queries(v, 16)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    seg.build_hnsw(seed=2, max_batch=256)
    seg.rabitq_encode()
    seg.save(str(tmp_path))
    raw = np.fromfile(tmp_path / "vectors.quant", dtype=np.uint8).reshape(n, d // 8 + 8)
    assert np.array_equal(raw, O.rabitq_encode(v, nthreads=4))
    want = seg.search(q, 10, method=_lib.NIDX_METHOD_HNSW_RABITQ)
    # a "reference-written" directory: the codes come from the file, nothing is re-encoded
    back = VectorSegment.open(str(tmp_path), d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    assert np.array_equal(back.rabitq_codes(), raw)
    got = back.search(q, 10, method=_lib.NIDX_METHOD_AUTO)         # AUTO: codes present + graph => the quantised walk
    assert all(np.array_equal(a, b) for a, b in zip(want, got))
    (tmp_path / "vectors.quant").write_bytes(raw.tobytes()[:-3])
    with pytest.raises(_lib.NidxError):
        VectorSegment.open(str(tmp_path), d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)


@pytest.mark.parametrize("shape", ["8", "4"])
def test_quantised_walk_with_the_reference_graph_constants(shape, monkeypatch):
    """params.rs:34-46: M = 30, M0 = 60 (adjacency rows of 64 slots: two passes of 32 neighbours per expansion), efC = 100."""
    monkeypatch.setenv("NIDX_B200_RQ_W", shape)
    n, d = 8000, 256
    v = make_vectors(n, d, seed=77)
    q = make_queries(v, 16)
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT, m=30, m0=60, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=512)
    seg.rabitq_encode()
    enc = O.rabitq_encode(v, nthreads=4)
    og = _oracle_graph(seg, n, 30, 60)
    ids, sc, cnt = seg.search(q, 10, method=_lib.NIDX_METHOD_HNSW_RABITQ)
    c = seg.counters_ex()
    oi, os_, oc, ocnt = O.hnsw_search_rabitq(v, enc, og, q, 10, nthreads=4)
    assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)
    assert c["expansions"] == int(ocnt[1]) and c["overflows"] == 0
