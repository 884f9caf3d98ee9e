"""GPU parity tests: the CUDA path (through the C ABI) against the oracle on the same seeded inputs."""
import numpy as np
import pytest

import oracle as O
from conftest import make_queries, make_vectors
from nucliadb_b200 import _lib
from nucliadb_b200.segment import VectorSegment

pytestmark = pytest.mark.gpu


def _seg(v, sim, **kw):
    return VectorSegment.create(v, v.shape[1], similarity=sim, **kw)


@pytest.mark.parametrize("sim", [_lib.NIDX_SIM_COSINE, _lib.NIDX_SIM_DOT])
@pytest.mark.parametrize("d", [128, 100, 384, 512, 1024, 1536, 2048, 3072, 4096])
def test_brute_force_matches_oracle(sim, d):
    v = make_vectors(5000, d, seed=5)
    if sim == _lib.NIDX_SIM_DOT:
        v = v * np.linspace(0.5, 1.5, len(v), dtype=np.float32)[:, None]
    q = make_queries(v, 37)
    seg = _seg(v, sim)
    ids, sc, cnt = seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)
    oi, os_, oc = O.brute_force(v, q, 10, sim=sim, nthreads=4)
    assert (cnt == oc).all()
    assert (ids == oi).all()                      # ids bit-exact
    assert np.array_equal(sc, os_)                # same summation order => scores bit-exact
    assert np.abs(sc - os_).max() <= 1e-5         # the stated tolerance


def test_brute_force_min_score_and_alive():
    v = make_vectors(3000, 64, seed=6)
    q = make_queries(v, 8)
    seg = _seg(v, _lib.NIDX_SIM_COSINE)
    alive = np.ones(3000, dtype=bool)
    alive[::3] = False
    words = np.zeros((3000 + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(alive, bitorder="little")
    words[: len(pb)] = pb
    bits = words.view(np.uint64)
    seg.set_alive(bits)
    ids, sc, cnt = seg.search(q, 20, min_score=0.5, method=_lib.NIDX_METHOD_BRUTE)
    oi, os_, oc = O.brute_force(v, q, 20, min_score=0.5, alive_bits=bits)
    assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)
    assert all(alive[i] for i in ids[ids != 0xFFFFFFFF])


def test_hnsw_search_matches_oracle_on_oracle_graph(small_data):
    v, q = small_data
    g = O.hnsw_build(v, M=16, M0=32, efC=100, max_batch=64, nthreads=8)
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=100)
    seg.set_graph(g.level, g.adj0, g.adjU, g.w0, g.wU)
    for ef in (30, 128):
        ids, sc, cnt = seg.search(q, 10, ef=ef, method=_lib.NIDX_METHOD_HNSW)
        oi, os_, oc, counters = O.hnsw_search(v, g, q, 10, ef, nthreads=8)
        assert (cnt == oc).all()
        assert (ids == oi).all()                  # same graph, same walk => identical ids
        assert np.array_equal(sc, os_)
        c = seg.counters()
        assert c["overflows"] == 0
        # the kernel carries the entry point's score down the layers instead of recomputing it
        # (search.rs:256-261 recomputes per layer_search): entry_layer fewer evaluations per query
        assert c["similarities"] == counters[0] - len(q) * g.entry_layer and c["expansions"] == counters[1]


def test_hnsw_search_with_dedup_and_filter(small_data):
    v, q = small_data
    v = v.copy()
    v[1000:1010] = v[0:10]          # exact duplicates
    g = O.hnsw_build(v, M=16, M0=32, efC=100, max_batch=64, nthreads=8)
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=100)
    seg.set_graph(g.level, g.adj0, g.adjU)
    keep = np.random.default_rng(3).random(len(v)) < 0.3
    words = np.zeros((len(v) + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(keep, bitorder="little")
    words[: len(pb)] = pb
    bits = words.view(np.uint64)
    qq = np.concatenate([q[:16], v[0:10]])
    ids, sc, cnt = seg.search(qq, 10, ef=64, min_score=0.0, with_duplicates=False, method=_lib.NIDX_METHOD_HNSW, filter_bits=bits)
    oi, os_, oc, _ = O.hnsw_search(v, g, qq, 10, 64, min_score=0.0, with_duplicates=False, filter_bits=bits, nthreads=4)
    assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)


def test_gpu_build_recall_and_invariants():
    v = make_vectors(30000, 96, seed=11)
    q = make_queries(v, 200)
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=1024)
    assert seg.counters()["overflows"] == 0
    g = seg.get_graph()
    # structural invariants (hnsw/params.rs:24-31): degree caps, targets in range and in the layer
    deg0 = (g["adj0"] != 0xFFFFFFFF).sum(1)
    assert deg0.max() <= 32 and deg0.min() >= 1
    assert (g["level"] == O.assign_levels(len(v), 16, 2)).all()
    valid = g["adj0"][g["adj0"] != 0xFFFFFFFF]
    assert valid.max() < len(v)
    bi, _, _ = seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)
    for ef, floor in ((30, 0.90), (128, 0.98)):
        hi, _, _ = seg.search(q, 10, ef=ef, method=_lib.NIDX_METHOD_HNSW)
        rec = np.mean([len(set(a) & set(b)) / 10 for a, b in zip(hi, bi)])
        print("gpu-built graph recall@10 ef", ef, rec)
        assert rec >= floor
    # the oracle searching the GPU-built graph agrees with the GPU searching it
    og = O.Graph(len(v), 16, 32, g["level"])
    og.adj0[:], og.adjU[:] = g["adj0"], g["adjU"][: og.adjU.shape[0]]
    og.entry_node, og.entry_layer = g["entry_node"], g["entry_layer"]
    hi, hs, _ = seg.search(q, 10, ef=64, method=_lib.NIDX_METHOD_HNSW)
    oi, os_, _, _ = O.hnsw_search(v, og, q, 10, 64, nthreads=8)
    assert (hi == oi).all() and np.array_equal(hs, os_)


def test_gpu_build_equals_oracle_batch_build():
    """Same levels, same batch schedule, same arithmetic order => the same graph, edge for edge."""
    v = make_vectors(4000, 64, seed=12)
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=8, m0=16, ef_construction=40)
    seg.build_hnsw(seed=2, max_batch=128)
    g = seg.get_graph()
    og = O.hnsw_build(v, M=8, M0=16, efC=40, seed=2, max_batch=128, nthreads=8)
    assert (g["level"] == og.level).all() and g["entry_node"] == og.entry_node
    same_rows = (g["adj0"] == og.adj0).all(1).mean()
    print("rows identical to the oracle's batch build:", same_rows)
    assert same_rows == 1.0
    assert np.array_equal(g["w0"], og.w0)
    assert (g["adjU"][: og.adjU.shape[0]] == og.adjU).all()


def test_parts_merge_matches_kmerge():
    """The text merge (nidx_merge_topk): per-part sorted lists of the segments of one index merged (score desc, part asc,
    position asc), take k -- part order is docaddr order there.  The vector merge, whose ties follow kmerge_by's heap instead,
    is tested in test_gpu_shard_merge.py."""
    import torch

    from nucliadb_b200.segment import merge_topk

    rng = np.random.default_rng(5)
    parts, nq, k = 5, 33, 10
    sc = np.sort(rng.random((parts, nq, k)).astype(np.float32), axis=2)[:, :, ::-1].copy()
    ids = rng.integers(0, 1 << 20, (parts, nq, k)).astype(np.int32)
    ids[3, :, 6:] = -1          # a short part (NIL padded)
    sc[3, :, 6:] = 0
    sc[1, 0, :3] = sc[0, 0, :3]  # exact ties across parts
    want_ids = np.empty((nq, k), np.int32)
    want_part = np.empty((nq, k), np.int32)
    for q in range(nq):
        items = sorted(((-float(sc[p, q, j]), p, j) for p in range(parts) for j in range(k) if ids[p, q, j] != -1))[:k]
        want_ids[q] = [ids[p, q, j] for _, p, j in items]
        want_part[q] = [p for _, p, j in items]
    dev = torch.device("cuda", 0)
    got = merge_topk(torch.tensor(ids, device=dev), torch.tensor(sc, device=dev))
    assert (got[0].cpu().numpy() == want_ids).all() and (got[2].cpu().numpy() == want_part).all()
    # the same data interleaved as an all-gather buffer [parts, 2, nq, k] merged in place
    buf = torch.empty((parts, 2, nq, k), dtype=torch.int32, device=dev)
    buf[:, 0] = torch.tensor(ids, device=dev)
    buf[:, 1] = torch.tensor(sc, device=dev).view(torch.int32)
    got2 = merge_topk(buf[:, 0], buf[:, 1].view(torch.float32), part_stride=2 * nq * k)
    assert (got2[0].cpu().numpy() == want_ids).all() and (got2[2].cpu().numpy() == want_part).all()


@pytest.mark.parametrize("sim,d", [(_lib.NIDX_SIM_COSINE, 384), (_lib.NIDX_SIM_DOT, 128), (_lib.NIDX_SIM_COSINE, 768), (_lib.NIDX_SIM_COSINE, 512),
                                   (_lib.NIDX_SIM_DOT, 1024), (_lib.NIDX_SIM_COSINE, 1536), (_lib.NIDX_SIM_DOT, 2048), (_lib.NIDX_SIM_COSINE, 3072),
                                   (_lib.NIDX_SIM_DOT, 4096)])
def test_tensor_core_filter_scan_is_bit_exact(sim, d, monkeypatch):
    """Batches of >= 64 queries with k <= 16 take the wgmma TF32 FILTER + exact REFINE path (scan_tc2.cuh): ids and scores must
    equal the oracle's bit for bit -- the tensor cores only decide which vectors are re-scored -- with deletions, min_score, a
    ragged last tile and a ragged last query block; NIDX_B200_SCAN=exact (the CUDA-core kernels) gives the same arrays."""
    n = 20000 + 77
    v = make_vectors(n, d, seed=8)
    if sim == _lib.NIDX_SIM_DOT:
        v *= np.random.default_rng(3).uniform(0.5, 2.0, (n, 1)).astype(np.float32)       # un-normalised: the Dot error bound scales with the norms
    q = make_queries(v, 300)
    seg = _seg(v, sim)
    for k, ms in ((10, -1.0), (16, 0.3), (1, -1.0)):
        oi, os_, oc = O.brute_force(v, q, k, sim=sim, min_score=ms, nthreads=8)
        monkeypatch.setenv("NIDX_B200_SCAN", "tensor")
        ids, sc, cnt = seg.search(q, k, min_score=ms, method=_lib.NIDX_METHOD_BRUTE)
        assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)
        c = seg.scan_counters()
        assert c["survivors"] > 0 and c["full_scans"] < len(q)    # the filter served the batch
        monkeypatch.setenv("NIDX_B200_SCAN", "exact")
        ids2, sc2, cnt2 = seg.search(q, k, min_score=ms, method=_lib.NIDX_METHOD_BRUTE)
        assert (ids2 == ids).all() and np.array_equal(sc2, sc) and (cnt2 == cnt).all()
    alive = np.ones(n, dtype=bool)
    alive[::3] = False
    words = np.zeros((n + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(alive, bitorder="little")
    words[: len(pb)] = pb
    seg.set_alive(words.view(np.uint64))
    monkeypatch.setenv("NIDX_B200_SCAN", "tensor")
    ids, sc, cnt = seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)
    oi, os_, oc = O.brute_force(v, q, 10, sim=sim, alive_bits=words.view(np.uint64), nthreads=8)
    assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)


def test_tensor_core_filter_overflow_falls_back_to_the_exact_scan(monkeypatch):
    """Hundreds of byte-identical vectors: more candidates inside the filter's error margin than a chunk's list holds, so the
    query is flagged and scanned exactly -- same answer as the oracle (ties broken by the lower address)."""
    v = make_vectors(9000, 128, seed=9)
    v[1000:1400] = v[999]                       # 401 copies inside one 2048-vector chunk
    q = make_queries(v, 80)
    q[:20] = v[999] + 1e-3 * q[:20]
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    seg = _seg(v, _lib.NIDX_SIM_COSINE)
    monkeypatch.setenv("NIDX_B200_SCAN", "tensor")
    ids, sc, cnt = seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)
    oi, os_, oc = O.brute_force(v, q, 10, sim=_lib.NIDX_SIM_COSINE, nthreads=8)
    assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)


def test_search_is_reentrant(small_data):
    """Searchers are shared behind an Arc and called from many blocking threads at once (index_cache.rs:41-47,
    shard_search.rs:139-155): concurrent calls on one handle must give the sequential answers."""
    import threading

    v, q = small_data
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=100)
    seg.build_hnsw(seed=2, max_batch=512)
    want_h = seg.search(q, 10, ef=64, method=_lib.NIDX_METHOD_HNSW)
    want_b = seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)
    errors = []

    def worker(kind):
        try:
            for _ in range(20):
                got = seg.search(q, 10, ef=64, method=_lib.NIDX_METHOD_HNSW) if kind else seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)
                want = want_h if kind else want_b
                assert (got[0] == want[0]).all() and np.array_equal(got[1], want[1])
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(i % 2,)) for i in range(6)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


@pytest.mark.parametrize("n", [0, 1, 2, 7, 33])
def test_tiny_segments(n):
    """Edge cases the reference tests exercise: empty segment, one node (hnsw_deserialize_one_node), fewer nodes than M."""
    d = 16
    v = make_vectors(max(n, 1), d, seed=40 + n)[:n]
    q = make_queries(make_vectors(8, d, seed=2), 4)
    seg = VectorSegment.create(v if n else np.zeros((0, d), np.float32), d, similarity=_lib.NIDX_SIM_COSINE, m=4, m0=8, ef_construction=16)
    ids, sc, cnt = seg.search(q, 5, method=_lib.NIDX_METHOD_BRUTE)
    if n == 0:
        assert (cnt == 0).all() and (ids == 0xFFFFFFFF).all()
        return
    oi, os_, oc = O.brute_force(v, q, 5)
    assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)
    seg.build_hnsw(seed=2, max_batch=4)
    g = seg.get_graph()
    og = O.hnsw_build(v, M=4, M0=8, efC=16, seed=2, max_batch=4)
    assert (g["adj0"] == og.adj0).all() and (g["level"] == og.level).all()
    hi, hs, hc = seg.search(q, 5, ef=8, method=_lib.NIDX_METHOD_HNSW)
    gi, gs, gc, _ = O.hnsw_search(v, og, q, 5, 8)
    assert (hc == gc).all() and (hi == gi).all() and np.array_equal(hs, gs)


def test_zero_vectors_and_large_k(small_data):
    """simsimd's cosine edge cases (both norms 0 -> similarity 1, ab == 0 -> 0) and k close to ef."""
    v, q = small_data
    v = v.copy()
    v[7] = 0.0
    qq = np.concatenate([q[:6], np.zeros((1, v.shape[1]), np.float32)])
    g = O.hnsw_build(v, M=16, M0=32, efC=100, max_batch=64, nthreads=8)
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=100)
    seg.set_graph(g.level, g.adj0, g.adjU)
    for k, ef in ((100, 128), (128, 30), (1, 1)):
        bi, bs, bc = seg.search(qq, k, method=_lib.NIDX_METHOD_BRUTE)
        oi, os_, oc = O.brute_force(v, qq, k, nthreads=4)
        assert (bc == oc).all() and (bi == oi).all() and np.array_equal(bs, os_)
        hi, hs, hc = seg.search(qq, k, ef=ef, method=_lib.NIDX_METHOD_HNSW)
        gi, gs, gc, _ = O.hnsw_search(v, g, qq, k, ef, nthreads=4)
        # the all-zero query scores every vector exactly 0 (one big tie): graph walks under exact ties are
        # unspecified in the reference (BinaryHeap order), so only its counts are compared
        assert (hc == gc).all() and (hi[:6] == gi[:6]).all() and np.array_equal(hs[:6], gs[:6])
        assert seg.counters()["overflows"] == 0
    assert bs[6, 0] == 1.0 and bi[6, 0] == 7      # zero query vs the zero vector: distance 0


def test_multi_vector_paragraphs_match_oracle():
    """VectorCardinality::Multi: brute force takes the best vector per paragraph (segment.rs:581-592), the HNSW walk
    keeps one vector per paragraph (NodeFilter.paragraphs, search.rs:159-165)."""
    rng = np.random.default_rng(9)
    n_par = 3000
    num = rng.integers(1, 5, n_par).astype(np.uint32)
    first = np.concatenate([[0], np.cumsum(num)[:-1]]).astype(np.uint32)
    n = int(num.sum())
    v = make_vectors(n, 64, seed=19)
    par_of = np.repeat(np.arange(n_par, dtype=np.uint32), num)
    q = make_queries(v, 24)
    seg = VectorSegment.create(v, 64, similarity=_lib.NIDX_SIM_DOT, m=8, m0=16, ef_construction=40, multi_vector=True, paragraph_of=par_of)
    ids, sc, cnt = seg.search(q, 10, min_score=0.0, method=_lib.NIDX_METHOD_BRUTE)
    oi, os_, oc = O.brute_force(v, q, 10, sim=O.SIM_DOT, min_score=0.0, first_vec=first, num_vec=num)
    assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)
    assert all(len(set(par_of[r[:c]])) == c for r, c in zip(ids, cnt))
    g = O.hnsw_build(v, sim=O.SIM_DOT, M=8, M0=16, efC=40, max_batch=64, nthreads=8)
    seg.set_graph(g.level, g.adj0, g.adjU)
    hi, hs, hc = seg.search(q, 10, ef=40, min_score=0.0, with_duplicates=True, method=_lib.NIDX_METHOD_HNSW)
    gi, gs, gc, _ = O.hnsw_search(v, g, q, 10, 40, sim=O.SIM_DOT, min_score=0.0, with_duplicates=True, multi_vector=True, paragraph_of=par_of, nthreads=4)
    assert (hc == gc).all() and (hi == gi).all() and np.array_equal(hs, gs)
    assert all(len(set(par_of[r[:c]])) == c for r, c in zip(hi, hc))


def test_extend_reuses_the_existing_graph():
    """merge_indexes' fast path (segment.rs:143-167): graph of the first n0 vectors kept, the rest inserted; equal to the oracle
    doing the same, and as good (recall) as a full rebuild."""
    v = make_vectors(6000, 64, seed=61)
    n0 = 4000
    first = _seg(v[:n0], _lib.NIDX_SIM_COSINE, m=8, m0=16, ef_construction=40)
    first.build_hnsw(seed=2, max_batch=256)
    g0 = first.get_graph()
    merged = _seg(v, _lib.NIDX_SIM_COSINE, m=8, m0=16, ef_construction=40)
    rows0 = int(g0["level"].astype(np.int64).sum())
    merged.extend_hnsw(n0, g0["level"], g0["adj0"], g0["adjU"][: max(rows0, 1)], g0["w0"], g0["wU"][: max(rows0, 1)], g0["entry_node"], g0["entry_layer"],
                       seed=2, max_batch=256)
    g = merged.get_graph()
    og0 = O.Graph(n0, 8, 16, g0["level"])
    og0.adj0[:], og0.w0[:] = g0["adj0"], g0["w0"]
    og0.adjU[:], og0.wU[:] = g0["adjU"][: og0.adjU.shape[0]], g0["wU"][: og0.wU.shape[0]]
    og0.entry_node, og0.entry_layer = g0["entry_node"], g0["entry_layer"]
    og = O.hnsw_extend(v, og0, efC=40, seed=2, max_batch=256, nthreads=8)
    assert (g["level"] == og.level).all() and g["entry_node"] == og.entry_node and g["entry_layer"] == og.entry_layer
    assert (g["adj0"] == og.adj0).all() and np.array_equal(g["w0"], og.w0)
    q = make_queries(v, 100)
    bi, _, _ = merged.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)
    hi, _, _ = merged.search(q, 10, ef=64, method=_lib.NIDX_METHOD_HNSW)
    # the oracle's extended graph gives 0.963 on this input, its full rebuild 0.966 (M=8, ef=64)
    assert np.mean([len(set(a) & set(b)) / 10 for a, b in zip(hi, bi)]) >= 0.95
    assert (hi >= n0).any() and (hi < n0).any()      # old and new vectors are both reachable


def test_extend_drops_broken_upper_links():
    """merge_indexes runs fix_broken_graph on the reused graph (segment.rs:162, ram_hnsw.rs:118-123): a layer-1 link to a
    node that only lives in layer 0 is dropped before the new vectors are inserted."""
    v = make_vectors(2500, 32, seed=62)
    n0 = 2000
    og0 = O.hnsw_build(v[:n0], M=8, M0=16, efC=40, max_batch=64, nthreads=8)
    src = int(np.nonzero(og0.level > 0)[0][0])
    bad = int(np.nonzero(og0.level == 0)[0][0])
    row = og0.adjU[int(og0.upper_off[src])]
    slot = min(int((row != O.NIL).sum()), len(row) - 1)
    row[slot] = bad                                        # broken link (appended, or over the last edge of a full row)
    og0.wU[int(og0.upper_off[src]), slot] = 0.25
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=8, m0=16, ef_construction=40)
    rows0 = max(int(og0.level.astype(np.int64).sum()), 1)
    seg.extend_hnsw(n0, og0.level, og0.adj0, og0.adjU[:rows0], og0.w0, og0.wU[:rows0], og0.entry_node, og0.entry_layer, seed=2, max_batch=64)
    og = O.hnsw_extend(v, og0, efC=40, seed=2, max_batch=64, nthreads=8)
    g = seg.get_graph()
    rows = int(og.level.astype(np.int64).sum())
    assert (g["adj0"] == og.adj0).all() and (g["adjU"][:rows] == og.adjU[:rows]).all()
    assert bad not in g["adjU"][int(og.upper_off[src])]


def test_extend_when_a_new_node_raises_the_top_layer():
    """A merge whose new vectors reach a layer the reused graph does not have: the raising node is inserted first from the old
    entry point and becomes the entry point afterwards (deliberate deviation from build.rs:49-55, see DESIGN.md); equal to the
    oracle doing the same, and the reused graph stays reachable."""
    v = make_vectors(3000, 32, seed=63)
    n0 = 2000
    og0 = O.hnsw_build(v[:n0], M=8, M0=16, efC=40, max_batch=64, nthreads=8)
    seed = next(s for s in range(3, 500) if O.assign_levels(len(v) - n0, 8, s).max() > og0.entry_layer)
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=8, m0=16, ef_construction=40)
    rows0 = max(int(og0.level.astype(np.int64).sum()), 1)
    seg.extend_hnsw(n0, og0.level, og0.adj0, og0.adjU[:rows0], og0.w0, og0.wU[:rows0], og0.entry_node, og0.entry_layer, seed=seed, max_batch=64)
    og = O.hnsw_extend(v, og0, efC=40, seed=seed, max_batch=64, nthreads=8)
    g = seg.get_graph()
    assert og.entry_layer > og0.entry_layer and og.entry_node >= n0
    assert g["entry_node"] == og.entry_node and g["entry_layer"] == og.entry_layer and (g["level"] == og.level).all()
    rows = int(og.level.astype(np.int64).sum())
    assert (g["adj0"] == og.adj0).all() and (g["adjU"][:rows] == og.adjU[:rows]).all()
    q = make_queries(v, 100)
    bi, _, _ = seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)
    hi, _, _ = seg.search(q, 10, ef=64, method=_lib.NIDX_METHOD_HNSW)
    assert np.mean([len(set(a) & set(b)) / 10 for a, b in zip(hi, bi)]) >= 0.97 and (hi < n0).any()


def test_l2_similarity_extension():
    """NIDX_SIM_L2 (north_star; the reference has none): -|q - v|^2 as a similarity.  Exact scan and HNSW walk equal the oracle's
    restatement bit for bit; the ranking is the Euclidean nearest-neighbour ranking of a float64 brute force."""
    n, d = 12000, 96
    v = make_vectors(n, d, seed=31) * np.random.default_rng(5).uniform(0.5, 1.5, (n, 1)).astype(np.float32)
    q = make_queries(v, 40) * 1.1
    seg = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_L2, m=16, m0=32, ef_construction=100)
    ids, sc, cnt = seg.search(q, 10, min_score=-1e30, method=_lib.NIDX_METHOD_BRUTE)
    oi, os_, oc = O.brute_force(v, q, 10, sim=O.SIM_L2, min_score=-1e30, nthreads=8)
    assert (cnt == oc).all() and (ids == oi).all() and np.array_equal(sc, os_)
    d2 = ((q[:, None, :].astype(np.float64) - v[None, :, :].astype(np.float64)) ** 2).sum(-1)
    exact = np.argsort(d2, axis=1)[:, :10]
    assert np.mean([len(set(a) & set(b)) / 10 for a, b in zip(ids, exact)]) >= 0.99
    assert np.allclose(-sc, np.take_along_axis(d2, ids.astype(np.int64), 1), rtol=1e-4, atol=1e-4)
    seg.build_hnsw(seed=2, max_batch=512)
    g = seg.get_graph()
    og = O.Graph(n, 16, 32, g["level"])
    og.adj0[:], og.adjU[:] = g["adj0"], g["adjU"][: og.adjU.shape[0]]
    og.entry_node, og.entry_layer = g["entry_node"], g["entry_layer"]
    hi, hs, hc = seg.search(q, 10, ef=64, min_score=-1e30, method=_lib.NIDX_METHOD_HNSW)
    gi, gs, gc, _ = O.hnsw_search(v, og, q, 10, 64, sim=O.SIM_L2, min_score=-1e30, nthreads=8)
    assert (hc == gc).all() and (hi == gi).all() and np.array_equal(hs, gs)
    assert np.mean([len(set(a) & set(b)) / 10 for a, b in zip(hi, ids)]) >= 0.95


@pytest.mark.gpu
def test_normalize_vectors_matches_the_reference_fold():
    """utils.rs:20-23 through nidx_normalize_vectors: sequential f32 fold, bit-identical to the oracle's restatement; host and
    device buffers, a leading dimension larger than d, the reference's own known answers (utils.rs:140-155)."""
    import ctypes as C

    import torch

    L = _lib.require_device()
    rng = np.random.default_rng(5)
    for n, d, ld in [(1, 4, 4), (37, 100, 100), (1000, 768, 768), (5, 3, 8)]:
        a = (rng.standard_normal((n, ld)) * rng.uniform(0.01, 100)).astype(np.float32)
        want = a.copy()
        for i in range(n):
            want[i, :d] = O.normalize(a[i, :d].copy())
        h = a.copy()
        _lib.check(L.nidx_normalize_vectors(0, _lib.ptr(h), C.c_uint64(n), d, ld, _lib.NIDX_MEM_HOST, None))
        assert h.tobytes() == want.tobytes()
        t = torch.from_numpy(a.copy()).cuda()
        _lib.check(L.nidx_normalize_vectors(0, _lib.ptr(t), C.c_uint64(n), d, ld, _lib.NIDX_MEM_DEVICE, None))
        torch.cuda.synchronize()
        assert t.cpu().numpy().tobytes() == want.tobytes()
    v = np.asarray([[3.0, 0.0, 4.0, 0.0]], dtype=np.float32)
    _lib.check(L.nidx_normalize_vectors(0, _lib.ptr(v), C.c_uint64(1), 4, 4, _lib.NIDX_MEM_HOST, None))
    assert v[0].tolist() == [np.float32(3.0) / np.float32(5.0), 0.0, np.float32(4.0) / np.float32(5.0), 0.0]


def test_calls_on_alternating_streams_overlap_and_agree(small_data):
    """One host thread, two streams, device buffers: every call gets a workspace that no call in flight is using (the pool
    hands out one per stream), so the results equal the one-stream results whatever the interleaving."""
    import torch

    v, q = small_data
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=64)
    seg.build_hnsw(seed=2, max_batch=256)
    dq = [torch.from_numpy(np.roll(q, i, axis=0).copy()).cuda() for i in range(6)]
    want = [tuple(t.clone() for t in seg.search(x, 10, ef=64, method=_lib.NIDX_METHOD_HNSW)) for x in dq]
    torch.cuda.synchronize()
    streams = [torch.cuda.Stream() for _ in range(2)]
    got = []
    for rep in range(3):
        for i, x in enumerate(dq):
            with torch.cuda.stream(streams[i % 2]):
                got.append((i, seg.search(x, 10, ef=64, method=_lib.NIDX_METHOD_HNSW)))
    torch.cuda.synchronize()
    for i, (ids, sc, cnt) in got:
        assert torch.equal(ids, want[i][0]) and torch.equal(sc, want[i][1]) and torch.equal(cnt, want[i][2])


def test_auto_with_a_very_large_top_k_takes_the_exact_scan(small_data):
    """The reference puts no limit on top_k; a walk for k = 700 would need more shared memory than a CTA has, so AUTO answers with
    the exhaustive scan (exact results) instead of failing, while an explicit HNSW request reports the limit."""
    v, q = small_data
    seg = _seg(v, _lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=64)
    seg.build_hnsw(seed=2, max_batch=256)
    ids, sc, cnt = seg.search(q[:4], 700, method=_lib.NIDX_METHOD_AUTO)
    bi, bs, bc = seg.search(q[:4], 700, method=_lib.NIDX_METHOD_BRUTE)
    assert (cnt == 700).all() and np.array_equal(ids, bi) and np.array_equal(sc, bs)
    with pytest.raises(_lib.NidxError):
        seg.search(q[:4], 700, method=_lib.NIDX_METHOD_HNSW)
