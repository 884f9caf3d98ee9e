"""The filter pipeline on the device (nidx_vec_set_inverted_index / nidx_vec_filter / nidx_vec_search_formula) against the host
restatement of ParagraphInvertedIndexes::filter (inverted_index/paragraph.rs:124-186) in nucliadb_b200/vector.py."""
import uuid

import numpy as np
import pytest

from nucliadb_b200 import _lib
from nucliadb_b200 import vector as V

pytestmark = pytest.mark.gpu


def _segment(n=700, dim=32, seed=4):
    rng = np.random.default_rng(seed)
    cfg = V.VectorConfig(dimension=dim, similarity=V.Similarity.Dot)
    rids = [f"{i:032x}" for i in range(1, 41)]
    pool = ["/l/a", "/l/ab", "/l/a/x", "/l/b", "/k/c", "/k/c/deep", "/e/PERSON/one", "/e/PERSON/two"]
    elems = []
    for i in range(n):
        labels = [l for l in pool if rng.random() < 0.25]
        field = rng.choice(["a/title", "a/summary", "f/file1", "t/text"])
        v = rng.standard_normal(dim).astype(np.float32)
        elems.append(V.Elem(f"{rids[i % len(rids)]}/{field}/{i}-{i + 1}", [v / np.linalg.norm(v)], labels=labels))
    return V.VectorIndexer.index_elems(elems, cfg), rids, pool


def _random_formula(rng, pool, rids, depth=0):
    r = rng.random()
    if depth >= 3 or r < 0.35:
        return V.Literal(str(rng.choice(pool + ["/l", "/none", "/e/PERSON"])))
    if r < 0.45:
        keys = [f"{rng.choice(rids)}/{rng.choice(['a/title', 'f/file1', 'x/none'])}" for _ in range(int(rng.integers(1, 6)))] + ["not-a-uuid/a/b"]
        return V._KeyPrefixSet(frozenset(keys))
    if r < 0.6:
        return V.Not(_random_formula(rng, pool, rids, depth + 1))
    return V.Operation(str(rng.choice(["and", "or"])), tuple(_random_formula(rng, pool, rids, depth + 1) for _ in range(int(rng.integers(1, 4)))))


def test_device_formula_equals_host_restatement():
    seg, rids, pool = _segment()
    rng = np.random.default_rng(9)
    for trial in range(60):
        clauses = [_random_formula(rng, pool, rids) for _ in range(int(rng.integers(1, 4)))]
        op_and = bool(rng.integers(0, 2))
        want = seg.filter_bitset(clauses, op_and)
        got, matching = seg.device_filter(clauses, op_and)
        assert np.array_equal(got, want), (trial, clauses)
        assert matching == int(want.sum())
    # deletions: the device result is the formula AND the alive set (segment.rs:523-526)
    seg.apply_deletions([f"{rids[0]}/a/title", rids[3]])
    clauses = [V.Not(V.Literal("/none"))]
    got, matching = seg.device_filter(clauses)
    assert np.array_equal(got, seg.alive) and matching == int(seg.alive.sum()) < seg.records


def test_search_with_a_device_formula_matches_the_bitset_path():
    seg, rids, pool = _segment(n=3000, dim=64, seed=6)
    rng = np.random.default_rng(2)
    q = rng.standard_normal((12, 64)).astype(np.float32)
    for clauses in ([V.Literal("/l/a")], [V.Operation("or", (V.Literal("/k/c"), V.Literal("/e/PERSON"))), V.Not(V.Literal("/l/b"))],
                    [V._KeyPrefixSet(frozenset(f"{r}/a/title" for r in rids[:7]))], [V.Literal("/none")]):
        for method in (_lib.NIDX_METHOD_AUTO, _lib.NIDX_METHOD_BRUTE, _lib.NIDX_METHOD_HNSW):
            ids, sc, cnt = seg.search_batch(q, 10, min_score=-1.0, with_duplicates=True, clauses=clauses, method=method)
            mask = seg.filter_bitset(clauses, True) & seg.alive
            if mask.sum() == 0:
                assert (cnt == 0).all() and (ids == 0xFFFFFFFF).all()
                continue
            words = np.zeros((seg.records + 63) // 64 * 8, dtype=np.uint8)
            pb = np.packbits(mask, bitorder="little")
            words[: len(pb)] = pb
            p = _lib.VecSearchParams(10, 0, -1.0, 1, method, words.ctypes.data, int(mask.sum()))
            import ctypes as C

            i2, s2, c2 = np.empty_like(ids), np.empty_like(sc), np.empty_like(cnt)
            _lib.check(_lib.load().nidx_vec_search(seg.segment._h, _lib.ptr(q), C.c_int32(len(q)), C.c_int32(64), _lib.NIDX_MEM_HOST, C.byref(p), _lib.ptr(i2), _lib.ptr(s2),
                                                   _lib.ptr(c2), None))
            assert (cnt == c2).all() and (ids == i2).all() and np.array_equal(sc, s2)
            assert all(mask[seg.paragraph_of(int(v))] for v in ids[ids != 0xFFFFFFFF])


def test_malformed_formulas_are_rejected():
    import ctypes as C

    seg, _, _ = _segment(n=50)
    nodes = (_lib.FilterNode * 2)()
    nodes[0].kind, nodes[0].n = _lib.NIDX_F_AND, 3          # claims three operands, one follows
    nodes[1].kind, nodes[1].n = _lib.NIDX_F_NOT, 0
    m = C.c_uint64()
    with pytest.raises(_lib.NidxError):
        _lib.check(_lib.load().nidx_vec_filter(seg.segment._h, nodes, C.c_int32(2), None, _lib.NIDX_MEM_HOST, C.byref(m), None))
