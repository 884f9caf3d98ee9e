"""The cross-part merges of a sharded search on one GPU, against the host models: nidx_shard_merge on crafted exchange records
(kmerge_by for vector shards, Fssc for the segments of one index), nidx_vec_shard_record on several segments of one GPU, the
de-duplication keys of shard_keys_kernel, the text merge against a whole-index BM25 search, and nidx_vec_search_sharded at world
size 1 against its two halves."""
import numpy as np
import pytest

from merge_model import merge_vector_responses
from nucliadb_b200 import _lib
from nucliadb_b200.dist import shard_merge, shard_record

pytestmark = pytest.mark.gpu
NIL = 0xFFFFFFFF
# few distinct values: exact ties within and across parts, ties straddling k, signed zeros and infinities
POOL = np.array([np.inf, 3.0, 2.0, 2.0, 1.0, 0.0, -0.0, -0.0, -1.0, -np.inf], dtype=np.float32)


def _dev():
    import torch

    return torch.device("cuda", 0)


def _crafted_parts(rng, n_parts, nq, k):
    """ids [n_parts, nq, k] u32 (NIL padded), scores f32 (each row sorted descending, garbage after the first NIL)."""
    ids = rng.integers(0, 1 << 30, (n_parts, nq, k), dtype=np.uint32)
    sc = np.full((n_parts, nq, k), 7.0, dtype=np.float32)          # past the first NIL: must never be read as a result
    lens = rng.integers(0, k + 1, (n_parts, nq))
    lens[rng.random((n_parts, nq)) < 0.2] = 0                      # empty parts
    lens[rng.random((n_parts, nq)) < 0.3] = k                      # full parts
    if nq > 2:
        lens[:, 1] = 0                                             # a query with every part empty
    for p in range(n_parts):
        for q in range(nq):
            n = lens[p, q]
            row = rng.choice(POOL, n)
            row = row[np.argsort(-row.astype(np.float64), kind="stable")]   # descending; -0.0 and 0.0 stay in drawn order
            sc[p, q, :n] = row
            ids[p, q, n:] = NIL
    return ids, sc, lens


def _records(ids, sc, par=None, vec=None):
    """Exchange records laid end to end: per part [ids][scores] (+ [par_key u64][vec_key u64])."""
    import torch

    n_parts = ids.shape[0]
    words = [ids.reshape(n_parts, -1), sc.view(np.uint32).reshape(n_parts, -1)]
    if par is not None:
        words += [par.reshape(n_parts, -1).view(np.uint32), vec.reshape(n_parts, -1).view(np.uint32)]
    flat = np.ascontiguousarray(np.concatenate(words, axis=1)).reshape(-1)
    return torch.from_numpy(flat.view(np.int32)).to(_dev())


def _np(out):
    import torch

    if isinstance(out[0], torch.Tensor):
        torch.cuda.synchronize()
        return out[0].cpu().numpy().view(np.uint32), out[1].cpu().numpy(), out[2].cpu().numpy(), out[3].cpu().numpy()
    return out


def _kmerge_expected(ids, sc, lens, k):
    n_parts, nq, _ = ids.shape
    e_ids = np.full((nq, k), NIL, dtype=np.uint32)
    e_sc = np.zeros((nq, k), dtype=np.float32)
    e_part = np.full((nq, k), -1, dtype=np.int32)
    e_cnt = np.zeros(nq, dtype=np.int32)
    for q in range(nq):
        got = merge_vector_responses([sc[p, q, :lens[p, q]].tolist() for p in range(n_parts)], k)
        for i, (p, j) in enumerate(got):
            e_ids[q, i], e_sc[q, i], e_part[q, i] = ids[p, q, j], sc[p, q, j], p
        e_cnt[q] = len(got)
    return e_ids, e_sc, e_part, e_cnt


def _assert_same(got, want):
    g_ids, g_sc, g_part, g_cnt = got
    w_ids, w_sc, w_part, w_cnt = want
    assert np.array_equal(g_cnt, w_cnt)
    assert np.array_equal(g_ids, w_ids)
    assert np.array_equal(g_part, w_part)
    assert np.array_equal(g_sc.view(np.uint32), w_sc.view(np.uint32))          # bit for bit: -0.0 stays -0.0


# ---- dedup = 0: merge_vector_responses ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 10, 100, 1024])
@pytest.mark.parametrize("n_parts", [1, 2, 3, 5, 8, 16, 64])
def test_kmerge_crafted_records(n_parts, k):
    rng = np.random.default_rng(1000 * n_parts + k)
    nq = 33
    ids, sc, lens = _crafted_parts(rng, n_parts, nq, k)
    want = _kmerge_expected(ids, sc, lens, k)
    rec = _records(ids, sc)
    _assert_same(_np(shard_merge(rec, n_parts, nq, k)), want)
    _assert_same(shard_merge(rec, n_parts, nq, k, host=True), want)


@pytest.mark.parametrize("nq,n_parts,k", [(1, 5, 10), (1, 3, 100), (1025, 5, 10), (1025, 3, 100)])
def test_kmerge_crafted_records_batch_edges(nq, n_parts, k):
    rng = np.random.default_rng(nq + 7 * n_parts + k)
    ids, sc, lens = _crafted_parts(rng, n_parts, nq, k)
    _assert_same(_np(shard_merge(_records(ids, sc), n_parts, nq, k)), _kmerge_expected(ids, sc, lens, k))


@pytest.mark.parametrize("n_parts", [2, 3, 5])
def test_kmerge_hand_ties_and_the_text_merge(n_parts):
    """Every part scores (1, 1, 0.5): the vector merge follows itertools' heap, the text merge (nidx_merge_topk) keeps (score desc,
    part asc, position asc), and the two differ -- already at k = 1, where the tie straddles k."""
    import torch

    from nucliadb_b200.segment import merge_topk, merge_vector_parts

    k, nq = 3, 2
    sc = np.tile(np.array([1.0, 1.0, 0.5], dtype=np.float32), (n_parts, nq, 1))
    ids = (np.arange(n_parts * nq * k, dtype=np.uint32) + 100).reshape(n_parts, nq, k)
    lens = np.full((n_parts, nq), k)
    for kk in (1, 2, k):
        want = merge_vector_responses([[1.0, 1.0, 0.5]] * n_parts, kk)
        sub_ids, sub_sc = np.ascontiguousarray(ids[:, :, :kk]), np.ascontiguousarray(sc[:, :, :kk])
        got = _np(shard_merge(_records(sub_ids, sub_sc), n_parts, nq, kk))
        assert [(int(p), int(i)) for p, i in zip(got[2][0], got[0][0])] == [(p, int(ids[p, 0, j])) for p, j in want]
        t_ids, t_sc = torch.from_numpy(sub_ids.view(np.int32)).to(_dev()), torch.from_numpy(sub_sc).to(_dev())
        vp = merge_vector_parts(t_ids, t_sc)
        tp = merge_topk(t_ids, t_sc)
        torch.cuda.synchronize()
        assert [(int(p), int(i)) for p, i in zip(vp[2][0].tolist(), vp[0][0].cpu().numpy().view(np.uint32))] == [(p, int(ids[p, 0, j])) for p, j in want]
        text_order = [int(p) for p in tp[2][0].tolist()]
        assert text_order == sorted(text_order)                                   # lower part first
        assert text_order != [p for p, _ in want]


def test_kmerge_parts_merge_in_place_with_stride():
    """nidx_merge_vector_parts on an all-gather buffer [parts, 2, nq, k] merged in place (part_stride = 2 nq k)."""
    import torch

    from nucliadb_b200.segment import merge_vector_parts

    rng = np.random.default_rng(9)
    n_parts, nq, k = 6, 17, 12
    ids, sc, lens = _crafted_parts(rng, n_parts, nq, k)
    e_ids, e_sc, e_part, _ = _kmerge_expected(ids, sc, lens, k)
    buf = torch.empty((n_parts, 2, nq, k), dtype=torch.int32, device=_dev())
    buf[:, 0] = torch.from_numpy(ids.view(np.int32)).to(_dev())
    buf[:, 1] = torch.from_numpy(sc.view(np.int32)).to(_dev())
    got = merge_vector_parts(buf[:, 0], buf[:, 1].view(torch.float32), part_stride=2 * nq * k)
    torch.cuda.synchronize()
    assert np.array_equal(got[0].cpu().numpy().view(np.uint32), e_ids) and np.array_equal(got[2].cpu().numpy(), e_part)
    assert np.array_equal(got[1].cpu().numpy().view(np.uint32), e_sc.view(np.uint32))


# ---- dedup = 1: Fssc -------------------------------------------------------------------------------------------------------------------
def _fssc_expected(ids, sc, par, vec, lens, k, with_duplicates):
    from nucliadb_b200.vector import _Fssc

    n_parts, nq, _ = ids.shape
    e_ids = np.full((nq, k), NIL, dtype=np.uint32)
    e_sc = np.zeros((nq, k), dtype=np.float32)
    e_part = np.full((nq, k), -1, dtype=np.int32)
    e_cnt = np.zeros(nq, dtype=np.int32)
    for q in range(nq):
        f = _Fssc(k, with_duplicates)
        for p in range(n_parts):
            for j in range(lens[p, q]):
                f.add(int(par[p, q, j]), float(sc[p, q, j]), (p, j), int(vec[p, q, j]))
        res = f.result()
        for i, (s, _, (p, j)) in enumerate(res):
            e_ids[q, i], e_sc[q, i], e_part[q, i] = ids[p, q, j], sc[p, q, j], p
        e_cnt[q] = len(res)
    return e_ids, e_sc, e_part, e_cnt


def _fssc_case(n_parts, nq, k, seed, key_pool):
    rng = np.random.default_rng(seed)
    ids, sc, lens = _crafted_parts(rng, n_parts, nq, k)
    par = rng.integers(0, key_pool, (n_parts, nq, k)).astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)   # keys repeated across parts
    vec = rng.integers(0, key_pool, (n_parts, nq, k)).astype(np.uint64) << np.uint64(33)                   # vectors repeated across parts
    return ids, sc, par, vec, lens


@pytest.mark.parametrize("with_duplicates", [0, 1])
@pytest.mark.parametrize("n_parts,k", [(1, 10), (2, 1), (3, 10), (5, 10), (8, 100), (16, 10), (64, 10)])
def test_fssc_crafted_records(n_parts, k, with_duplicates):
    """Repeated paragraph keys (evict-then-skip shrinks the collection), repeated vectors, tied minima at eviction (the first in
    insertion order goes): equal to _Fssc exactly."""
    nq = 33
    ids, sc, par, vec, lens = _fssc_case(n_parts, nq, k, 31 * n_parts + k + with_duplicates, key_pool=max(2, k))
    want = _fssc_expected(ids, sc, par, vec, lens, k, with_duplicates)
    assert k == 1 or (want[3] < np.minimum(lens.sum(0), k)).any()   # the keys did suppress entries
    rec = _records(ids, sc, par, vec)
    _assert_same(_np(shard_merge(rec, n_parts, nq, k, dedup=True, with_duplicates=with_duplicates)), want)
    _assert_same(shard_merge(rec, n_parts, nq, k, dedup=True, with_duplicates=with_duplicates, host=True), want)


def test_fssc_evict_then_skip_by_hand():
    """Full at k = 2 with {a: 1.0, b: 0.5}; a candidate (a, 0.9) evicts b then finds `a` present: the collection shrinks to 1."""
    ids = np.array([[[10, 11]], [[20, NIL]]], dtype=np.uint32)
    sc = np.array([[[1.0, 0.5]], [[0.9, 7.0]]], dtype=np.float32)
    par = np.array([[[1, 2]], [[1, 0]]], dtype=np.uint64)
    vec = np.array([[[5, 6]], [[7, 0]]], dtype=np.uint64)
    got = _np(shard_merge(_records(ids, sc, par, vec), 2, 1, 2, dedup=True, with_duplicates=1))
    assert got[3].tolist() == [1] and got[0][0].tolist() == [10, NIL] and got[2][0].tolist() == [0, -1]


@pytest.mark.parametrize("n_parts,k,fits", [(120, 100, True), (121, 100, False), (64, 100, True)])
def test_fssc_shared_memory_edges(n_parts, k, fits):
    """per = 16 k + 8 n_parts k bytes per query: 97 600 B at 120 parts fits 96 KiB (one thread per block), 98 400 B at 121 is
    refused; 52 800 B at 64 parts takes the opt-in above 48 KiB."""
    nq = 3
    ids, sc, par, vec, lens = _fssc_case(n_parts, nq, k, n_parts, key_pool=300)
    rec = _records(ids, sc, par, vec)
    if not fits:
        with pytest.raises(_lib.NidxError, match="too large"):
            shard_merge(rec, n_parts, nq, k, dedup=True, with_duplicates=0)
        return
    for with_duplicates in (0, 1):
        want = _fssc_expected(ids, sc, par, vec, lens, k, with_duplicates)
        _assert_same(_np(shard_merge(rec, n_parts, nq, k, dedup=True, with_duplicates=with_duplicates)), want)


# ---- nidx_vec_shard_record on several segments of one GPU ----------------------------------------------------------------------------
def _segments(d, n, n_parts, multi=False, seed=3):
    """n_parts segments sharing byte-identical rows (exact score ties across parts), each with an HNSW graph."""
    from nucliadb_b200.segment import VectorSegment

    rng = np.random.default_rng(seed)
    shared = rng.standard_normal((n // 4, d)).astype(np.float32)
    segs, rows, pofs = [], [], []
    for r in range(n_parts):
        v = rng.standard_normal((n, d)).astype(np.float32)
        v[: n // 4] = shared
        pof = np.repeat(np.arange(n // 2, dtype=np.uint32), 2) if multi else None
        s = VectorSegment.create(v, d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64, multi_vector=multi, paragraph_of=pof)
        s.build_hnsw(seed=2, max_batch=256)
        segs.append(s)
        rows.append(v)
        pofs.append(pof)
    q = shared[rng.integers(0, n // 4, 24)] + 0.01 * rng.standard_normal((24, d)).astype(np.float32)
    return segs, rows, pofs, q.astype(np.float32)


def _filter_bits(n_par, seed):
    keep = np.random.default_rng(seed).random(n_par) < 0.5
    words = np.zeros((n_par + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(keep, bitorder="little")
    words[: len(pb)] = pb
    return words.view(np.uint64)


@pytest.mark.parametrize("method", [_lib.NIDX_METHOD_HNSW, _lib.NIDX_METHOD_BRUTE, _lib.NIDX_METHOD_AUTO])
@pytest.mark.parametrize("multi", [False, True])
def test_records_of_segments_merge_like_the_models(method, multi):
    import torch

    from nucliadb_b200.vector import _Fssc

    n_parts, n, d, k = 4, 2000, 64, 10
    segs, rows, pofs, q = _segments(d, n, n_parts, multi=multi)
    n_par = n // 2 if multi else n
    tq = torch.from_numpy(q).to(_dev())
    for filtered in (False, True):
        fb = _filter_bits(n_par, 5) if filtered else None
        fb_t = torch.from_numpy(fb.view(np.int64)).to(_dev()) if filtered else None
        kw = dict(ef=64, method=method, filter_bits=fb)
        kw_t = dict(kw, filter_bits=fb_t)
        # ---- dedup = 0 over host and device queries ----
        plain = [s.search(q, k, **kw) for s in segs]
        for queries, kwq in ((q, kw), (tq, kw_t)):
            rec = torch.cat([shard_record(s, queries, k, rank=r, **kwq) for r, s in enumerate(segs)])
            torch.cuda.synchronize()
            for r in range(n_parts):
                part = rec[r * 2 * len(q) * k:(r + 1) * 2 * len(q) * k].cpu().numpy()
                assert np.array_equal(part[: len(q) * k].view(np.uint32), plain[r][0].reshape(-1))
                assert np.array_equal(part[len(q) * k:].view(np.uint32), plain[r][1].reshape(-1).view(np.uint32))
            ids = np.stack([p[0] for p in plain])
            sc = np.stack([p[1] for p in plain])
            lens = np.stack([p[2] for p in plain])
            _assert_same(_np(shard_merge(rec, n_parts, len(q), k)), _kmerge_expected(ids, sc, lens, k))
        # ---- dedup = 1: paragraph keys unset ((rank << 32) | p) and set (shared across parts), with_duplicates 0 and 1 ----
        for keyed in (False, True):
            for r, s in enumerate(segs):
                s.set_paragraph_keys(np.arange(n_par, dtype=np.uint64) * np.uint64(7) + np.uint64(1) if keyed else None)
            for with_dup in (True, False):
                loc = [s.search(q, k, with_duplicates=with_dup, **kw) for s in segs]
                rec = torch.cat([shard_record(s, tq, k, rank=r, dedup=True, with_duplicates=with_dup, **kw_t) for r, s in enumerate(segs)])
                got = _np(shard_merge(rec, n_parts, len(q), k, dedup=True, with_duplicates=with_dup))
                for i in range(len(q)):
                    f = _Fssc(k, with_dup)
                    for r in range(n_parts):
                        li, ls, lc = loc[r]
                        for j in range(int(lc[i])):
                            a = int(li[i, j])
                            p = int(pofs[r][a]) if multi else a
                            key = p * 7 + 1 if keyed else (r << 32) | p
                            f.add(key, float(ls[i, j]), (r, a), rows[r][a].tobytes())
                    res = f.result()
                    assert int(got[3][i]) == len(res)
                    assert [(int(got[2][i, j]), int(got[0][i, j])) for j in range(len(res))] == [pl for _, _, pl in res]
                    assert np.array_equal(got[1][i, :len(res)], np.array([s for s, _, _ in res], dtype=np.float32))
        for s in segs:
            s.set_paragraph_keys(None)


@pytest.mark.parametrize("d", [100, 4096])
def test_record_vector_hash_and_paragraph_keys(d):
    """vec_key is equal for byte-identical rows and differs for a one-ulp change and for -0.0 against +0.0 (first, middle and last
    element), and for equal values at swapped positions; par_key = (rank << 32) | p without keys, keys[p] with them.  Every row is
    a one-vector segment of its own, so the search's own duplicate suppression cannot hide one."""
    import torch

    from nucliadb_b200.segment import VectorSegment

    rng = np.random.default_rng(d)
    base = rng.standard_normal(d).astype(np.float32)
    positions = [0, d // 2, d - 1]
    base[positions] = 0.0
    variants = [base.copy(), base.copy()]                             # 0 and 1: byte-identical
    for i in positions:
        v = base.copy()
        v[i] = -0.0                                                   # signed zero
        variants.append(v)
        v = base.copy()
        v[i] = np.nextafter(np.float32(0.0), np.float32(1.0))         # one element one ulp away
        variants.append(v)
    for x, y in ((1.0, 2.0), (2.0, 1.0)):                             # the same values at swapped positions
        v = base.copy()
        v[positions[0]], v[positions[1]] = x, y
        variants.append(v)
    q = np.ones((1, d), dtype=np.float32)
    constants = set()
    for rank, keyed in ((0, False), (5, False), (2, True)):
        hashes = []
        for i, row in enumerate(variants):
            seg = VectorSegment.create(row[None], d, similarity=_lib.NIDX_SIM_DOT)
            if keyed:
                seg.set_paragraph_keys(np.array([0x1234567 * (i + 1)], dtype=np.uint64))
            rec = shard_record(seg, q, 1, rank=rank, dedup=True, min_score=-np.inf, method=_lib.NIDX_METHOD_BRUTE, with_duplicates=False)
            torch.cuda.synchronize()
            w = rec.cpu().numpy().view(np.uint32)
            assert w[0] == 0
            par, vec = int(w[2:4].view(np.uint64)[0]), int(w[4:6].view(np.uint64)[0])
            assert par == (0x1234567 * (i + 1) if keyed else rank << 32)
            hashes.append(vec)
            kept = shard_record(seg, q, 1, rank=rank, dedup=True, min_score=-np.inf, method=_lib.NIDX_METHOD_BRUTE, with_duplicates=True)
            torch.cuda.synchronize()
            constants.add(int(kept.cpu().numpy().view(np.uint32)[4:6].view(np.uint64)[0]))
            seg.close()
        assert hashes[0] == hashes[1]
        assert len(set(hashes[1:])) == len(variants) - 1
    assert len(constants) == 1                                        # duplicates kept: the rows are not hashed


# ---- the text merge: N parts of one index scored with the whole index's statistics -------------------------------------------------
@pytest.mark.parametrize("n_parts", [1, 3, 7])
def test_text_parts_merge_equals_whole_index(n_parts):
    import torch

    import oracle as O
    from nucliadb_b200.segment import TextSegment, merge_topk

    rng = np.random.default_rng(40 + n_parts)
    n_docs, n_terms = 3000, 300
    lens = rng.integers(3, 40, n_docs)
    doc_off = np.concatenate([[0], np.cumsum(lens)])
    tokens = (rng.zipf(1.3, doc_off[-1]) % n_terms).astype(np.uint32)
    for src in range(0, n_docs, 10):                                   # duplicated documents: exact score ties across parts
        a, b = doc_off[src], doc_off[src + 1]
        dst = n_docs - 1 - src
        if doc_off[dst + 1] - doc_off[dst] == b - a:
            tokens[doc_off[dst]:doc_off[dst + 1]] = tokens[a:b]
    whole = O.Postings(doc_off, tokens, n_terms)
    wseg = TextSegment.create(whole.n_docs, whole.n_terms, whole.term_off, whole.post_doc, whole.post_tf, whole.fieldnorm_id)
    cuts = np.sort(rng.choice(np.arange(1, n_docs), n_parts - 1, replace=False)) if n_parts > 1 else np.array([], dtype=np.int64)
    bounds = np.concatenate([[0], cuts, [n_docs]]).astype(np.int64)
    parts = []
    for r in range(n_parts):
        lo, hi = bounds[r], bounds[r + 1]
        P = O.Postings(doc_off[lo:hi + 1] - doc_off[lo], tokens[doc_off[lo]:doc_off[hi]], n_terms)
        t = TextSegment.create(P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id)
        t.set_stats(whole.n_docs, whole.total_tokens, whole.doc_freq)
        parts.append(t)
    queries = [list(rng.integers(0, n_terms, rng.integers(1, 5))) for _ in range(40)]
    qoff = np.concatenate([[0], np.cumsum([len(x) for x in queries])]).astype(np.uint32)
    qt = np.concatenate(queries).astype(np.uint32)
    nq = len(queries)
    for mode in (_lib.NIDX_BM25_OR, _lib.NIDX_BM25_AND):
        for k, min_score in ((1, 0.0), (10, 0.0), (37, 0.0), (20, 4.0)):
            wd, ws, wc, wt = wseg.search(qt, qoff, k, mode=mode, min_score=min_score)
            res = [t.search(qt, qoff, k, mode=mode, min_score=min_score) for t in parts]
            ids = torch.from_numpy(np.stack([r[0] for r in res]).view(np.int32)).to(_dev())
            sc = torch.from_numpy(np.stack([r[1] for r in res])).to(_dev())
            md, ms, mp = merge_topk(ids, sc)
            torch.cuda.synchronize()
            md, ms, mp = md.cpu().numpy().view(np.uint32), ms.cpu().numpy(), mp.cpu().numpy()
            gdoc = np.where(mp >= 0, bounds[np.maximum(mp, 0)] + md.astype(np.int64), NIL).astype(np.uint32)
            assert np.array_equal(gdoc, wd)
            assert np.array_equal(ms.view(np.uint32), ws.view(np.uint32))
            assert np.array_equal((md != NIL).sum(1), wc)
            assert np.array_equal(sum(r[3].astype(np.int64) for r in res), wt.astype(np.int64))


# ---- world size 1: nidx_vec_search_sharded = nidx_vec_shard_record + nidx_shard_merge ------------------------------------------
def test_world_size_1_equals_record_then_merge():
    import torch

    from nucliadb_b200.dist import ShardComm

    comm = ShardComm(0, 1, 0, exchange=lambda b: b)
    segs, rows, pofs, q = _segments(64, 2000, 1, seed=8)
    seg = segs[0]
    seg.set_paragraph_keys(np.arange(2000, dtype=np.uint64) % np.uint64(700))
    tq = torch.from_numpy(q).to(_dev())
    for dedup in (False, True):
        for with_dup in (True, False):
            for method in (_lib.NIDX_METHOD_HNSW, _lib.NIDX_METHOD_BRUTE):
                a = comm.search_vectors(seg, q, 10, ef=64, dedup=dedup, with_duplicates=with_dup, method=method)
                rec = shard_record(seg, tq, 10, rank=0, dedup=dedup, ef=64, with_duplicates=with_dup, method=method)
                b = shard_merge(rec, 1, len(q), 10, dedup=dedup, with_duplicates=with_dup, host=True)
                _assert_same(b, a)
                c = _np(comm.search_vectors(seg, tq, 10, ef=64, dedup=dedup, with_duplicates=with_dup, method=method))
                _assert_same(c, a)
    seg.set_paragraph_keys(None)
    comm.close()
