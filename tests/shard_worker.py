"""Worker of tests/test_gpu_shard_nccl.py: launched once per rank by torch.distributed.run (WORLD_SIZE ranks, one GPU each).
Every rank builds ALL the parts on its own GPU as well (small data), so it can compute what the sharded calls must return
without the exchange -- local searches merged on the host by the reference's rules -- and compare."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def fssc_merge(parts, k, with_duplicates):
    """searcher.rs:150-199 over parts = [(ids, scores, par_keys, vec_bytes)] of ONE query (the Python _Fssc of vector.py)."""
    from nucliadb_b200.vector import _Fssc

    f = _Fssc(k, with_duplicates)
    for part, (ids, scores, keys, vbytes) in enumerate(parts):
        for i in range(len(ids)):
            if ids[i] == 0xFFFFFFFF:
                break
            f.add(int(keys[i]), float(scores[i]), (part, int(ids[i])), vbytes[i])
    return [(s, p) for s, _, p in f.result()]


def main():
    import torch
    import torch.distributed as dist

    import oracle as O
    from merge_model import merge_vector_responses
    from nucliadb_b200 import _lib
    from nucliadb_b200.dist import ShardComm
    from nucliadb_b200.segment import TextSegment, VectorSegment

    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")          # only to hand the NCCL id round: the data path is the library's own communicator
    comm = ShardComm(rank, world, local)
    rng = np.random.default_rng(5)
    n, d, nq, k = 3000, 64, 40, 10
    # parts share some byte-identical vectors and some paragraph keys, so the de-duplicating merge has work to do
    base = rng.standard_normal((n, d)).astype(np.float32)
    base /= np.linalg.norm(base, axis=1, keepdims=True)
    parts_v, parts_keys = [], []
    for r in range(world):
        v = rng.standard_normal((n, d)).astype(np.float32)
        v /= np.linalg.norm(v, axis=1, keepdims=True)
        v[: n // 10] = base[: n // 10]                      # the same vectors in every part
        keys = (np.arange(n, dtype=np.uint64) + np.uint64(r * 10 * n))
        keys[n // 10: n // 5] = np.arange(n // 10, n // 5, dtype=np.uint64) + np.uint64(77_000_000)   # the same paragraph ids in every part
        parts_v.append(v)
        parts_keys.append(keys)
    q = base[rng.integers(0, n // 5, nq)] + 0.05 * rng.standard_normal((nq, d)).astype(np.float32)
    q = (q / np.linalg.norm(q, axis=1, keepdims=True)).astype(np.float32)
    segs = []
    for r in range(world):
        s = VectorSegment.create(parts_v[r], d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64, device=local)
        s.build_hnsw(seed=2, max_batch=256)
        s.set_paragraph_keys(parts_keys[r])
        segs.append(s)
    local_res = [s.search(q, k, ef=64, method=_lib.NIDX_METHOD_HNSW) for s in segs]

    # ---- dedup = 0: merge_vector_responses (kmerge_by(score >=) over the parts in rank order; ties as itertools' heap orders them) ----
    ids, sc, part, cnt = comm.search_vectors(segs[rank], q, k, ef=64, dedup=False)
    for i in range(nq):
        cand = merge_vector_responses([local_res[r][1][i, :int(local_res[r][2][i])].tolist() for r in range(world)], k)
        exp = [(r, int(local_res[r][0][i, j]), float(local_res[r][1][i, j])) for r, j in cand]
        got = [(int(part[i, j]), int(ids[i, j]), float(sc[i, j])) for j in range(int(cnt[i]))]
        assert got == exp, (rank, i, got, exp)
    # ---- dedup = 1: Fssc, with and without byte-identical suppression; device and host paths ----
    for with_dup in (True, False):
        ids, sc, part, cnt = comm.search_vectors(segs[rank], q, k, ef=64, dedup=True, with_duplicates=with_dup)
        tq = torch.from_numpy(q).cuda(local)
        tids, tsc, tpart, tcnt = comm.search_vectors(segs[rank], tq, k, ef=64, dedup=True, with_duplicates=with_dup)
        torch.cuda.synchronize()
        assert np.array_equal(tids.cpu().numpy().astype(np.uint32), ids) and np.array_equal(tsc.cpu().numpy(), sc) and np.array_equal(tpart.cpu().numpy(), part)
        loc = [s.search(q, k, ef=64, method=_lib.NIDX_METHOD_HNSW, with_duplicates=with_dup) for s in segs]
        for i in range(nq):
            parts = []
            for r in range(world):
                li, ls, lc = loc[r]
                c = int(lc[i])
                vb = [parts_v[r][int(x)].tobytes() for x in li[i, :c]]
                parts.append((li[i, :c], ls[i, :c], parts_keys[r][li[i, :c].astype(np.int64)], vb))
            exp = fssc_merge(parts, k, with_dup)
            got = [(float(sc[i, j]), (int(part[i, j]), int(ids[i, j]))) for j in range(int(cnt[i]))]
            assert got == exp, (rank, with_dup, i, got, exp)

    # ---- BM25 over a document-partitioned index ----
    n_docs, n_terms = 4000 * world, 500
    lens = rng.integers(5, 60, n_docs)
    doc_off = np.concatenate([[0], np.cumsum(lens)])
    tokens = (rng.zipf(1.3, doc_off[-1]) % n_terms).astype(np.uint32)
    whole = O.Postings(doc_off, tokens, n_terms)
    per = n_docs // world
    tsegs = []
    for r in range(world):
        lo, hi = r * per, (r + 1) * per
        P = O.Postings(doc_off[lo:hi + 1] - doc_off[lo], tokens[doc_off[lo]:doc_off[hi]], n_terms)
        t = TextSegment.create(P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id, device=local)
        t.set_stats(whole.n_docs, whole.total_tokens, whole.doc_freq)
        tsegs.append(t)
    queries = [list(rng.integers(0, n_terms, 4)) for _ in range(24)]
    qoff = np.concatenate([[0], np.cumsum([len(x) for x in queries])]).astype(np.uint32)
    qt = np.concatenate(queries).astype(np.uint32)
    docs, sc, part, cnt, total = comm.search_text(tsegs[rank], qt, qoff, 20, mode=_lib.NIDX_BM25_OR, use_tf=True)
    od, osc, oc, otot = O.bm25_search(whole, queries, 20, mode=O.BM25_OR, use_tf=True)
    assert (total == otot).all() and (cnt == oc).all()
    assert np.allclose(sc, osc, rtol=1e-5, atol=1e-5)
    gdoc = np.where(part >= 0, part.astype(np.int64) * per + docs.astype(np.int64), -1)
    for i in range(len(queries)):
        c = int(cnt[i])
        assert set(gdoc[i, :c].tolist()) == set(od[i, :c].astype(np.int64).tolist()) or abs(osc[i, c - 1] - osc[i, c - 2]) < 2e-5
    dist.barrier()
    comm.close()
    dist.destroy_process_group()
    if rank == 0:
        print("shard worker ok")


if __name__ == "__main__":
    main()
