"""The N>1 exchange path on CPU: world_size 2 over gloo.  Checks the all_gather plumbing and the global
id mapping of nucliadb_b200.dist against the host model of shard_merge.rs:332-348 (tests/merge_model.py; the CUDA
merge kernels themselves are covered by the gpu tests)."""
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
from merge_model import merge_vector_responses


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from nucliadb_b200.dist import gather_partials, global_ids

    rng = np.random.default_rng(100 + rank)
    nq, k = 7, 5
    scores = np.sort(rng.random((nq, k)).astype(np.float32), axis=1)[:, ::-1].copy()
    ids = rng.integers(0, 1000, (nq, k)).astype(np.int32)
    ids_all, sc_all = gather_partials(torch.from_numpy(ids), torch.from_numpy(scores))
    assert ids_all.shape == (world, nq, k)
    # merge_vector_responses: kmerge_by(score >=) of per-rank lists in rank order, take k
    merged_ids, merged_part = [], []
    for q in range(nq):
        items = merge_vector_responses([sc_all[r, q].tolist() for r in range(world)], k)
        merged_ids.append([int(ids_all[r, q, j]) for r, j in items])
        merged_part.append([r for r, j in items])
    g = global_ids(torch.tensor(merged_ids, dtype=torch.int32), torch.tensor(merged_part, dtype=torch.int32), 1000)
    np.save(os.path.join(out_dir, f"r{rank}.npy"), g.numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_world_size_2_gather_and_global_ids(tmp_path):
    world, port = 2, _free_port()
    mp.spawn(_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    a, b = np.load(tmp_path / "r0.npy"), np.load(tmp_path / "r1.npy")
    assert (a == b).all()                      # every rank ends with the same merged answer
    assert ((a >= 0) & (a < 2000)).all() and (a >= 1000).any() and (a < 1000).any()


def _vector_merge(slot, nq, k):
    """merge_vector_responses (shard_merge.rs:332-348) on the gathered exchange buffer [world, 2, nq, k] (ids, score bits)."""
    g = slot["gathered"].numpy()
    ids, sc = g[:, 0], g[:, 1].view(np.float32)
    out_ids = np.empty((nq, k), dtype=np.int32)
    out_part = np.empty((nq, k), dtype=np.int32)
    for q in range(nq):
        items = merge_vector_responses([sc[r, q].tolist() for r in range(g.shape[0])], k)
        out_ids[q] = [ids[r, q, j] for r, j in items]
        out_part[q] = [r for r, j in items]
    return out_ids, out_part


def _text_merge(slot, nq, k):
    """The text merge (nidx_merge_topk) on the gathered buffer: (score desc, part asc, position asc) -- the parts are segments of
    one index, so part order is docaddr order."""
    g = slot["gathered"].numpy()
    ids, sc = g[:, 0], g[:, 1].view(np.float32)
    out_ids = np.empty((nq, k), dtype=np.int32)
    out_part = np.empty((nq, k), dtype=np.int32)
    for q in range(nq):
        items = sorted(((-float(sc[r, q, j]), r, j) for r in range(g.shape[0]) for j in range(k)))[:k]
        out_ids[q] = [ids[r, q, j] for _, r, j in items]
        out_part[q] = [r for _, r, j in items]
    return out_ids, out_part


def _pipeline_worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from nucliadb_b200.dist import ShardedSearcher

    nq, k, n_batches = 6, 4, 5

    def local_search(batch, ef, slot):          # this rank's segment: deterministic per (rank, batch) partial top-k
        rng = np.random.default_rng(1000 * rank + batch)
        sc = np.sort(rng.random((nq, k)).astype(np.float32), axis=1)[:, ::-1].copy()
        slot["local"][0].copy_(torch.from_numpy(rng.integers(0, 1000, (nq, k)).astype(np.int32)))
        slot["local"][1].copy_(torch.from_numpy(sc.view(np.int32)))

    s = ShardedSearcher(None, nq, k, "cpu", local_search=local_search, merge=lambda slot: _vector_merge(slot, nq, k))
    sequential = [s.search(b, 0) for b in range(n_batches)]
    pipelined = []
    for b in range(n_batches):                  # two batches in flight: exchange of b overlaps the search of b + 1
        s.submit(b, 0)
        if b > 0:
            pipelined.append(s.collect())
    pipelined.append(s.collect())
    for (a_ids, a_part), (b_ids, b_part) in zip(sequential, pipelined):
        assert (a_ids == b_ids).all() and (a_part == b_part).all()
    s.submit(0, 0)
    s.submit(1, 0)
    with pytest.raises(RuntimeError):
        s.submit(2, 0)                          # depth 2
    s.collect(), s.collect()
    with pytest.raises(RuntimeError):
        s.collect()
    np.save(os.path.join(out_dir, f"p{rank}.npy"), np.stack([np.stack(p) for p in pipelined]))
    dist.barrier()
    dist.destroy_process_group()


def test_world_size_2_pipelined_exchange(tmp_path):
    world, port = 2, _free_port()
    mp.spawn(_pipeline_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    a, b = np.load(tmp_path / "p0.npy"), np.load(tmp_path / "p1.npy")
    assert (a == b).all() and (a[:, 1] == 1).any() and (a[:, 1] == 0).any()       # same merged answer on both ranks, from both parts


def _text_worker(rank, world, port, out_dir):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from nucliadb_b200.dist import ShardedTextSearcher, docaddr

    nq, k = 5, 4

    def local_search(batch, ef, slot, **kw):      # this rank's doc partition: partial top-k (score desc, doc asc) + local Count
        rng = np.random.default_rng(7000 * rank + batch)
        sc = np.sort(rng.integers(1, 6, (nq, k)).astype(np.float32), axis=1)[:, ::-1].copy()      # few distinct scores: ties across parts
        docs = np.sort(rng.integers(0, 100, (nq, k)).astype(np.int32), axis=1)
        slot["local"][0].copy_(torch.from_numpy(docs))
        slot["local"][1].copy_(torch.from_numpy(sc.view(np.int32)))
        slot["total"].copy_(torch.full((nq,), 10 + rank, dtype=torch.int64))

    s = ShardedTextSearcher(None, nq, k, "cpu", local_search=local_search, merge=lambda slot: _text_merge(slot, nq, k))
    docs, part, total = s.search(0, None)
    assert (total == 10 + 11).all()                                   # Count collector: summed over the parts
    g = s.slots[0]["gathered"].numpy()
    for q in range(nq):                                               # merge_document_responses: bm25 desc, then shard, then lower docaddr
        items = sorted((-float(g[r, 1].view(np.float32)[q, j]), r, int(g[r, 0][q, j])) for r in range(world) for j in range(k))[:k]
        assert [(r, d) for _, r, d in items] == list(zip(part[q].tolist(), docs[q].tolist()))
    addr = docaddr(torch.from_numpy(docs), torch.from_numpy(part))
    assert ((addr >> 32).numpy() == part).all() and ((addr & 0xFFFFFFFF).numpy() == docs).all()
    np.save(os.path.join(out_dir, f"t{rank}.npy"), addr.numpy())
    dist.barrier()
    dist.destroy_process_group()


def test_world_size_2_sharded_bm25(tmp_path):
    world, port = 2, _free_port()
    mp.spawn(_text_worker, args=(world, port, str(tmp_path)), nprocs=world, join=True)
    assert (np.load(tmp_path / "t0.npy") == np.load(tmp_path / "t1.npy")).all()
