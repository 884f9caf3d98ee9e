"""nidx_vec_search_sharded / nidx_txt_search_sharded over the library's own NCCL communicator: world size 2, one process per
GPU, launched with torch.distributed.run (the rendezvous only hands the NCCL id round).  Needs two GPUs: skipped on a
one-GPU machine (`python -m pytest tests/test_gpu_shard_nccl.py -m gpu` on a machine with two GPUs)."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_sharded_search_world_size_2():
    import torch

    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    env = dict(os.environ, OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1", "--master-port", "29541",
                        os.path.join(ROOT, "tests", "shard_worker.py")], env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0 and "shard worker ok" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]


def test_sharded_entry_points_world_size_1():
    """A one-rank communicator: the sharded entry points (search -> ncclAllGather -> merge, all on one stream) must return the
    plain search's results; runs on every GPU box, so the exchange code is exercised by the default GPU suite."""
    import numpy as np

    import oracle as O
    from nucliadb_b200 import _lib
    from nucliadb_b200.dist import ShardComm
    from nucliadb_b200.segment import TextSegment, VectorSegment

    comm = ShardComm(0, 1, 0, exchange=lambda b: b)
    rng = np.random.default_rng(3)
    v = rng.standard_normal((2000, 64)).astype(np.float32)
    v[100:200] = v[:100]                                    # byte-identical pairs
    q = v[rng.integers(0, 2000, 16)] + 0.05 * rng.standard_normal((16, 64)).astype(np.float32)
    seg = VectorSegment.create(v, 64, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=64)
    seg.build_hnsw(seed=2, max_batch=256)
    for dedup in (False, True):
        for with_dup in (True, False):
            li, ls, lc = seg.search(q, 10, ef=64, method=_lib.NIDX_METHOD_HNSW, with_duplicates=with_dup)
            ids, sc, part, cnt = comm.search_vectors(seg, q, 10, ef=64, dedup=dedup, with_duplicates=with_dup)
            assert (cnt == lc).all() and np.array_equal(ids, li) and np.array_equal(sc, ls) and (part[ids != 0xFFFFFFFF] == 0).all()
    lens = rng.integers(5, 60, 3000)
    doc_off = np.concatenate([[0], np.cumsum(lens)])
    P = O.Postings(doc_off, (rng.zipf(1.3, doc_off[-1]) % 400).astype(np.uint32), 400)
    ts = TextSegment.create(P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id)
    ts.set_stats(P.n_docs, P.total_tokens, P.doc_freq)
    queries = [list(rng.integers(0, 400, 4)) for _ in range(12)]
    qoff = np.concatenate([[0], np.cumsum([len(x) for x in queries])]).astype(np.uint32)
    qt = np.concatenate(queries).astype(np.uint32)
    d0, s0, c0, t0 = ts.search(qt, qoff, 20)
    d1, s1, p1, c1, t1 = comm.search_text(ts, qt, qoff, 20)
    assert np.array_equal(d0, d1) and np.array_equal(s0, s1) and (c0 == c1).all() and (t0 == t1).all()
    comm.close()
