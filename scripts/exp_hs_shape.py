"""(Round-2 experiment; the NIDX_B200_HS_PAIR / NIDX_B200_HS_GRID switches it used were removed with the variants they selected.)  Experiment: HNSW search CTA shape (8 warps x 4 CTAs/SM vs 4 warps x 7 CTAs/SM) and batch size, one index, several configurations.
    python scripts/exp_hs_shape.py [n_vectors]"""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench as B  # noqa: E402
from nucliadb_b200 import _lib  # noqa: E402
from nucliadb_b200.segment import VectorSegment  # noqa: E402

n = int(sys.argv[1]) if len(sys.argv) > 1 else 2_000_000
d, k, ef = 768, 10, 128
dev = torch.device("cuda", 0)


class A:
    data, latent, noise = "latent", 16, 0.15


vecs = B.make_vectors(A, n, d, dev, seed=1234567890)
seg = VectorSegment.create(vecs, d, similarity=_lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=200, ef_search=ef, device=0)
qs = {b: [B.gen_queries(vecs, b, seed=123 + i) for i in range(12)] for b in (592, 1024, 1036, 1184, 2048)}
del vecs
seg.build_hnsw(seed=2, max_batch=8192)
torch.cuda.synchronize()
gt = {b: seg.search(qs[b][0], k, method=_lib.NIDX_METHOD_BRUTE)[0].cpu().numpy() for b in qs}
configs = [("8", "0", 1024, "0", "0"), ("8", "0", 1024, "0", "512"), ("8", "0", 1024, "0", "544"), ("8", "0", 1024, "0", "0")]
for w, bits, b, pair, grid in configs:
    os.environ["NIDX_B200_HS_W"], os.environ["NIDX_B200_HS_W4_BITS"], os.environ["NIDX_B200_HS_PAIR"], os.environ["NIDX_B200_HS_GRID"] = w, bits, pair, grid
    out = (torch.empty((b, k), dtype=torch.int32, device=dev), torch.empty((b, k), dtype=torch.float32, device=dev), torch.empty((b,), dtype=torch.int32, device=dev))
    for i in range(3):
        seg.search(qs[b][i], k, ef=ef, method=_lib.NIDX_METHOD_HNSW, out=out)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(12):
        seg.search(qs[b][i], k, ef=ef, method=_lib.NIDX_METHOD_HNSW, out=out)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 12
    ids = seg.search(qs[b][0], k, ef=ef, method=_lib.NIDX_METHOD_HNSW)[0].cpu().numpy()
    c = seg.counters()
    print(json.dumps({"grid": grid, "pair": pair, "warps": w, "hash_bits": bits, "batch": b, "ms": ms, "qps": b / ms * 1e3, "kernel_ms": seg.last_kernel_ms(), "recall": B.recall_at_k(ids, gt[b]),
                      "overflows": c["overflows"], "sims_per_q": c["similarities"] / b}), flush=True)
