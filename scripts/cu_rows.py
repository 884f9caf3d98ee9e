"""f32 rows per query of the HNSW search at bench.py's flagship shape (10 M x 768 cosine, M = 16, efC = 200, ef = 128, batch 1024,
bench.py's `latent` data and queries), with and without the reads of closest_up_nodes.

At k = 1 closest_up_nodes returns the list's top entry without expanding it, so k = 10 and k = 1 walk the same layers and differ
only by closest_up_nodes.  Before it deferred the neighbours the layer-0 walk had visited, it read one row for each of its
similarities: rows(k = 10) = rows(k = 1) + similarities(k = 10) - similarities(k = 1).  One JSON line, with the card's name and
power limit.

    python scripts/cu_rows.py [--vectors 10000000] [--batches 3]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              check=True).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--vectors", type=int, default=10_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--batches", type=int, default=3)
    ap.add_argument("--ef", type=int, default=128)
    a = ap.parse_args()
    import torch

    import bench
    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import VectorSegment

    _lib.require_device()
    dev = torch.device("cuda", 0)
    vecs = bench.gen_vectors(a.vectors, a.dim, dev, seed=1234567890, latent=16, noise=0.15)
    queries = [bench.gen_queries(vecs, a.batch, seed=123 + i) for i in range(a.batches)]
    seg = VectorSegment.create(vecs, a.dim, similarity=_lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=200, ef_search=a.ef)
    del vecs
    torch.cuda.empty_cache()
    seg.build_hnsw(seed=2, max_batch=8192)
    per = {}
    for k in (1, 10):
        sims = rows = overflows = 0
        for q in queries:
            seg.search(q, k, ef=a.ef, method=_lib.NIDX_METHOD_HNSW)
            torch.cuda.synchronize()
            c = seg.counters()
            sims += c["similarities"]
            overflows += c["overflows"]
            rows += seg.exact_rows()
        nq = a.batch * a.batches
        per[k] = dict(similarities=sims / nq, rows=rows / nq, overflows=overflows)
    before = per[1]["rows"] + per[10]["similarities"] - per[1]["similarities"]
    print(json.dumps({"metric": "f32 rows per query", "workload": f"HNSW search {a.vectors}x{a.dim} cosine, ef={a.ef}, {a.batches} batches of {a.batch}",
                      "k10_rows_without_deferral": before, "k10_rows": per[10]["rows"], "k1_rows": per[1]["rows"],
                      "row_bytes": a.dim * 4, "per_k": per, "card": card()}))


if __name__ == "__main__":
    main()
