"""SearchRequest.json_filter at 1 M and 5 M resources: the JSON pass and each hand-off, timed with CUDA events.

Corpus: one JSON document per resource, {"price": int in [0, 1000), "cat": one of 50 words, "ok": bool} under t/p, 30 % of the
resources in one of 100 access groups; one paragraph per resource in a vector segment (dimension 4, no graph: only the hand-off is
timed) and in a paragraph segment.  Timed, each as the whole call (they end in a synchronise, as the search path calls them):
  json_pass         JsonIndex.prefilter: the host compile, nidx_txt_prefilter and nidx_txt_resource_bits, for
                    AND(price range, OR(cat, NOT ok)) ANDed with a two-group security tree;
  vector_json       nidx_vec_prefilter_bits with the resources alone (text All under AND);
  vector_json_text  the same under OR with a text result of 30 % of the fields;
  paragraph_mask    nidx_txt_join_mask with the security bits, the text bits and the resource bits under OR.
Medians of --steps calls after --warmup, with min and max; the card's name and power limit are read in the same process.  One
JSON line.

    python scripts/json_filter_bench.py [--resources 1000000 5000000] [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def timed(fn, steps, warmup):
    import torch

    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return {"median_ms": float(np.median(ms)), "min_ms": float(np.min(ms)), "max_ms": float(np.max(ms))}


def one_size(n, steps, warmup):
    import torch

    from test_json_model import op, path

    from nucliadb_b200 import _lib
    from nucliadb_b200 import json_index as J
    from nucliadb_b200.segment import TextSegment, VectorSegment

    rng = np.random.default_rng(n)
    dev = torch.device("cuda", 0)
    price, cat, ok = rng.integers(0, 1000, n), rng.integers(0, 50, n), rng.random(n) < 0.5
    grp = np.where(rng.random(n) < 0.3, rng.integers(0, 100, n), -1)
    rids = [f"{r + 1:032x}" for r in range(n)]   # ascending as strings and as uuid bytes
    t0 = time.perf_counter()
    docs = [(rids[r], [("t/p\x01price", "num", int(price[r])), ("t/p\x01cat", "text", f"w{cat[r]:02d}"), ("t/p\x01ok", "bool", bool(ok[r]))],
             (f"g{grp[r]}",) if grp[r] >= 0 else ()) for r in range(n)]
    ix = J.JsonIndex(docs, device=0)
    build_s = time.perf_counter() - t0
    expr = op("and", path("t/p", "price", int_range=(100, 600)), op("or", path("t/p", "cat", text="w07"), op("not", path("t/p", "ok", boolean=True))))
    security = ["g3", "g42"]
    out = {"resources": n, "index_build_s": build_s}
    out["json_pass"] = timed(lambda: ix.prefilter(expr, security), steps, warmup)
    _, matching, res_bits = ix.prefilter(expr, security)
    out["json_matching"] = int(matching)

    # one paragraph per resource: field key = 16 uuid bytes + "a/title", postings = the paragraph itself
    vec = VectorSegment.create(rng.standard_normal((n, 4)).astype(np.float32), 4, device=0)
    uuid_bytes = np.frombuffer(b"".join(int(r, 16).to_bytes(16, "big") for r in rids), dtype=np.uint8).reshape(n, 16)
    key_bytes = np.ascontiguousarray(np.concatenate([uuid_bytes, np.tile(np.frombuffer(b"a/title", dtype=np.uint8), (n, 1))], axis=1))
    key_off = np.arange(n + 1, dtype=np.uint64) * 23
    post_off = np.arange(n + 1, dtype=np.uint64)
    post = np.arange(n, dtype=np.uint32)
    _lib.check(_lib.load().nidx_vec_set_inverted_index(vec._h, _lib.NIDX_INV_FIELDS, n, _lib.ptr(key_bytes), _lib.ptr(key_off), _lib.ptr(post_off),
                                                       _lib.ptr(post)))
    ranges = torch.from_numpy(np.stack([post_off[:-1], post_off[1:]], axis=1).astype(np.uint64).view(np.int64)).to(dev)
    words = (n + 63) // 64
    text_mask = rng.random(n) < 0.3
    text_words = np.zeros(words * 8, dtype=np.uint8)
    packed = np.packbits(text_mask, bitorder="little")
    text_words[: len(packed)] = packed
    text_bits = torch.from_numpy(text_words.view(np.int64)).to(dev)
    join = torch.from_numpy(np.arange(n, dtype=np.int32)).to(dev)
    out["vector_json"] = timed(lambda: vec.prefilter_bits(None, None, 0, res_bits, ranges, n, n), steps, warmup)
    out["vector_json_text"] = timed(lambda: vec.prefilter_bits(text_bits, join, n, res_bits, ranges, n, n, doc_op=_lib.NIDX_F_OR), steps, warmup)
    _, m1 = vec.prefilter_bits(None, None, 0, res_bits, ranges, n, n)
    _, m2 = vec.prefilter_bits(text_bits, join, n, res_bits, ranges, n, n, doc_op=_lib.NIDX_F_OR)
    out["vector_matching"] = [int(m1), int(m2)]

    par = TextSegment.create(n, 0, np.zeros(1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32), np.zeros(n, dtype=np.uint8))
    sec_bits = torch.from_numpy(np.random.default_rng(1).integers(0, 2 ** 63, words, dtype=np.int64)).to(dev)
    out["paragraph_mask"] = timed(lambda: par.join_mask(sec_bits, text_bits, n, join, res_bits, n, join, _lib.NIDX_F_OR), steps, warmup)
    par.close()
    vec.close()
    ix.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--resources", type=int, nargs="+", default=[1_000_000, 5_000_000])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    from nucliadb_b200 import _lib

    _lib.require_device()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    print(json.dumps({"gpu": gpu, "sizes": [one_size(n, a.steps, a.warmup) for n in a.resources]}))


if __name__ == "__main__":
    main()
