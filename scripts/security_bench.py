"""SearchRequest.security on one text segment of prefilter_bench's corpus shape (Zipf(1.07) vocabulary, lognormal lengths of mean
64, three fields per resource, 64 labels), with access groups added: 1 000 groups under 10 top-level groups, 3 per grouped resource,
30 % of the resources public.  Reports prefilter_eval_kernel's time for the security tree of a 3-group request alone and ANDed with a
facet, and the BM25 OR-50 top-100 call (nidx_txt_search) unmasked against the same call on a masked view (nidx_txt_view + the search
+ closing the view), alternating, at batch 1 and 1024, with a check that a view under an all-ones mask returns the unmasked bytes.

One JSON line; kernel times from CUDA events, call times from a host clock around work that ends in a synchronise, medians after
warm-up; the card's name and power limit are read in the same process.

    python scripts/security_bench.py [--docs 5000000] [--steps 20] [--warmup 3]
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
sys.path.insert(0, os.path.join(ROOT, "scripts"))

N_GROUPS, GROUPS_PER_RES, PUBLIC = 1000, 3, 0.3


def group_column(n, seed=5):
    """Group keys (facet order: g{00..09}\\0s{000..099}) and every document's ords, a resource being three consecutive documents."""
    rng = np.random.default_rng(seed)
    keys = sorted(b"g%02d\0s%03d" % (i // 100, i % 100) for i in range(N_GROUPS))
    n_res = (n + 2) // 3
    ords = np.sort(rng.integers(0, N_GROUPS, (n_res, GROUPS_PER_RES)), axis=1)
    keep = np.ones_like(ords, dtype=bool)
    keep[:, 1:] = ords[:, 1:] != ords[:, :-1]
    keep[rng.random(n_res) < PUBLIC] = False
    per_res = keep.sum(1)
    res = np.arange(n) // 3
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum(per_res[res])
    return keys, off, ords[res][keep[res]].astype(np.uint32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=5_000_000)
    ap.add_argument("--terms", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import torch

    from phrase_bench import make_positional_corpus
    from prefilter_bench import LABELS_PER_DOC, N_LABELS, columns, node_array

    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import TextSegment
    from nucliadb_b200.text import fieldnorm_to_id

    _lib.require_device()
    dev = torch.device("cuda", 0)
    n = a.docs
    c = make_positional_corpus(n, a.terms, dev)
    lut = np.asarray([fieldnorm_to_id(i) for i in range(int(c["lens"].max()) + 1)], dtype=np.uint8)
    df = np.diff(c["term_off"].astype(np.int64)).astype(np.uint64)
    ts = TextSegment.create(n, a.terms, c["term_off"], c["post_doc"], c["post_tf"], lut[c["lens"]])
    ts.set_stats(n, int(c["lens"].sum()), df)
    _res, _fld, off, ords, _created = columns(n)
    ts.set_facets([b"l\0%03d" % i for i in range(N_LABELS)], off, ords)
    keys, goff, gords = group_column(n)
    ts.set_doc_groups(keys, goff, gords)
    P = _lib
    # a request of three groups: one top-level group (100 keys), two leaves
    security = [(P.NIDX_P_OR, 4, 0, 0, None), (P.NIDX_P_PUBLIC, 0, 0, 0, None), (P.NIDX_P_GROUP, 0, 300, 400, None),
                (P.NIDX_P_GROUP, 0, 17, 18, None), (P.NIDX_P_GROUP, 0, 905, 906, None)]
    shapes = {"security": security, "security_and_facet": [(P.NIDX_P_AND, 2, 0, 0, None)] + security + [(P.NIDX_P_FACET, 0, 8, 16, None)]}
    words = (n + 63) // 64
    bits = torch.empty(words, dtype=torch.int64, device=dev)
    out = {"docs": n, "gpu": torch.cuda.get_device_name(0), "groups": N_GROUPS, "group_ords": int(goff[-1])}
    for name, spec in shapes.items():
        nodes, _keep = node_array(spec)
        for _ in range(a.warmup):
            ts.prefilter(nodes, out=bits)
        k_ms = []
        for _ in range(a.steps):
            _, matching = ts.prefilter(nodes, out=bits)
            k_ms.append(ts.last_kernel_ms())
        out[name] = dict(kernel_ms=round(float(np.median(k_ms)), 4), matching=int(matching))
    nodes, _keep = node_array(security)
    _, matching = ts.prefilter(nodes, out=bits)   # the mask of the BM25 comparison
    ones = torch.full((words,), -1, dtype=torch.int64, device=dev)
    rng_q = np.random.default_rng(11)
    band = np.nonzero((df >= 1_000) & (df <= 100_000))[0]
    for nq in (1, 1024):
        queries = [rng_q.choice(band, 50, replace=False).astype(np.uint32) for _ in range(nq)]
        qo = torch.tensor(np.concatenate([[0], np.cumsum([len(x) for x in queries])]), dtype=torch.int32, device=dev)
        qt = torch.tensor(np.concatenate(queries).astype(np.int64), dtype=torch.int32, device=dev)

        def plain():
            return ts.search(qt, qo, 100, mode=_lib.NIDX_BM25_OR, use_tf=False)

        def masked(mask=bits):
            v = ts.view(mask)
            r = v.search(qt, qo, 100, mode=_lib.NIDX_BM25_OR, use_tf=False)
            v.close()
            return r

        same = all(torch.equal(x, y) for x, y in zip(plain(), masked(ones)))
        for _ in range(a.warmup):
            plain(); masked()
        torch.cuda.synchronize()
        t_plain, t_masked = [], []
        for _ in range(a.steps):
            for f, acc in ((plain, t_plain), (masked, t_masked)):
                t0 = time.perf_counter()
                r = f()
                torch.cuda.synchronize()
                acc.append((time.perf_counter() - t0) * 1e3)
        out[f"or50_top100_nq{nq}"] = dict(unmasked_ms=round(float(np.median(t_plain)), 3), masked_ms=round(float(np.median(t_masked)), 3),
                                          spread_unmasked_ms=round(float(np.std(t_plain)), 3), spread_masked_ms=round(float(np.std(t_masked)), 3),
                                          masked_total_q0=int(r[3][0]), mask_matching=int(matching), all_ones_mask_identical=bool(same))
    out["labels_per_doc"] = LABELS_PER_DOC
    try:
        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        out["power_limit"] = "unknown"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
