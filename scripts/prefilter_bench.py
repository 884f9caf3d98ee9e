"""The prefilter on one text segment of bench_extra's BM25 corpus shape (Zipf(1.07) vocabulary, lognormal lengths of mean 64, every
token's position kept), with resources, fields, labels and dates added: prefilter_eval_kernel's time per expression shape, its byte
model over that time as a share of the HBM peak, the whole nidx_txt_prefilter call, the hand-off to a vector segment
(nidx_vec_prefilter_bits), and the host loop the device prefilter replaced (binding._doc_matches) on the same documents.

One JSON line; kernel times from CUDA events around the pass after warm-up, the card's name and power limit read in the same process.

    python scripts/prefilter_bench.py [--docs 5000000] [--steps 20] [--warmup 3] [--loop-docs 5000000]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s
N_FIELDS, N_LABELS, LABELS_PER_DOC = 8, 64, 3


def columns(n, seed=3):
    rng = np.random.default_rng(seed)
    res = (np.arange(n) // 3).astype(np.uint32)                           # three fields per resource
    fld = rng.integers(0, N_FIELDS, n).astype(np.uint32)
    ords = np.sort(rng.integers(0, N_LABELS, (n, LABELS_PER_DOC)), axis=1)
    keep = np.ones_like(ords, dtype=bool)
    keep[:, 1:] = ords[:, 1:] != ords[:, :-1]                               # strictly ascending per document
    off = np.zeros(n + 1, dtype=np.uint64)
    off[1:] = np.cumsum(keep.sum(1))
    created = rng.integers(1_500_000_000, 1_700_000_000, n).astype(np.int64)
    created[rng.random(n) < 0.05] = np.iinfo(np.int64).min                  # undated
    return res, fld, off, ords[keep].astype(np.uint32), created


def node_array(spec):
    from nucliadb_b200 import _lib

    nodes = (_lib.PrefilterNode * len(spec))()
    keep = []
    for i, (kind, n, lo, hi, terms) in enumerate(spec):
        nodes[i].kind, nodes[i].n, nodes[i].lo, nodes[i].hi = kind, n, lo, hi
        if terms is not None:
            t = np.asarray(terms, dtype=np.uint32)
            keep.append(t)
            nodes[i].terms = t.ctypes.data
    return nodes, keep


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=5_000_000)
    ap.add_argument("--terms", type=int, default=1 << 20)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--loop-docs", type=int, default=5_000_000)
    a = ap.parse_args()
    import torch

    from phrase_bench import make_positional_corpus

    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import TextSegment, VectorSegment

    _lib.require_device()
    dev = torch.device("cuda", 0)
    n = a.docs
    c = make_positional_corpus(n, a.terms, dev)
    fn = np.minimum(c["lens"], 255).astype(np.uint8)   # the fieldnorm code does not matter to the prefilter
    ts = TextSegment.create(n, a.terms, c["term_off"], c["post_doc"], c["post_tf"], fn)
    ts.set_positions(c["positions"])
    res, fld, off, ords, created = columns(n)
    ts.set_doc_columns(res, fld)
    ts.set_facets([b"l\0%03d" % i for i in range(N_LABELS)], off, ords)
    ts.set_dates(created, created + 86_400)
    # a phrase cut from a real document: its first two tokens
    d0 = int(np.argmax(c["lens"] >= 2))
    phrase = [int(c["tokens"][c["doc_start"][d0]]), int(c["tokens"][c["doc_start"][d0] + 1])]
    P = _lib
    mid = 1_600_000_000
    shapes = {
        "facet": ([(P.NIDX_P_FACET, 0, 8, 16, None)], 4 + 4 * LABELS_PER_DOC),
        "field_and_date": ([(P.NIDX_P_AND, 2, 0, 0, None), (P.NIDX_P_FIELD, 0, 2, 4, None), (P.NIDX_P_DATE, 0, mid, mid + 30 * 86_400, None)], 4 + 8),
        "not_facet": ([(P.NIDX_P_NOT, 1, 0, 0, None), (P.NIDX_P_FACET, 0, 8, 16, None)], 4 + 4 * LABELS_PER_DOC),
        "keyword_phrase": ([(P.NIDX_P_KEYWORD, 2, 0, 0, phrase)], 1 / 8),   # the pass reads the leaf's bits; the phrase pass before it is not in kernel_ms
    }
    words = (n + 63) // 64
    bits = torch.empty(words, dtype=torch.int64, device=dev)
    out = {"docs": n, "gpu": torch.cuda.get_device_name(0)}
    for name, (spec, per_doc) in shapes.items():
        nodes, _keep = node_array(spec)
        for _ in range(a.warmup):
            ts.prefilter(nodes, out=bits)
        k_ms, call_ms = [], []
        for _ in range(a.steps):
            t0 = time.perf_counter()
            _, matching = ts.prefilter(nodes, out=bits)   # returns when the bits and the count are in place
            call_ms.append((time.perf_counter() - t0) * 1e3)
            k_ms.append(ts.last_kernel_ms())
        k = float(np.median(k_ms))
        model_bytes = n * per_doc + n / 8   # the columns the program reads + the output bits (no alive set here)
        out[name] = dict(kernel_ms=round(k, 4), call_ms=round(float(np.median(call_ms)), 3), matching=int(matching), bytes=int(model_bytes),
                         gbps=round(model_bytes / (k * 1e-3) / 1e9, 1), share_of_hbm_peak=round(model_bytes / (k * 1e-3) / HBM_PEAK, 3))
    # the hand-off: 1 M field keys of 2 paragraphs each in a vector segment, the documents joined to them
    n_keys, dim = 1_000_000, 8
    vs = VectorSegment.create(np.random.default_rng(1).standard_normal((2 * n_keys, dim)).astype(np.float32), dim, similarity=_lib.NIDX_SIM_DOT)
    keys = [b"%016d" % i for i in range(n_keys)]
    key_bytes = np.frombuffer(b"".join(keys), dtype=np.uint8)
    key_off = np.arange(0, 16 * (n_keys + 1), 16, dtype=np.uint64)
    post_off = np.arange(0, 2 * (n_keys + 1), 2, dtype=np.uint64)
    check = _lib.check
    check(_lib.load().nidx_vec_set_inverted_index(vs._h, _lib.NIDX_INV_FIELDS, n_keys, _lib.ptr(key_bytes), _lib.ptr(key_off), _lib.ptr(post_off),
                                                  _lib.ptr(np.arange(2 * n_keys, dtype=np.uint32))))
    join = torch.from_numpy((np.arange(n) % n_keys).astype(np.uint32).view(np.int32)).to(dev)
    nodes, _keep = node_array(shapes["facet"][0])
    _, doc_matching = ts.prefilter(nodes, out=bits)
    for _ in range(a.warmup):
        vs.prefilter_bits(bits, join, n, None, None, 0, 2 * n_keys)
    j_ms = []
    for _ in range(a.steps):
        t0 = time.perf_counter()
        _, par_matching = vs.prefilter_bits(bits, join, n, None, None, 0, 2 * n_keys)
        j_ms.append((time.perf_counter() - t0) * 1e3)
    out["join"] = dict(call_ms=round(float(np.median(j_ms)), 3), docs_matched=int(doc_matching), paragraphs_matched=int(par_matching))
    # the host loop it replaced, on the same documents (facet AND field), as the binding ran it
    from nucliadb_b200 import nidx_protos as PB
    from nucliadb_b200.binding import _doc_matches
    from nucliadb_b200.text import TextDoc

    m = min(a.loop_docs, n)
    fields = [f"/a/f{i}" for i in range(N_FIELDS)]
    docs = [TextDoc("%032x" % int(res[d]), fields[fld[d]], "", tuple("/l/%03d" % o for o in ords[off[d]:off[d + 1]])) for d in range(m)]
    e = PB.FilterExpression()
    e.bool_and.operands.add().facet.facet = "/l/008"
    e.bool_and.operands.add().field.field_type = "a"
    t0 = time.perf_counter()
    hits = sum(1 for d in docs if _doc_matches(e, d))
    out["python_loop"] = dict(docs=m, seconds=round(time.perf_counter() - t0, 3), matched=hits)
    try:
        import subprocess

        out["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    except OSError:
        out["power_limit"] = "unknown"
    print(json.dumps(out))


if __name__ == "__main__":
    main()
