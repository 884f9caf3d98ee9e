#!/usr/bin/env python
"""bench_extra.py — the other BASELINE.json configs, one JSON line each (same keys as bench.py):

  scan   configs[0]: nidx_vector brute-force cosine top-10, 100k x 384 f32, 1k queries (segment.rs:569-623)
  bm25   configs[3]: BM25 5M docs / 50-term queries, top-100, postings in HBM
         - "or_basic": nidx_paragraph semantics (OR of TermQuery(Basic), tf == 1)
         - "and_tf":   nidx_text semantics (conjunction, real tf) on 3-term queries
  facets the bm25 corpus + seeded labels: OR-50 top-100 with / without faceted=["/l"], and the all-documents facet count
  order  the bm25 corpus + seeded created / modified seconds: OR-50 top-100 and AND-3 ordered by date against the same searches by
         score, ordered + faceted=["/l"], and the catalogue listing (empty body, top-100 by date over every alive document)

bench.py (the driver's contract) stays the HNSW headline; this file produces the side measurements.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import effective_cores  # noqa: E402


def peaks():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        return {}


def ncu_traffic(workload):
    """DRAM bytes per launch of an ncu capture of this exact workload (profiles/ncu_traffic.json, when one is kept), or None."""
    try:
        return json.load(open(os.path.join(ROOT, "profiles", "ncu_traffic.json"))).get(workload, {}).get("dram_bytes_per_launch")
    except Exception:
        return None


def timed(fn, steps, warmup):
    import torch

    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def bench_scan(args):
    import torch

    import oracle as O
    from bench import gen_queries, gen_vectors
    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import VectorSegment

    dev = torch.device("cuda", 0)
    n, d, nq, k = 100_000, 384, 1000, 10
    vecs = gen_vectors(n, d, dev, seed=1234567890, latent=16, noise=0.15)
    q = gen_queries(vecs, nq, seed=123)
    host_v, host_q = vecs.cpu().numpy(), q.cpu().numpy()
    seg = VectorSegment.create(vecs, d, similarity=_lib.NIDX_SIM_COSINE)
    out = (torch.empty((nq, k), dtype=torch.int32, device=dev), torch.empty((nq, k), dtype=torch.float32, device=dev), torch.empty((nq,), dtype=torch.int32, device=dev))
    lines = []
    for label, qq in (("batch of 1000 queries", q), ("single query", q[:1].contiguous())):
        o = tuple(t[: qq.shape[0]] for t in out)
        ms = timed(lambda: seg.search(qq, k, method=_lib.NIDX_METHOD_BRUTE, out=o), args.steps, args.warmup)
        kms = seg.last_kernel_ms()
        passes = (qq.shape[0] + 7) // 8                     # every 8-query tile re-reads the vector block (L2 absorbs most of it)
        alg = n * d * 4                                        # algorithmic bytes: the block once per launch
        ids = o[0].cpu().numpy().astype(np.uint32)
        sc = o[1].cpu().numpy()
        oi, os_, _ = O.brute_force(host_v, host_q[: qq.shape[0]], k, nthreads=effective_cores())
        t0 = time.perf_counter()
        O.brute_force(host_v, host_q[: min(qq.shape[0], 256)], k, nthreads=effective_cores())
        cpu_dt = time.perf_counter() - t0
        pk = float(peaks().get("hbm_gbs", 3350.0))
        ach = alg / (kms * 1e-3) / 1e9
        wl = f"nidx_vector brute-force cosine top-10, {n}x{d} f32, {label}"
        if qq.shape[0] >= 128:   # tensor-core filter: ONE TF32 pass over Q x N (2 N d Q flops); TF32 dense peak = half the measured bf16 peak
            tf = 2.0 * n * d * qq.shape[0] / (kms * 1e-3) / 1e12
            tpk = float(peaks().get("bf16_tflops", 989.0)) / 2
            roof = {"bound": "tensor", "achieved": tf, "peak": tpk, "unit": "TFLOP/s", "frac": tf / tpk, "kernel": "scan_tc_filter_kernel", "kernel_ms": kms,
                    "traffic": ncu_traffic(wl), "note": "2 N d Q flops of the single TF32 pass / the filter kernel's time; peak = MEASURED_PEAKS bf16_tflops / 2 "
                    "(TF32 runs at half the bf16 rate); the exact refine of the survivors is in ms_per_step, not here"}
        else:
            roof = {"bound": "hbm", "achieved": ach, "peak": pk, "unit": "GB/s", "frac": ach / pk, "kernel": "scan_scores_kernel_t", "kernel_ms": kms, "traffic": ncu_traffic(wl)}
        lines.append({"metric": "exact k-NN QPS (brute force)", "value": qq.shape[0] / (ms * 1e-3), "unit": "queries/s", "n_gpus": 1, "steps": args.steps,
                      "warmup": args.warmup, "ms_per_step": ms, "higher_is_better": True, "dtype": "f32", "data": "synthetic",
                      "config": {"workload": wl, "passes_over_block": passes},
                      "parity": {"ids_identical_to_oracle": bool((ids == oi).all()), "max_abs_score_diff": float(np.abs(sc - os_).max())},
                      "roofline": roof,
                      "cpu_baseline": {"value": min(qq.shape[0], 256) / cpu_dt, "unit": "queries/s", "cores": effective_cores(), "kind": "port",
                                       "sample": f"{min(qq.shape[0], 256)} queries"}})
    return lines


def bench_build(args):
    """configs[2]: HNSW index build (per 1M x 768 here; bench.py reports the 10M build of the headline run) at the
    BASELINE constants (M=16, efC=200) and at the reference's compile-time constants (M=30/60, efC=100)."""
    import torch

    from bench import gen_queries, gen_vectors, recall_at_k
    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import VectorSegment

    dev = torch.device("cuda", 0)
    n, d = args.build_vectors, 768
    vecs = gen_vectors(n, d, dev, seed=1234567890, latent=16, noise=0.15)
    q = gen_queries(vecs, 1024, seed=123)
    lines = []
    for m, m0, efc in ((16, 32, 200), (30, 60, 100)):
        seg = VectorSegment.create(vecs, d, similarity=_lib.NIDX_SIM_COSINE, m=m, m0=m0, ef_construction=efc)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        seg.build_hnsw(seed=2, max_batch=8192)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        c = seg.counters()
        gt = seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)[0].cpu().numpy()
        rec = {ef: recall_at_k(seg.search(q, 10, ef=ef, method=_lib.NIDX_METHOD_HNSW)[0].cpu().numpy(), gt) for ef in (30, 128)}
        alg = c["similarities"] * (d * 4 + 4)
        pk = float(peaks().get("hbm_gbs", 3350.0))
        lines.append({"metric": "HNSW build vectors/s", "value": n / dt, "unit": "vectors/s", "n_gpus": 1, "higher_is_better": True, "dtype": "f32", "data": "synthetic",
                      "config": {"workload": f"HNSW index build {n}x{d}, M={m} M0={m0} efC={efc}", "max_batch": 8192}, "seconds": dt,
                      "similarities": c["similarities"], "visited_overflows": c["overflows"], "recall_at_10": rec,
                      "roofline": {"bound": "hbm", "achieved": alg / dt / 1e9, "peak": pk, "unit": "GB/s", "frac": alg / dt / 1e9 / pk,
                                   "note": "whole build (search + select + reverse-link + sort) over the search kernel's algorithmic bytes"}})
        seg.close()
    return lines


def bench_merge(args):
    """merge_indexes (segment.rs:143-167): a segment of --build-vectors vectors without deletions plus 10% new vectors.  The
    graph of the large segment is reused and only the new vectors are inserted; timed beside the full rebuild."""
    import torch

    from bench import gen_queries, gen_vectors, recall_at_k
    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import VectorSegment

    dev = torch.device("cuda", 0)
    n0, d = args.build_vectors, 768
    n = n0 + n0 // 10
    vecs = gen_vectors(n, d, dev, seed=1234567890, latent=16, noise=0.15)
    q = gen_queries(vecs, 1024, seed=123)
    kw = dict(similarity=_lib.NIDX_SIM_COSINE, m=16, m0=32, ef_construction=200)
    first = VectorSegment.create(vecs[:n0].contiguous(), d, **kw)
    first.build_hnsw(seed=2, max_batch=8192)
    g = first.get_graph()
    first.close()
    rows = max(int(g["upper_rows"]), 1)
    out = {}
    for name in ("reuse", "rebuild"):
        seg = VectorSegment.create(vecs, d, **kw)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        if name == "reuse":
            seg.extend_hnsw(n0, g["level"], g["adj0"], g["adjU"][:rows], g["w0"], g["wU"][:rows], g["entry_node"], g["entry_layer"], seed=2, max_batch=8192)
        else:
            seg.build_hnsw(seed=2, max_batch=8192)
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        gt = seg.search(q, 10, method=_lib.NIDX_METHOD_BRUTE)[0].cpu().numpy()
        out[name] = {"seconds": dt, "recall_at_10_ef128": recall_at_k(seg.search(q, 10, ef=128, method=_lib.NIDX_METHOD_HNSW)[0].cpu().numpy(), gt)}
        seg.close()
    return [{"metric": "merge inserted vectors/s", "value": (n - n0) / out["reuse"]["seconds"], "unit": "vectors/s", "n_gpus": 1, "higher_is_better": True,
             "dtype": "f32", "data": "synthetic", "config": {"workload": f"merge {n0}x{d} (graph reused) + {n - n0} new, M=16 M0=32 efC=200", "max_batch": 8192},
             "reuse": out["reuse"], "rebuild": out["rebuild"], "note": "reuse time includes the host->device copy of the existing graph"}]


def make_corpus(n_docs, n_terms, dev, seed=7, mean_len=64, zipf_s=1.07):
    """5M docs, vocabulary 1M Zipf(1.07), doc length lognormal (mean 64) — BASELINE.md row 4.  Built on the GPU with torch
    (sorting 3e8 tokens on the host takes minutes); returned as host CSR arrays."""
    import torch

    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    sigma = 0.5
    lens = torch.exp(torch.randn(n_docs, generator=g, device=dev) * sigma + (np.log(mean_len) - sigma * sigma / 2)).clamp_(min=1).to(torch.int64)
    total = int(lens.sum().item())
    ranks = torch.arange(1, n_terms + 1, device=dev, dtype=torch.float64)
    cdf = torch.cumsum(ranks.pow(-zipf_s), 0)
    cdf /= cdf[-1].clone()
    doc_of = torch.repeat_interleave(torch.arange(n_docs, device=dev, dtype=torch.int64), lens)
    keys = torch.empty(total, dtype=torch.int64, device=dev)
    chunk = 50_000_000
    for i in range(0, total, chunk):
        m = min(chunk, total - i)
        u = torch.rand(m, generator=g, device=dev, dtype=torch.float64)
        term = torch.searchsorted(cdf, u).clamp_(max=n_terms - 1)
        keys[i:i + m] = term * n_docs + doc_of[i:i + m]
    del doc_of
    uniq, tf = torch.unique(keys, return_counts=True)   # sorted by (term, doc)
    del keys
    term = torch.div(uniq, n_docs, rounding_mode="floor")
    doc = (uniq - term * n_docs).to(torch.int32)
    term_off = torch.zeros(n_terms + 1, dtype=torch.int64, device=dev)
    term_off[1:] = torch.cumsum(torch.bincount(term, minlength=n_terms), 0)
    return dict(lens=lens.cpu().numpy(), total_tokens=total, term_off=term_off.cpu().numpy().astype(np.uint64), post_doc=doc.cpu().numpy().astype(np.uint32),
                post_tf=tf.to(torch.int32).cpu().numpy().astype(np.uint32))


def bench_bm25(args):
    import torch

    import oracle as O
    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import TextSegment
    from nucliadb_b200.text import fieldnorm_to_id

    dev = torch.device("cuda", 0)
    n_docs, n_terms, nq, k = args.docs, 1_000_000, 1024, 100
    t0 = time.perf_counter()
    c = make_corpus(n_docs, n_terms, dev)
    lut = np.asarray([fieldnorm_to_id(i) for i in range(int(c["lens"].max()) + 1)], dtype=np.uint8)
    fieldnorm = lut[c["lens"]]
    df = np.diff(c["term_off"].astype(np.int64)).astype(np.uint64)
    ts = TextSegment.create(n_docs, n_terms, c["term_off"], c["post_doc"], c["post_tf"], fieldnorm)
    ts.set_stats(n_docs, c["total_tokens"], df)
    t_setup = time.perf_counter() - t0
    rng = np.random.default_rng(11)
    band = np.nonzero((df >= 1_000) & (df <= 100_000))[0]
    lines = []

    class P:  # the oracle's view of the same segment
        pass

    P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id, P.doc_freq, P.total_tokens = (
        n_docs, n_terms, c["term_off"], c["post_doc"], c["post_tf"], fieldnorm, df, c["total_tokens"])
    for name, nterms, mode, use_tf in (("or_basic", 50, _lib.NIDX_BM25_OR, False), ("and_tf", 3, _lib.NIDX_BM25_AND, True)):
        queries = [rng.choice(band, nterms, replace=False).astype(np.uint32) for _ in range(nq)]
        qoff = torch.tensor(np.concatenate([[0], np.cumsum([len(x) for x in queries])]), dtype=torch.int32, device=dev)
        qt = torch.tensor(np.concatenate(queries).astype(np.int64), dtype=torch.int32, device=dev)
        out = (torch.empty((nq, k), dtype=torch.int32, device=dev), torch.empty((nq, k), dtype=torch.float32, device=dev),
               torch.empty((nq,), dtype=torch.int32, device=dev), torch.empty((nq,), dtype=torch.int64, device=dev))
        ms = timed(lambda: ts.search(qt, qoff, k, mode=mode, use_tf=use_tf, out=out), args.steps, args.warmup)
        kms = ts.last_kernel_ms()
        postings = sum(int(df[t]) for q in queries for t in q)
        alg = postings * ((8 if use_tf else 4) + 1)
        # host path (e2e): numpy in / numpy out through the C ABI
        qt_h, qo_h = np.concatenate(queries), np.concatenate([[0], np.cumsum([len(x) for x in queries])]).astype(np.uint32)
        ts.search(qt_h, qo_h, k, mode=mode, use_tf=use_tf)
        t0 = time.perf_counter()
        for _ in range(args.steps):
            docs, sc, cnt, tot = ts.search(qt_h, qo_h, k, mode=mode, use_tf=use_tf)
        e2e = nq * args.steps / (time.perf_counter() - t0)
        # oracle on a bounded sample (every thread's scratch is allocated by an untimed warm-up call first)
        ns = min(nq, 1024)
        O.bm25_search(P, [list(x) for x in queries[: 4 * effective_cores()]], k, mode=mode, use_tf=use_tf, nthreads=effective_cores())
        t0 = time.perf_counter()
        od, osc, oc, otot = O.bm25_search(P, [list(x) for x in queries[:ns]], k, mode=mode, use_tf=use_tf, nthreads=effective_cores())
        cpu_dt = time.perf_counter() - t0
        ok_counts = bool((cnt[:ns] == oc).all() and (tot[:ns] == otot).all())
        rel = float(np.max(np.abs(sc[:ns] - osc) / np.maximum(1.0, np.abs(osc))))
        same_ids = float(np.mean(docs[:ns] == od))
        pk = float(peaks().get("hbm_gbs", 3350.0))
        ach = alg / (kms * 1e-3) / 1e9
        lines.append({"metric": "BM25 QPS", "value": nq / (ms * 1e-3), "unit": "queries/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                      "ms_per_step": ms, "higher_is_better": True, "dtype": "f32 (u32 fixed-point accumulate)", "data": "synthetic",
                      "config": {"workload": f"BM25 {n_docs} docs / {nterms}-term queries, top-{k}, {name}", "vocab": n_terms, "postings": int(c['term_off'][-1]),
                                 "postings_per_query": postings / nq, "setup_seconds": t_setup},
                      "parity": {"counts_identical_to_oracle": ok_counts, "max_rel_score_diff": rel, "ids_identical_fraction": same_ids, "sample": ns},
                      "roofline": {"bound": "hbm", "achieved": ach, "peak": pk, "unit": "GB/s", "frac": ach / pk, "kernel": "bm25_kernel", "kernel_ms": kms,
                                   "traffic": ncu_traffic(f"BM25 {n_docs} docs / {nterms}-term queries, top-{k}, {name}"),
                                   "parity_note": "BM25 parity is UNPINNED: the oracle restates tantivy 0.26's published formula, tantivy itself is not in the tree",
                                   "alg_bytes_note": "postings x (8 with tf, 4 + 1 for tf == 1: SURVEY 8d); the records read are 8 B either way"},
                      "cpu_baseline": {"value": ns / cpu_dt, "unit": "queries/s", "cores": effective_cores(), "kind": "port", "sample": f"{ns} queries"},
                      "e2e": {"value": e2e, "unit": "queries/s", "h2d_bytes_per_step": int(qt_h.nbytes + qo_h.nbytes), "d2h_bytes_per_step": nq * k * 8 + nq * 12}})
    return lines


def gpu_identity():
    """The card's name and power limit, read in the same process as the measurement (a number is only worth something with them)."""
    import subprocess

    import torch

    out = {"name": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"], capture_output=True, text=True, timeout=30)
        out["power_limit_and_max_sm_clock"] = q.stdout.strip()
    except Exception as e:  # noqa: BLE001
        out["power_limit_and_max_sm_clock"] = f"unavailable: {e}"
    return out


def bench_facets(args):
    """tantivy's FacetCollector on the BM25 corpus of `bm25` plus seeded labels: /l/s{00..99}/x{00..99} (a three-level hierarchy of
    10 k leaf labels), 1..4 labels per document, Zipf over the leaves.  Reports OR-50 top-100 with and without faceted=["/l"] (the
    same call, alternating), the all-documents count (empty body / only_faceted catalogue) against the HBM peak and the CPU
    restatement (tests/facet_oracle.py, numpy, one process), and exact parity with it on a sample."""
    import torch

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import facet_oracle as FO
    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import TextSegment
    from nucliadb_b200.text import fieldnorm_to_id

    dev = torch.device("cuda", 0)
    n_docs, n_terms, nq, k = args.docs, 1_000_000, 1024, 100
    c = make_corpus(n_docs, n_terms, dev)
    lut = np.asarray([fieldnorm_to_id(i) for i in range(int(c["lens"].max()) + 1)], dtype=np.uint8)
    df = np.diff(c["term_off"].astype(np.int64)).astype(np.uint64)
    ts = TextSegment.create(n_docs, n_terms, c["term_off"], c["post_doc"], c["post_tf"], lut[c["lens"]])
    ts.set_stats(n_docs, c["total_tokens"], df)
    # labels
    rng = np.random.default_rng(12)
    keys = sorted(f"l\0s{a:02d}\0x{b:02d}".encode() for a in range(100) for b in range(100))
    zipf = 1.0 / np.arange(1, len(keys) + 1) ** 1.0
    perm = rng.permutation(len(keys))   # popularity does not follow the key order
    n_lab = rng.integers(1, 5, n_docs)
    doc = np.repeat(np.arange(n_docs, dtype=np.int64), n_lab)
    leaf = perm[np.searchsorted(np.cumsum(zipf / zipf.sum()), rng.random(len(doc))).clip(max=len(keys) - 1)]
    pairs = np.unique(doc * len(keys) + leaf)
    ords = (pairs % len(keys)).astype(np.uint32)
    doc_off = np.zeros(n_docs + 1, dtype=np.uint64)
    doc_off[1:] = np.cumsum(np.bincount(pairs // len(keys), minlength=n_docs))
    ts.set_facets(keys, doc_off, ords)
    alive_b = rng.random(n_docs) >= 0.01
    alive = np.packbits(alive_b, bitorder="little")
    alive = np.concatenate([alive, np.zeros(-len(alive) % 8, np.uint8)]).view(np.uint64)
    ts.set_alive(alive)
    request = [b"l"]
    # OR-50 top-100, with and without the facets, alternating
    rng_q = np.random.default_rng(11)
    band = np.nonzero((df >= 1_000) & (df <= 100_000))[0]
    queries = [rng_q.choice(band, 50, replace=False).astype(np.uint32) for _ in range(nq)]
    qoff = torch.tensor(np.concatenate([[0], np.cumsum([len(x) for x in queries])]), dtype=torch.int32, device=dev)
    qt = torch.tensor(np.concatenate(queries).astype(np.int64), dtype=torch.int32, device=dev)
    out = (torch.empty((nq, k), dtype=torch.int32, device=dev), torch.empty((nq, k), dtype=torch.float32, device=dev),
           torch.empty((nq,), dtype=torch.int32, device=dev), torch.empty((nq,), dtype=torch.int64, device=dev))
    plain_fn = lambda: ts.search(qt, qoff, k, mode=_lib.NIDX_BM25_OR, use_tf=False, out=out)
    facet_fn = lambda: ts.search_faceted(qt, qoff, k, request, mode=_lib.NIDX_BM25_OR, use_tf=False)
    plain_ms, facet_ms, plain_kms, facet_kms = [], [], [], []
    for _ in range(5):
        plain_ms.append(timed(plain_fn, args.steps, args.warmup)); plain_kms.append(ts.last_kernel_ms())
        facet_ms.append(timed(facet_fn, args.steps, args.warmup)); facet_kms.append(ts.last_kernel_ms())
    med = lambda x: float(np.median(x))
    # parity on a sample: top-k / Count bit for bit against the search without facets, counts against the restatement
    fd, fs, fc, ft, fcnt = facet_fn()
    plain_fn()
    torch.cuda.synchronize()
    same_search = all(torch.equal(a, b) for a, b in zip(out, (fd, fs, fc, ft)))
    bucket, b_req, _ = FO.plan(keys, request)
    sample = 8
    got = fcnt[:sample].cpu().numpy().astype(np.int64)
    want = np.stack([FO.count(doc_off, ords, bucket, len(b_req), FO.matched(n_docs, c["term_off"], c["post_doc"], q.tolist(), False, alive)) for q in queries[:sample]])
    # all documents
    all_fn = lambda: ts.facet_count_all(request, device_out=True)
    all_ms = timed(all_fn, args.steps, args.warmup)
    all_kms = ts.last_kernel_ms()
    dev_all = all_fn().cpu().numpy().astype(np.int64)
    t0 = time.perf_counter()
    cpu_all = FO.count(doc_off, ords, bucket, len(b_req), alive_b)
    cpu_s = time.perf_counter() - t0
    nbytes = 4 * (n_docs + 1) + 4 * len(ords) + 8 * len(alive)
    pk = float(peaks().get("hbm_gbs", 3350.0))
    ach = nbytes / (all_kms * 1e-3) / 1e9
    return [{"metric": "facet overhead (OR-50 top-100, faceted=[\"/l\"])", "value": med(facet_ms) / med(plain_ms), "unit": "x (faceted / plain call)", "n_gpus": 1,
             "steps": args.steps, "warmup": args.warmup, "gpu": gpu_identity(), "higher_is_better": False, "data": "synthetic",
             "config": {"workload": f"BM25 {n_docs} docs / 50-term OR queries x {nq}, top-{k}, tf == 1", "facet_keys": len(keys), "facet_ords": int(len(ords)),
                        "buckets": int(len(b_req)), "rounds": 5},
             "plain": {"ms_per_call": med(plain_ms), "kernel_ms": med(plain_kms), "kernel": "bm25_kernel"},
             "faceted": {"ms_per_call": med(facet_ms), "kernel_ms": med(facet_kms), "kernel": "bm25_facet_kernel"},
             "kernel_ratio": med(facet_kms) / med(plain_kms),
             "parity": {"search_identical_to_plain": bool(same_search), "counts_identical_to_oracle": bool(np.array_equal(got, want)), "sample": sample}},
            {"metric": "facet count, all documents", "value": all_ms, "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "gpu": gpu_identity(),
             "higher_is_better": False, "data": "synthetic",
             "config": {"workload": f"FacetCollector over {n_docs} alive-masked documents, faceted=[\"/l\"]", "facet_ords": int(len(ords)), "buckets": int(len(b_req))},
             "roofline": {"bound": "hbm", "achieved": ach, "peak": pk, "unit": "GB/s", "frac": ach / pk, "kernel": "facet_count_all_kernel", "kernel_ms": all_kms,
                          "alg_bytes": nbytes, "alg_bytes_note": "doc_off (4 B per document) + ords (4 B each) + alive bits, each read once"},
             "parity": {"counts_identical_to_oracle": bool(np.array_equal(dev_all, cpu_all))},
             "cpu_baseline": {"value": cpu_s * 1e3, "unit": "ms", "cores": 1, "kind": "numpy restatement (tests/facet_oracle.py), one process"}}]


def bench_order(args):
    """TopDocs::order_by_fast_field on the BM25 corpus of `bm25` with seeded dates: created spread over ten years at minute
    granularity with 10 % of the documents on 20 shared dates (heavy ties) and 1 % undated, modified a month at most later, 1 % of
    the documents deleted, 100 labels /l/s{00..99}.  Runs and its unordered twin alternate within one call; the listing's bytes are
    the algorithmic ones (rank column 4 B + alive bit per document, plus the top-k out); parity with tests/order_oracle.py on a sample."""
    import torch

    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import order_oracle as OO
    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import TextSegment
    from nucliadb_b200.text import fieldnorm_to_id

    dev = torch.device("cuda", 0)
    n_docs, n_terms, nq, k = args.docs, 1_000_000, 1024, 100
    c = make_corpus(n_docs, n_terms, dev)
    lut = np.asarray([fieldnorm_to_id(i) for i in range(int(c["lens"].max()) + 1)], dtype=np.uint8)
    df = np.diff(c["term_off"].astype(np.int64)).astype(np.uint64)
    ts = TextSegment.create(n_docs, n_terms, c["term_off"], c["post_doc"], c["post_tf"], lut[c["lens"]])
    ts.set_stats(n_docs, c["total_tokens"], df)
    rng = np.random.default_rng(13)
    keys = sorted(f"l\0s{a:02d}".encode() for a in range(100))
    ords = rng.integers(0, len(keys), n_docs).astype(np.uint32)
    ts.set_facets(keys, np.arange(n_docs + 1, dtype=np.uint64), ords)
    created = (1_450_000_000 + rng.integers(0, 10 * 365 * 1440, n_docs) * 60).astype(np.int64)
    tie = rng.random(n_docs) < 0.10
    created[tie] = 1_600_000_000 + rng.integers(0, 20, int(tie.sum())) * 86_400
    created[rng.random(n_docs) < 0.01] = OO.NONE
    modified = np.where(created == OO.NONE, OO.NONE, created + rng.integers(0, 30 * 86_400, n_docs)).astype(np.int64)
    t0 = time.perf_counter()
    ts.set_dates(created, modified)
    t_dates = time.perf_counter() - t0
    alive_b = rng.random(n_docs) >= 0.01
    alive = np.packbits(alive_b, bitorder="little")
    alive = np.concatenate([alive, np.zeros(-len(alive) % 8, np.uint8)]).view(np.uint64)
    ts.set_alive(alive)
    rng_q = np.random.default_rng(11)
    band = np.nonzero((df >= 1_000) & (df <= 100_000))[0]
    med = lambda x: float(np.median(x))
    gpu = gpu_identity()
    lines = []
    for name, nterms, mode, use_tf in (("OR-50", 50, _lib.NIDX_BM25_OR, False), ("AND-3", 3, _lib.NIDX_BM25_AND, True)):
        queries = [rng_q.choice(band, nterms, replace=False).astype(np.uint32) for _ in range(nq)]
        qoff = torch.tensor(np.concatenate([[0], np.cumsum([len(x) for x in queries])]), dtype=torch.int32, device=dev)
        qt = torch.tensor(np.concatenate(queries).astype(np.int64), dtype=torch.int32, device=dev)
        runs = {"by score": lambda: ts.search(qt, qoff, k, mode=mode, use_tf=use_tf),
                "by date": lambda: ts.search_ordered(qt, qoff, k, _lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_DESC, mode)}
        if name == "OR-50":
            runs["by score + faceted"] = lambda: ts.search_faceted(qt, qoff, k, [b"l"], mode=mode, use_tf=use_tf)
            runs["by date + faceted"] = lambda: ts.search_ordered(qt, qoff, k, _lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_DESC, mode, facets=[b"l"])
        ms, kms = {r: [] for r in runs}, {r: [] for r in runs}
        for _ in range(5):
            for r, fn in runs.items():
                ms[r].append(timed(fn, args.steps, args.warmup)); kms[r].append(ts.last_kernel_ms())
        # parity on a sample: ids, dates, counts, totals against the restatement; total against the search by score
        got = ts.search_ordered(qt, qoff, k, _lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_DESC, mode)
        plain = ts.search(qt, qoff, k, mode=mode, use_tf=use_tf)
        torch.cuda.synchronize()
        gd, gs, gc, gt = [x.cpu().numpy() for x in got]
        ok = bool(np.array_equal(gt, plain[3].cpu().numpy()))
        sample = 8
        for i in range(sample):
            d, s, tot = OO.search(n_docs, c["term_off"], c["post_doc"], queries[i].tolist(), mode == _lib.NIDX_BM25_AND, alive, created, k, OO.DESC)
            ok &= int(gc[i]) == len(d) and int(gt[i]) == tot and np.array_equal(gd[i, :len(d)].astype(np.int64), d) and np.array_equal(gs[i, :len(d)], s)
        lines.append({"metric": f"order by date ({name} top-{k})", "value": med(ms["by date"]) / med(ms["by score"]), "unit": "x (by date / by score call)",
                      "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "gpu": gpu, "higher_is_better": False, "data": "synthetic",
                      "config": {"workload": f"BM25 {n_docs} docs / {nterms}-term {'AND, tf' if use_tf else 'OR, tf == 1'} queries x {nq}, top-{k}, created DESC",
                                 "rounds": 5, "set_dates_seconds": t_dates, "distinct_created": int(len(np.unique(created)))},
                      "runs": {r: {"ms_per_call": med(ms[r]), "kernel_ms": med(kms[r])} for r in runs},
                      "parity": {"identical_to_oracle_and_total_to_search": bool(ok), "sample": sample}})
    # the catalogue listing
    list_fn = lambda: ts.list_ordered(k, _lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_DESC, device_out=True)
    l_ms, l_kms = [], []
    for _ in range(5):
        l_ms.append(timed(list_fn, args.steps, args.warmup)); l_kms.append(ts.last_kernel_ms())
    ok = True
    for field, secs in ((_lib.NIDX_ORDER_CREATED, created), (_lib.NIDX_ORDER_MODIFIED, modified)):
        for typ in (_lib.NIDX_ORDER_DESC, _lib.NIDX_ORDER_ASC):
            docs, dates, count, total = ts.list_ordered(k, field, typ)
            d, s, tot = OO.list_all(n_docs, alive, secs, k, typ)
            ok &= count == len(d) and total == tot and np.array_equal(docs[:count].astype(np.int64), d) and np.array_equal(dates[:count], s)
    nbytes = 4 * n_docs + n_docs // 8 + k * 12
    pk = 3350.0
    ach = nbytes / (med(l_kms) * 1e-3) / 1e9
    lines.append({"metric": f"order by date, catalogue listing top-{k}", "value": med(l_ms), "unit": "ms", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                  "gpu": gpu, "higher_is_better": False, "data": "synthetic",
                  "config": {"workload": f"empty body, created DESC, top-{k} over {n_docs} documents (1 % deleted)", "rounds": 5},
                  "roofline": {"bound": "hbm", "achieved": ach, "peak": pk, "unit": "GB/s", "frac": ach / pk, "kernel": "date_topk_all_kernel + date_merge_kernel",
                               "kernel_ms": med(l_kms), "alg_bytes": nbytes,
                               "alg_bytes_note": "rank column (4 B per document) + alive bits, each read once, + the top-k out; peak = H100 SXM data sheet"},
                  "parity": {"identical_to_oracle": bool(ok), "checked": "CREATED / MODIFIED x DESC / ASC"}})
    ts.close()
    return lines


def bench_rabitq(args):
    """SURVEY 8f rank 1: the HNSW walk with a RaBitQ query on a Dot index (hnsw/search.rs:306-383: estimate-ranked walk, k * 100
    layer-0 results, exact rerank) -- what the reference runs on every Dot index that carries vectors.quant -- next to the dense
    walk on the same graph.  Algorithmic bytes per query = estimates x code bytes + expansions x adjacency row + exact
    similarities x row bytes, from the kernel's counters."""
    import torch

    from bench import gen_queries, gen_vectors, recall_at_k
    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import VectorSegment

    dev = torch.device("cuda", 0)
    n, d, nq, k = args.build_vectors, 768, 1024, 10
    vecs = gen_vectors(n, d, dev, seed=1234567890, latent=16, noise=0.15)
    queries = [gen_queries(vecs, nq, seed=123 + i) for i in range(args.steps + args.warmup)]
    seg = VectorSegment.create(vecs, d, similarity=_lib.NIDX_SIM_DOT, m=16, m0=32, ef_construction=200)
    del vecs
    torch.cuda.empty_cache()
    t0 = time.perf_counter()
    seg.build_hnsw(seed=2, max_batch=8192)
    torch.cuda.synchronize()
    t_build = time.perf_counter() - t0
    seg.rabitq_encode()
    gt = seg.search(queries[0], k, method=_lib.NIDX_METHOD_BRUTE)[0].cpu().numpy()
    out = (torch.empty((nq, k), dtype=torch.int32, device=dev), torch.empty((nq, k), dtype=torch.float32, device=dev), torch.empty((nq,), dtype=torch.int32, device=dev))
    lines = []
    pk = float(peaks().get("hbm_gbs", 3350.0))
    for name, method, ef in (("quantised walk (RaBitQ query, 1000 layer-0 candidates, exact rerank)", _lib.NIDX_METHOD_HNSW_RABITQ, 0),
                             ("dense walk ef=128", _lib.NIDX_METHOD_HNSW, 128)):
        idx = [0]

        def step():
            seg.search(queries[idx[0] % len(queries)], k, ef=ef, method=method, out=out)
            idx[0] += 1

        ms = timed(step, args.steps, args.warmup)
        seg.search(queries[0], k, ef=ef, method=method, out=out)
        kms = seg.last_kernel_ms()
        c = seg.counters_ex()
        rec = recall_at_k(out[0].cpu().numpy(), gt)
        stride = (d // 8 + 8 + 15) // 16 * 16
        alg = c["estimates"] * stride + c["expansions"] * 32 * 4 + c["similarities"] * (d * 4 + 4)
        lines.append({"metric": "k-NN QPS @ recall@10", "value": nq / (ms * 1e-3), "unit": "queries/s", "n_gpus": 1, "steps": args.steps, "warmup": args.warmup,
                      "ms_per_step": ms, "higher_is_better": True, "dtype": "f32 + 1-bit codes" if method == _lib.NIDX_METHOD_HNSW_RABITQ else "f32", "data": "synthetic",
                      "config": {"workload": f"HNSW search {n}x{d} dot, {name}, k={k}, batch={nq}", "M": 16, "M0": 32, "efC": 200, "build_seconds": t_build},
                      "recall_at_10": rec, "counters_per_query": {kk: v / nq for kk, v in c.items()},
                      "roofline": {"bound": "hbm", "achieved": alg / (kms * 1e-3) / 1e9, "peak": pk, "unit": "GB/s", "frac": alg / (kms * 1e-3) / 1e9 / pk,
                                   "kernel": "hnsw_rabitq_kernel" if method == _lib.NIDX_METHOD_HNSW_RABITQ else "hnsw_search_kernel", "kernel_ms": kms,
                                   "alg_bytes_per_query": alg / nq, "traffic": None,
                                   "note": "latency bound: ~1000 dependent expansions per query, 1024 queries in flight" if method == _lib.NIDX_METHOD_HNSW_RABITQ else None}})
    seg.close()
    return lines


def driver_extras(steps=5, warmup=3):
    """The `extra` block of bench.py's line (N = 1): BASELINE configs[0] (exact scan), configs[3] (BM25) and the quantised walk on a
    1 M x 768 Dot index, each reduced to the keys a reader needs; the full lines are what `bench_extra.py` prints."""
    import torch

    class A:
        pass

    a = A()
    a.steps, a.warmup, a.docs, a.build_vectors = steps, warmup, 5_000_000, 1_000_000

    def compact(line):
        keep = ("metric", "value", "unit", "ms_per_step", "config", "parity", "recall_at_10", "roofline", "cpu_baseline", "e2e", "counters_per_query")
        return {kk: line[kk] for kk in keep if kk in line}

    out = {}
    for name, fn in (("scan", bench_scan), ("bm25", bench_bm25), ("rabitq_walk", bench_rabitq)):
        try:
            out[name] = [compact(x) for x in fn(a)]
        except Exception as e:  # noqa: BLE001
            out[name] = {"error": f"{type(e).__name__}: {e}"}
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("which", choices=["scan", "bm25", "build", "merge", "rabitq", "facets", "order", "all"])
    ap.add_argument("--build-vectors", type=int, default=1_000_000)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--docs", type=int, default=5_000_000)
    args = ap.parse_args()
    lines = []
    if args.which in ("scan", "all"):
        lines += bench_scan(args)
    if args.which in ("bm25", "all"):
        lines += bench_bm25(args)
    if args.which in ("build", "all"):
        lines += bench_build(args)
    if args.which == "merge":
        lines += bench_merge(args)
    if args.which == "rabitq":
        lines += bench_rabitq(args)
    if args.which == "facets":
        lines += bench_facets(args)
    if args.which == "order":
        lines += bench_order(args)
    for line in lines:
        print(json.dumps(line))


if __name__ == "__main__":
    main()
