"""Exact-phrase keyword search on one segment: the phrase pass (phrase_match_kernel + phrase_compact_kernel + the virtual lists'
skip rows) and the whole nidx_txt_search_phrases call, against the same words searched as a plain OR.

The corpus is bench_extra.make_corpus's shape (Zipf(1.07) vocabulary, lognormal lengths of mean 64) with every token's position
kept; queries are 2- and 3-word phrases cut from real documents, so that they match.  One JSON line: times from CUDA events after
warm-up, the phrase-pass kernels' time from torch.profiler in a run of its own, a byte model of the pass over that time as a share
of the HBM peak, a sample of the outputs checked against a brute-force count over the token stream, and the card's name and power
limit read in the same process.

    python scripts/phrase_bench.py [--docs 1000000] [--batch 1024] [--steps 10] [--warmup 3]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12   # H100 SXM data sheet, bytes/s


def make_positional_corpus(n_docs, n_terms, dev, seed=7, mean_len=64, zipf_s=1.07):
    import torch

    g = torch.Generator(device=dev)
    g.manual_seed(seed)
    sigma = 0.5
    lens = torch.exp(torch.randn(n_docs, generator=g, device=dev) * sigma + (np.log(mean_len) - sigma * sigma / 2)).clamp_(min=1).to(torch.int64)
    total = int(lens.sum().item())
    ranks = torch.arange(1, n_terms + 1, device=dev, dtype=torch.float64)
    cdf = torch.cumsum(ranks.pow(-zipf_s), 0)
    cdf /= cdf[-1].clone()
    u = torch.rand(total, generator=g, device=dev, dtype=torch.float64)
    tokens = torch.searchsorted(cdf, u).clamp_(max=n_terms - 1)
    del u
    doc_start = torch.zeros(n_docs, dtype=torch.int64, device=dev)
    doc_start[1:] = torch.cumsum(lens, 0)[:-1]
    doc_of = torch.repeat_interleave(torch.arange(n_docs, device=dev, dtype=torch.int64), lens)
    pos = torch.arange(total, device=dev, dtype=torch.int64) - doc_start[doc_of]
    keys = tokens * n_docs + doc_of
    keys, perm = torch.sort(keys, stable=True)   # (term, doc), positions ascending inside
    positions = pos[perm].to(torch.int32)
    uniq, tf = torch.unique_consecutive(keys, return_counts=True)
    term = torch.div(uniq, n_docs, rounding_mode="floor")
    doc = (uniq - term * n_docs).to(torch.int32)
    term_off = torch.zeros(n_terms + 1, dtype=torch.int64, device=dev)
    term_off[1:] = torch.cumsum(torch.bincount(term, minlength=n_terms), 0)
    return dict(lens=lens.cpu().numpy(), tokens=tokens.to(torch.int32).cpu().numpy(), doc_start=doc_start.cpu().numpy(),
                term_off=term_off.cpu().numpy().astype(np.uint64), post_doc=doc.cpu().numpy().astype(np.uint32),
                post_tf=tf.to(torch.int32).cpu().numpy().astype(np.uint32), positions=positions.cpu().numpy().astype(np.uint32))


def brute_count(c, phrase):
    """Documents holding the phrase, from the token stream itself."""
    tok, n = c["tokens"], len(phrase)
    ok = np.ones(len(tok) - n + 1, bool)
    for i, t in enumerate(phrase):
        ok &= tok[i:len(tok) - n + 1 + i] == t
    starts = np.nonzero(ok)[0]
    d0 = np.searchsorted(c["doc_start"], starts, side="right") - 1
    d1 = np.searchsorted(c["doc_start"], starts + n - 1, side="right") - 1
    return set(d0[d0 == d1].tolist())


def byte_model(c, phrases, n_fine):
    """Bytes the phrase pass reads: every driver posting (8 B) and its positions (4 B each); per driver posting and other term a
    binary search over the term's slice of one fine tile (8 B a step) and that term's positions in the document (an upper bound:
    its mean tf); the compaction reads and writes each slot once."""
    df = np.diff(c["term_off"].astype(np.int64))
    tf_sum = np.add.reduceat(c["post_tf"].astype(np.int64), c["term_off"][:-1].astype(np.int64)) if len(c["post_tf"]) else np.zeros_like(df)
    mean_tf = np.where(df > 0, tf_sum / np.maximum(df, 1), 0)
    drv = post = probe = posb = 0
    for p in phrases:
        d = min(p, key=lambda t: df[t])
        D = int(df[d])
        drv += D
        post += D * 8 + D * mean_tf[d] * 4
        for t in p:
            if t == d:
                continue
            sl = df[t] / n_fine if df[t] >= 256 else df[t]
            steps = int(np.ceil(np.log2(sl + 1))) + 1
            probe += D * steps * 8
            posb += D * mean_tf[t] * 4
    return {"driver_postings": drv, "driver_bytes": int(post), "probe_bytes": int(probe), "position_bytes": int(posb),
            "compact_bytes": drv * 16, "total_bytes": int(post + probe + posb + drv * 16)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--docs", type=int, default=1_000_000)
    ap.add_argument("--terms", type=int, default=1_000_000)
    ap.add_argument("--batch", type=int, default=1024)
    ap.add_argument("--k", type=int, default=100)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()

    import torch

    import bench_extra as BX
    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import TextSegment
    from nucliadb_b200.text import fieldnorm_to_id

    dev = torch.device("cuda", 0)
    c = make_positional_corpus(args.docs, args.terms, dev)
    lut = np.asarray([fieldnorm_to_id(i) for i in range(int(c["lens"].max()) + 1)], dtype=np.uint8)
    ts = TextSegment.create(args.docs, args.terms, c["term_off"], c["post_doc"], c["post_tf"], lut[c["lens"]])
    ts.set_positions(c["positions"])
    rng = np.random.default_rng(11)
    phrases = []
    while len(phrases) < args.batch:
        d = int(rng.integers(args.docs))
        m = 2 + len(phrases) % 2
        if c["lens"][d] < m:
            continue
        s = int(c["doc_start"][d] + rng.integers(c["lens"][d] - m + 1))
        phrases.append([int(t) for t in c["tokens"][s:s + m]])
    empty_t, empty_o = np.zeros(0, np.uint32), np.zeros(args.batch + 1, np.uint32)
    ph = [(i, p) for i, p in enumerate(phrases)]
    or_t = np.asarray([t for p in phrases for t in p], np.uint32)
    or_o = np.zeros(args.batch + 1, np.uint32)
    or_o[1:] = np.cumsum([len(p) for p in phrases])

    def call_phrase():
        return ts.search_phrases(empty_t, empty_o, ph, args.k, mode=_lib.NIDX_BM25_OR, use_tf=False)

    def call_or():
        return ts.search(or_t, or_o, args.k, mode=_lib.NIDX_BM25_OR, use_tf=False)

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(args.steps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            b.synchronize()
            ms.append(a.elapsed_time(b))
        return float(np.median(ms))

    phrase_ms, or_ms = timed(call_phrase), timed(call_or)
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.steps):
            call_phrase()
        torch.cuda.synchronize()
    kern = {}
    for e in prof.key_averages():
        if any(n in e.key for n in ("phrase_match_kernel", "phrase_compact_kernel", "bm25_build_skip_kernel", "bm25_kernel")):
            kern[e.key.split("(")[0]] = getattr(e, "device_time_total", getattr(e, "cuda_time_total", 0)) / args.steps / 1e3   # ms per call
    pass_ms = sum(v for k, v in kern.items() if "bm25_kernel" not in k)
    bm = byte_model(c, phrases, (args.docs + 4095) // 4096)
    docs, scores, counts, total = call_phrase()
    sample = list(range(0, args.batch, max(1, args.batch // 16)))
    mism = 0
    for q in sample:
        want = brute_count(c, phrases[q])
        got = set(int(x) for x in docs[q][: int(counts[q])])
        mism += int(int(total[q]) != len(want) or not got <= want)
    print(json.dumps({"metric": "phrase search", "docs": args.docs, "tokens": int(c["lens"].sum()), "postings": int(c["term_off"][-1]),
                      "queries": args.batch, "words_per_phrase": "2 and 3 alternating", "k": args.k,
                      "phrase_call_ms": phrase_ms, "or_call_ms": or_ms, "phrase_pass_kernels_ms": kern, "phrase_pass_ms": pass_ms,
                      "byte_model": bm, "phrase_pass_hbm_share": bm["total_bytes"] / (pass_ms * 1e-3) / HBM_PEAK if pass_ms else None,
                      "sample_checked": len(sample), "sample_mismatches": mism, "gpu": BX.gpu_identity()}))
    return 1 if mism else 0


if __name__ == "__main__":
    sys.exit(main())
