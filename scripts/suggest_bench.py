"""Suggest on one GPU: CUDA-event medians of the fuzzy pass split into dictionary pass (nidx_suggest_last_ms) and clause bitsets,
scored pass, top-k and matches (nidx_txt_suggest_last_times), for fuzzy terms and prefixes whose expansions hold frequent, rare
or mixed terms (with the number of expanded terms and of their postings), and the wall time of the keyword call (the paragraph
search's BM25 on a view under the suggest mask), over bench_extra's BM25 corpus in one segment; then the entity suggest (a NODES search of fuzzy prefix groups) over a synthetic relation
index.  Prints one JSON line per measurement with the card's name and power limit.

    python scripts/suggest_bench.py --paragraphs 5000000 --relations 1000000 --reps 20
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from graph_bench import card, synthetic   # noqa: E402


def _letters(i):
    """The i-th (1-based) word of the bijective base-26 numbering: a .. z, aa .. zz, aaa .."""
    out = []
    while i:
        i, r = divmod(i - 1, 26)
        out.append(chr(97 + r))
    return "".join(reversed(out))


def bm25_searcher(n):
    """The BM25 corpus of bench_extra.make_corpus (n paragraphs, lognormal lengths of mean 64, 1 M terms drawn Zipf(1.07)) as one paragraph
    segment.  Term id i is the word _letters(i + 1) below 500 000 (every word of up to 4 letters: the frequent ones) and "9z" +
    _letters(i - 499 999) from there (the rare half), so "9zq1" expands to rare terms only."""
    import torch

    from bench_extra import make_corpus
    from nucliadb_b200.text import ParagraphSearcher, TextDoc, TextIndexSegment, fieldnorm_to_id

    n_terms = 1_000_000
    c = make_corpus(n, n_terms, torch.device("cuda", 0))
    vocab = {(_letters(i + 1) if i < 500_000 else "9z" + _letters(i - 499_999)): i for i in range(n_terms)}
    seg = object.__new__(TextIndexSegment)   # the segment's arrays as the host indexer makes them, without tokenising text
    seg.docs, seg.n_docs, seg.device, seg._gpu = [TextDoc("0" * 32, "/a/summary", "", ())] * n, n, 0, None
    seg.lens = c["lens"]
    seg.total_tokens = int(c["total_tokens"])
    seg.n_terms = n_terms
    seg.post_term = np.repeat(np.arange(n_terms, dtype=np.int64), np.diff(c["term_off"].astype(np.int64)))
    seg.post_doc, seg.post_tf = c["post_doc"], c["post_tf"]
    lut = np.asarray([fieldnorm_to_id(i) for i in range(int(seg.lens.max()) + 1)], dtype=np.uint8)
    seg.fieldnorm_id = lut[seg.lens]
    seg.positions = np.zeros(0, dtype=np.uint32)
    return ParagraphSearcher([seg], vocab)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--paragraphs", type=int, default=5_000_000)
    ap.add_argument("--relations", type=int, nargs="*", default=[1_000_000])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--k", type=int, default=20)
    a = ap.parse_args()
    import torch

    from nucliadb_b200 import graph as G
    from nucliadb_b200 import suggest as S

    name, power = card()
    t0 = time.time()
    ps = bm25_searcher(a.paragraphs)
    print(f"# {a.paragraphs} paragraphs indexed in {time.time() - t0:.0f} s, {len(ps.vocab)} terms", file=sys.stderr, flush=True)
    masks = ps.suggest_masks()
    seg = ps.segments[0]._gpu
    ps._bench_df = ps.segments[0].doc_freq(len(ps.vocab)).astype(np.int64)
    # a frequent word; 4-byte fuzzy prefixes whose expansions hold terms of every frequency; a 3-byte fuzzy term that reaches the
    # frequent "ad"; a prefix that expands to rare terms only
    rows = {"keyword": "ad", "fuzzy_prefix_4_bytes": "ab1d", "fuzzy_prefix_mixed": "b1cd", "fuzzy_frequent": "ad1", "fuzzy_prefix_rare": "9zq1"}
    for qname, body in rows.items():
        ps.suggest(body, a.k, masks)   # warm-up (and the vocabulary upload)
        walls, parts, dict_ms = [], [], []
        for _ in range(a.reps):
            torch.cuda.synchronize()
            t = time.perf_counter()
            r = ps.suggest(body, a.k, masks)
            walls.append((time.perf_counter() - t) * 1e3)
            if r.fuzzy:
                parts.append(seg.suggest_last_times())
                dict_ms.append(ps._suggest_dict.last_ms())
        row = {"paragraphs": a.paragraphs, "query": qname, "body": body, "fuzzy": r.fuzzy, "hits": len(r.hits), "card": name, "power_limit": power,
               "call_ms_wall": float(np.median(walls)), "call_ms_wall_min": float(np.min(walls)), "call_ms_wall_max": float(np.max(walls))}
        if parts:
            med = np.median(np.asarray(parts), axis=0)
            auto = [(body, S.FUZZY_DISTANCE, True)] if len(body.encode()) >= S.MIN_FUZZY_PREFIX_LEN else [(body, S.FUZZY_DISTANCE, False)]
            bits, counts = ps._suggest_dict.expand(auto)
            exp = np.unpackbits(bits[0].cpu().numpy().view(np.uint8), bitorder="little")[: len(ps.vocab)].astype(bool)
            df = ps._bench_df[exp]
            row.update({"expanded_terms": int(counts[0]), "expanded_postings": int(df.sum()), "largest_expanded_df": int(df.max(initial=0)), "dict_ms": float(np.median(dict_ms)), "bitsets_ms": float(med[0]),
                        "scored_ms": float(med[1]), "topk_ms": float(med[2]), "matches_ms": float(med[3])})
        print(json.dumps(row), flush=True)
    for n in a.relations:
        t0 = time.time()
        ix = G.GraphIndex(synthetic(n))
        print(f"# {n} relations indexed in {time.time() - t0:.0f} s", file=sys.stderr, flush=True)
        req = S.entity_request("new yo", a.k)
        searcher = G.GraphSearcher(ix)
        searcher.search(req)
        times = []
        for _ in range(a.reps):
            resp = searcher.search(req)
            times.append(ix.last_times())
        t = np.asarray(times)
        med = np.median(t, axis=0)
        print(json.dumps({"relations": n, "query": "entities 'new yo'", "nodes": len(resp.nodes), "card": name, "power_limit": power,
                          "dict_ms": float(med[0]), "scored_ms": float(med[1]), "collect_ms": float(med[2]), "call_ms": float(med[3]),
                          "call_ms_min": float(t[:, 3].min()), "call_ms_max": float(t[:, 3].max())}), flush=True)
        ix.close()


if __name__ == "__main__":
    main()
