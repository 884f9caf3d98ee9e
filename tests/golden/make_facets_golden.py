"""Writes tests/golden/facets_small.npz: a seeded corpus (postings, alive bits, label strings per document), queries and facet
requests, and the expected facet counts, computed by a literal transcription of the counting rule over the label strings:
for a requested facet F and each direct child C of F, the number of matched documents (query match AND alive; OR and AND) that
carry C or a descendant of C, once per document.  Run from the repository root: python tests/golden/make_facets_golden.py"""
import os

import numpy as np

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "facets_small.npz")
REQUESTS = [["/l"], ["/l", "/e", "/k"], ["/"], ["/l/a", "/l/b", "/e"]]


def main():
    rng = np.random.default_rng(20261015)
    n_docs, n_terms = 500, 60
    vocab = ["/l", "/l/a", "/l/a/x", "/l/a/y", "/l/b", "/l/b/z", "/l/c", "/e/p", "/e/q/r", "/e", "/k/1", "/k/2/3", "/la/x", "/ll"]
    labels = [sorted(set(rng.choice(vocab, size=rng.integers(0, 5)).tolist())) for _ in range(n_docs)]
    pairs = sorted({(int(rng.integers(0, n_terms)), d) for d in range(n_docs) for _ in range(8)})
    term_off = np.zeros(n_terms + 1, dtype=np.uint64)
    term_off[1:] = np.cumsum(np.bincount([p[0] for p in pairs], minlength=n_terms))
    post_doc = np.asarray([p[1] for p in pairs], dtype=np.uint32)
    alive_b = rng.random(n_docs) < 0.8
    alive = np.packbits(alive_b, bitorder="little")
    alive = np.concatenate([alive, np.zeros(-len(alive) % 8, np.uint8)]).view(np.uint64)
    queries = [[1, 2, 3], [7], [4, 9, 11, 20, 33]]
    label_off = np.concatenate([[0], np.cumsum([len(l) for l in labels])]).astype(np.int64)
    exp = []
    for qi, terms in enumerate(queries):
        sets = [set(post_doc[int(term_off[t]):int(term_off[t + 1])].tolist()) for t in terms]
        for conj in (0, 1):
            docs = set.intersection(*sets) if conj else set.union(*sets)
            for ri, request in enumerate(REQUESTS):
                for f in request:
                    fs = [] if f == "/" else f[1:].split("/")
                    counts = {}
                    for d in sorted(docs):
                        if not alive_b[d]:
                            continue
                        kids = {"/" + "/".join(l[1:].split("/")[: len(fs) + 1]) for l in labels[d]
                                if len(l[1:].split("/")) > len(fs) and l[1:].split("/")[: len(fs)] == fs}
                        for c in kids:
                            counts[c] = counts.get(c, 0) + 1
                    exp += [(qi, conj, ri, f, c, n) for c, n in sorted(counts.items())]
    np.savez_compressed(
        OUT, term_off=term_off, post_doc=post_doc, alive=alive, label_off=label_off,
        labels=np.asarray([l for ls in labels for l in ls]), query_off=np.asarray([0] + list(np.cumsum([len(q) for q in queries])), dtype=np.uint32),
        query_terms=np.asarray([t for q in queries for t in q], dtype=np.uint32), request_off=np.asarray([0] + list(np.cumsum([len(r) for r in REQUESTS]))),
        requests=np.asarray([f for r in REQUESTS for f in r]), exp_q=np.asarray([e[0] for e in exp]), exp_conj=np.asarray([e[1] for e in exp]),
        exp_req=np.asarray([e[2] for e in exp]), exp_group=np.asarray([e[3] for e in exp]), exp_tag=np.asarray([e[4] for e in exp]),
        exp_count=np.asarray([e[5] for e in exp]))


if __name__ == "__main__":
    main()
