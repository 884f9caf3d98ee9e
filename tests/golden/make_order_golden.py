"""Writes tests/golden/order_small.npz: a small corpus with created / modified seconds (heavy ties, undated documents, the ends
of the i64 range), alive bits and queries, plus the expected date-ordered top-k of every (query, AND/OR, field, direction)
computed by the order rule as written (tests/order_oracle.py literal_order: sorted() on Python ints) over a plain-Python matched
set.  Deterministic: `python tests/golden/make_order_golden.py` reproduces the file byte for byte on the same numpy."""
import os

import numpy as np

NONE = -(1 << 63)
K = 12


def build():
    rng = np.random.default_rng(20261015)
    n_docs, n_terms = 400, 30
    pairs = sorted({(int(rng.integers(0, n_terms)), d) for d in range(n_docs) for _ in range(5)})
    term_off = np.zeros(n_terms + 1, dtype=np.uint64)
    term_off[1:] = np.cumsum(np.bincount([p[0] for p in pairs], minlength=n_terms))
    post_doc = np.asarray([p[1] for p in pairs], dtype=np.uint32)
    base = 1_600_000_000
    created = (base + rng.integers(0, 25, n_docs) * 3600).astype(np.int64)   # 25 distinct dates over 400 documents
    modified = created + rng.integers(0, 3, n_docs).astype(np.int64) * 60
    created[rng.random(n_docs) < 0.1] = NONE
    modified[rng.random(n_docs) < 0.1] = NONE
    created[[5, 6, 7]] = [-(1 << 63) + 1, (1 << 63) - 1, -1]
    modified[[8, 9]] = [(1 << 63) - 1, -(1 << 62)]
    alive_b = rng.random(n_docs) < 0.85
    alive = np.packbits(alive_b, bitorder="little")
    alive = np.concatenate([alive, np.zeros(-len(alive) % 8, np.uint8)]).view(np.uint64)
    queries = [[1, 2, 3], [4], [0, 5, 9, 11, 17, 22], [6, 7], [999]]
    posting_sets = [set(post_doc[int(term_off[t]):int(term_off[t + 1])].tolist()) for t in range(n_terms)]
    exp_q, exp_conj, exp_field, exp_type, exp_docs, exp_total = [], [], [], [], [], []
    for qi, terms in enumerate(queries):
        sets = [posting_sets[t] if t < n_terms else set() for t in terms]
        for conj in (0, 1):
            hit = set.intersection(*sets) if conj else set.union(*sets)
            docs = [d for d in sorted(hit) if alive_b[d]]
            for field, secs in enumerate((created, modified)):
                for typ in (0, 1):
                    def key(d):
                        s = int(secs[d])
                        return (s == NONE, 0 if s == NONE else (s if typ == 1 else -s), d)
                    top = sorted(docs, key=key)[:K]
                    exp_q.append(qi); exp_conj.append(conj); exp_field.append(field); exp_type.append(typ)
                    exp_docs.append(top + [-1] * (K - len(top))); exp_total.append(len(docs))
    qo = np.asarray([0] + list(np.cumsum([len(q) for q in queries])), dtype=np.uint32)
    return dict(term_off=term_off, post_doc=post_doc, created=created, modified=modified, alive=alive, query_terms=np.asarray(sum(queries, []), dtype=np.uint32),
                query_off=qo, k=np.asarray(K), exp_q=np.asarray(exp_q, np.int32), exp_conj=np.asarray(exp_conj, np.int32), exp_field=np.asarray(exp_field, np.int32),
                exp_type=np.asarray(exp_type, np.int32), exp_docs=np.asarray(exp_docs, np.int64), exp_total=np.asarray(exp_total, np.int64))


if __name__ == "__main__":
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), "order_small.npz"), **build())
