"""A host model of the graph search (nucliadb_b200/graph.py's module docstring states the rules): every relation document is scored
by walking the query tree, fuzzy leaves by a full restricted Damerau-Levenshtein DP, then PATH / NODES / RELATIONS are collected
and ordered.  It shares only the query tree (graph.path_query / node_query, which restate graph_query_parser.rs), normalisation and
the f32 leaf formula with the device path; dictionaries, ords, the program and the collection are its own."""
from __future__ import annotations

import numpy as np

from nucliadb_b200 import graph as G
from nucliadb_b200.text import facet_key


def osa(a: str, b: str) -> int:
    """Restricted Damerau-Levenshtein (optimal string alignment) distance on code points."""
    m, n = len(a), len(b)
    D = [[0] * (n + 1) for _ in range(m + 1)]
    for i in range(m + 1):
        D[i][0] = i
    for j in range(n + 1):
        D[0][j] = j
    for i in range(1, m + 1):
        for j in range(1, n + 1):
            D[i][j] = min(D[i - 1][j] + 1, D[i][j - 1] + 1, D[i - 1][j - 1] + (a[i - 1] != b[j - 1]))
            if i > 1 and j > 1 and a[i - 1] == b[j - 2] and a[i - 2] == b[j - 1]:
                D[i][j] = min(D[i][j], D[i - 2][j - 2] + 1)
    return D


def fuzzy_match(term: str, entry: str, d: int, prefix: bool) -> bool:
    D = osa(term, entry)
    if prefix:
        return min(D[len(term)][j] for j in range(len(entry) + 1)) <= d
    return D[len(term)][len(entry)] <= d


def _facet_terms(facets) -> set:
    out = set()
    for f in facets:
        k = facet_key(f)
        if k is None:
            continue
        out.add(b"")
        out.update(k[:i] for i, c in enumerate(k) if c == 0)
        out.add(k)
    return out


def some_mask(docs, fields) -> list:
    """The Some prefilter's rule (reader.rs:52-95, AddMetadataFieldIterator): fields = [(resource uuid hex, field path or None)]; a
    relation passes when its (resource, field) is listed (the path without its leading '/'), or when its field is a/metadata and its
    resource is listed at all."""
    listed = {(r, f.lstrip("/")) for r, f in fields if f is not None}
    resources = {r for r, _ in fields}
    return [(d.rid, d.field) in listed or (d.field == G.META_FIELD and d.rid in resources) for d in docs]


class Model:
    """Every leaf is evaluated over all documents at once (numpy): a term or fuzzy leaf on the distinct values of its field, then
    mapped to the documents; f32 sums elementwise in the order of the rules."""

    _SINGLE = ("src_norm", "dst_norm", "src_type", "dst_type", "src_sub", "dst_sub", "rel_type", "label")

    def __init__(self, docs, alive=None):
        self.docs = list(docs)
        n = len(self.docs)
        self.alive = np.ones(n, dtype=bool) if alive is None else np.asarray(alive, dtype=bool)
        terms = [G.doc_terms(d) for d in self.docs]
        self.n = int(self.alive.sum())
        self.col = {}   # field -> (distinct values, each document's index into them)
        for f in self._SINGLE:
            vals = [ts[f][0] for ts in terms]
            uniq = sorted(set(vals), key=lambda v: (str(type(v)), v))
            at = {v: i for i, v in enumerate(uniq)}
            self.col[f] = (uniq, np.asarray([at[v] for v in vals], dtype=np.int64))
        self.multi = {}  # field -> (distinct terms, term index per entry, document per entry)
        for f, get in (("src_tok", lambda i: terms[i]["src_tok"]), ("dst_tok", lambda i: terms[i]["dst_tok"]),
                       ("facet", lambda i: sorted(_facet_terms(self.docs[i].facets)))):
            ent = [(t, i) for i in range(n) for t in get(i)]
            uniq = sorted({t for t, _ in ent})
            at = {t: j for j, t in enumerate(uniq)}
            self.multi[f] = (uniq, np.asarray([at[t] for t, _ in ent], dtype=np.int64), np.asarray([i for _, i in ent], dtype=np.int64))
        self._df = {}

    def _hit(self, f, pred):
        """Documents with a term of field f for which pred(term) holds."""
        n = len(self.docs)
        if f in self.col:
            uniq, idx = self.col[f]
            ok = np.asarray([pred(v) for v in uniq], dtype=bool)
            return ok[idx] if len(uniq) else np.zeros(n, dtype=bool)
        uniq, tid, doc = self.multi[f]
        ok = np.asarray([pred(v) for v in uniq], dtype=bool)
        hit = np.zeros(n, dtype=bool)
        if len(tid):
            hit[doc[ok[tid]]] = True
        return hit

    def df(self, f, v) -> int:
        key = (f, v if f != "facet" else facet_key(v))
        if key not in self._df:
            self._df[key] = int((self._hit(f, lambda t: t == key[1]) & self.alive).sum())
        return self._df[key]

    def eval(self, q):
        """-> (matched bool [n], f32 scores [n], 0 where unmatched)."""
        n = len(self.docs)
        zero, one = np.zeros(n, dtype=np.float32), np.ones(n, dtype=np.float32)
        kind = q[0]
        if kind in ("all", "prefilter"):
            return np.ones(n, dtype=bool), one
        if kind == "empty":
            return np.zeros(n, dtype=bool), zero
        if kind == "term":
            f, v = q[1], q[2]
            key = facet_key(v) if f == "facet" else v
            hit = self._hit(f, lambda t: t == key) if key is not None else np.zeros(n, dtype=bool)
            return hit, np.where(hit, G.leaf_score(self.n, self.df(f, v)), np.float32(0)).astype(np.float32)
        if kind == "termset":
            want = set(q[2])
            hit = self._hit(q[1], lambda t: t in want)
            return hit, np.where(hit, one, zero)
        if kind == "fuzzy":
            f, t, d, p = q[1:]
            hit = self._hit(f, lambda e: fuzzy_match(t, e, d, p))
            return hit, np.where(hit, one, zero)
        musts = [self.eval(c) for o, c in q[1] if o == G.MUST]
        shoulds = [self.eval(c) for o, c in q[1] if o == G.SHOULD]
        nots = [self.eval(c)[0] for o, c in q[1] if o == G.MUST_NOT]
        if not musts and not shoulds:
            return np.zeros(n, dtype=bool), zero
        ok = np.logical_and.reduce([m for m, _ in musts]) if musts else np.logical_or.reduce([m for m, _ in shoulds])
        for x in nots:
            ok = ok & ~x
        s_must = s_should = None
        if musts:
            s_must = musts[0][1]
            for _, s in musts[1:]:
                s_must = (s_must + s).astype(np.float32)
        if shoulds:
            s_should = np.where(shoulds[0][0], shoulds[0][1], zero)
            for m, s in shoulds[1:]:
                s_should = (s_should + np.where(m, s, zero)).astype(np.float32)
        score = (s_must + s_should).astype(np.float32) if s_must is not None and s_should is not None else (s_must if s_must is not None else s_should)
        return ok, np.where(ok, score, zero).astype(np.float32)

    def matches(self, q, mask=None) -> list:
        ok, score = self.eval(q)
        ok = ok & self.alive
        if mask is not None:
            ok = ok & np.asarray(mask, dtype=bool)
        idx = np.nonzero(ok)[0]
        return [(int(i), np.float32(score[i])) for i in idx]

    def search(self, trees, kind: int, k: int, mask=None) -> list:
        """-> [(key, score)]: PATH keys are documents, NODES keys (value, type, subtype), RELATIONS keys (type, label)."""
        if kind == G.PATH:
            hits = self.matches(trees[0], mask)
            return sorted(hits, key=lambda t: (-t[1], t[0]))[:k]
        best: dict = {}
        sides = [(trees[0], "source"), (trees[1], "target")] if kind == G.NODES else [(trees[0], None)]
        for tree, side in sides:
            for i, s in self.matches(tree, mask):
                d = self.docs[i]
                key = getattr(d, side) if side else (d.rel_type, d.label)
                if key not in best or s > best[key]:
                    best[key] = s
        return sorted(best.items(), key=lambda t: (-t[1], t[0]))[:k]

    def request(self, request, some_mask=None) -> list:
        """GraphSearchRequest -> the model's [(key, score)] (some_mask: the documents a Some prefilter admits)."""
        if not request.HasField("query") or not request.query.HasField("path") or request.top_k == 0:
            return []
        pq, kind, some = request.query.path, int(request.kind), some_mask is not None
        trees = [G.with_prefilter(G.node_query(pq, "src"), some), G.with_prefilter(G.node_query(pq, "dst"), some)] if kind == G.NODES else \
            [G.with_prefilter(G.path_query(pq), some)]
        return self.search(trees, kind, int(request.top_k), some_mask)
