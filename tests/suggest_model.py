"""TEST INFRASTRUCTURE: a host model of Suggest's paragraph pass (nucliadb_b200/suggest.py states the rules) and a loader of the golden
suggest shard.

The keyword pass is the paragraph search's: tests/phrase_model.py's fixed-point BM25 (Basic terms, phrases at their frequency) over the
documents of the mask.  The fuzzy pass is restated from scratch: expansions by a full restricted Damerau-Levenshtein DP
(tests/graph_model.fuzzy_match) over the vocabulary, clause matches from each document's own tokens and positions, and the score
0.5 * (f32 sum in clause order of 1.0 per fuzzy clause, w_t * f32(1 / (1 + norm)) per exact term, w_p * f32(f / (f + norm)) per
phrase).  Hits are ordered by (score desc, segment, doc); matches are the sorted expanded terms of more than 2 bytes in the hit, one per
(fuzzy clause, term), for the first 10 hits."""
from __future__ import annotations

import json
import os

import numpy as np

import bm25_model as M
import graph_model as GM
import phrase_model as PM
from nucliadb_b200 import suggest as S
from nucliadb_b200.text import TextIndexSegment, paragraph_query_tokens, parse_paragraph_query, tokenize_with_positions

_f = np.float32
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "suggest_shard.json")


def golden_resources() -> list:
    return json.load(open(GOLDEN))["resources"]


class SuggestModel:
    """The paragraph documents of one index (segments of nucliadb_b200.text.TextDoc, one vocabulary, union statistics)."""

    def __init__(self, segments_docs):
        self.vocab: dict = {}
        self.segs = [TextIndexSegment(d, self.vocab) for d in segments_docs]
        n_terms = len(self.vocab)
        self.terms = sorted(self.vocab, key=self.vocab.get)
        self.total_docs = max(sum(s.n_docs for s in self.segs), 1)
        self.total_tokens = max(sum(s.total_tokens for s in self.segs), 1)
        self.df = np.zeros(n_terms, dtype=np.int64)
        for s in self.segs:
            self.df += s.doc_freq(n_terms).astype(np.int64)
        self.models, self.toks = [], []
        for s in self.segs:
            term_off = np.zeros(n_terms + 1, dtype=np.int64)
            term_off[1:] = np.cumsum(np.bincount(s.post_term, minlength=n_terms)) if n_terms else []
            toks = [tokenize_with_positions(d.text) for d in s.docs]
            pos = PM.token_positions([[(p, self.vocab[t]) for p, t in ts] for ts in toks])
            self.models.append(PM.PhraseModel(s.n_docs, n_terms, term_off, s.post_doc, s.post_tf, s.fieldnorm_id, total_docs=self.total_docs,
                                               total_tokens=self.total_tokens, doc_freq=self.df, pos=pos))
            self.toks.append(toks)
        self.norm = M.norm_cache(self.total_docs, self.total_tokens)

    def _id(self, t):
        return self.vocab.get(t, 0xFFFFFFF0)

    def keyword(self, body: str, k: int, masks) -> list:
        words, phrases = parse_paragraph_query(body)
        if not words and not phrases:
            return []
        q = ([self._id(t) for t in words], [[self._id(t) for t in p] for p in phrases])
        rows = []
        for o, (m, mask) in enumerate(zip(self.models, masks)):
            m.alive, m._ranked = np.asarray(mask, dtype=bool), {}
            docs, scores = m.ranked(q, M.OR, use_tf=False)[:2]
            rows += [(-float(s), o, int(d)) for d, s in zip(docs, scores)]
        rows.sort()
        return [(-n, o, d) for n, o, d in rows[:k]]

    def expansion(self, term: str, prefix: bool) -> set:
        return {e for e in self.terms if GM.fuzzy_match(term, e, S.FUZZY_DISTANCE, prefix)}

    def fuzzy(self, body: str, k: int, masks):
        """-> ([(score, segment, doc)] best first, {(segment, doc): matches} for the first 10)."""
        return self.fuzzy_pass(S.fuzzy_clauses(paragraph_query_tokens(body)), k, masks)

    def fuzzy_pass(self, clauses, k: int, masks):
        """The fuzzy pass over given clauses [(kind, value)] (suggest.fuzzy_clauses' format)."""
        if not clauses:
            return [], {}
        exp = [self.expansion(v, kind == S.FUZZY_PREFIX) if kind in (S.FUZZY, S.FUZZY_PREFIX) else None for kind, v in clauses]
        rows = []
        for o, (m, toks, mask) in enumerate(zip(self.models, self.toks, masks)):
            for d in np.nonzero(np.asarray(mask, dtype=bool))[0]:
                d = int(d)
                words = {t for _, t in toks[d]}
                fn = int(m.fieldnorm_id[d])
                s, hit = _f(0.0), False
                for (kind, v), e in zip(clauses, exp):
                    if e is not None:
                        if not (words & e):
                            continue
                        val = _f(1.0)
                    elif kind == S.TERM:
                        if v not in words:
                            continue
                        val = _f(M.term_weight(self.df[self.vocab[v]], self.total_docs) * _f(_f(1.0) / _f(_f(1.0) + self.norm[fn])))
                    else:
                        lists = [[p for p, t in toks[d] if t == w] for w in v]
                        f = PM.phrase_freq(lists) if all(lists) else 0
                        if not f:
                            continue
                        w = m.phrase_weight([self._id(t) for t in v])
                        val = _f(w * _f(_f(f) / _f(_f(f) + self.norm[fn])))
                    hit = True
                    s = _f(s + val)
                if hit:
                    rows.append((-float(_f(_f(0.5) * s)), o, d))
        rows.sort()
        hits = [(-n, o, d) for n, o, d in rows[:k]]
        matches = {}
        for _, o, d in hits[: S.RESULTS_PER_PAGE]:
            words = {t for _, t in self.toks[o][d]}
            matches[(o, d)] = sorted(t for e in exp if e is not None for t in e & words if len(t.encode("utf-8")) > 2)
        return hits, matches

    def suggest(self, body: str, k: int, masks):
        """-> (hits [(score, segment, doc)], fuzzy, matches {(segment, doc): [terms]})."""
        hits = self.keyword(body, k, masks)
        if hits:
            return hits, False, {}
        hits, matches = self.fuzzy(body, k, masks)
        return hits, True, matches
