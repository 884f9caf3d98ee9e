"""TEST INFRASTRUCTURE: phrase clauses on top of tests/bm25_model.py -- the kernel's fixed-point scores bit for bit with exact phrases
(nucliadb_b200/csrc/phrase.cuh and bm25_body's virtual lists), and an independent restatement of what a phrase matches.

Semantics (tantivy 0.26 PhraseQuery, slop 0 [recalled]):
  * a token's position is its index in the SimpleTokenizer stream before RemoveLongFilter(40): a dropped token leaves a gap;
  * freq(doc) = |intersection over i of {p - i : p in pos(t_i, doc)}|, a match when freq >= 1 ("a a" on "a a a" counts 2);
  * weight = f32(f32 sum of idf(t_i) in phrase order, repeats counted) * f32(1 + K1), idf from the index's (union) statistics;
    0 when a term id is not in the dictionary (the phrase then matches nothing);
  * the phrase is one clause, scored like a TF term with freq as tf -- also beside Basic (tf == 1) terms.
The fixed-point shift counts a phrase as one clause and its weight in the maximum."""
import numpy as np

import bm25_model as M

_f = np.float32


def phrase_freq(positions, start_offsets=None):
    """Independent restatement: positions = [sorted positions of t_0 in doc, of t_1, ...] -> freq (plain sets, no merge)."""
    starts = set(positions[0])
    for i, ps in enumerate(positions[1:], 1):
        starts &= {p - i for p in ps}
    return len([s for s in starts if s >= 0])


def token_positions(docs_tokens):
    """[[(position, term id)] per doc] -> {(term, doc): [positions ascending]}."""
    out = {}
    for d, toks in enumerate(docs_tokens):
        for p, t in toks:
            out.setdefault((int(t), d), []).append(int(p))
    return out


def positions_in_posting_order(term_off, post_doc, pos):
    """The nidx_txt_set_positions array: for every posting (term by term, doc ascending) its positions."""
    n_terms = len(term_off) - 1
    out = []
    for t in range(n_terms):
        for i in range(int(term_off[t]), int(term_off[t + 1])):
            out += pos[(t, int(post_doc[i]))]
    return np.asarray(out, dtype=np.uint32)


class PhraseModel(M.Bm25Model):
    """Bm25Model whose queries are (terms, phrases): `pos` = {(term, doc): positions} of the segment."""

    def __init__(self, *args, pos=None, **kw):
        super().__init__(*args, **kw)
        self.pos = pos or {}
        self.idf_cache = {}

    def idf(self, t) -> np.float32:
        if t not in self.idf_cache:
            self.idf_cache[t] = _f(M.O.bm25_idf(int(self.df[t]), int(self.total_docs)))
        return self.idf_cache[t]

    def phrase_weight(self, phrase) -> np.float32:
        if any(int(t) >= self.n_terms for t in phrase):
            return _f(0.0)
        s = _f(0.0)
        for t in phrase:
            s = _f(s + self.idf(int(t)))
        return _f(s * (_f(1.0) + M.K1))

    def phrase_postings(self, phrase):
        """(docs ascending, freq) of one phrase in this segment."""
        phrase = [int(t) for t in phrase]
        if any(t >= self.n_terms or self.term_off[t] == self.term_off[t + 1] for t in phrase):
            return np.zeros(0, np.int64), np.zeros(0, np.int64)
        t0 = phrase[0]
        docs, freqs = [], []
        for d in self.post_doc[self.term_off[t0]:self.term_off[t0 + 1]]:
            lists = [self.pos.get((t, int(d))) for t in phrase]
            if any(x is None for x in lists):
                continue
            f = phrase_freq(lists)
            if f:
                docs.append(int(d)); freqs.append(f)
        return np.asarray(docs, np.int64), np.asarray(freqs, np.int64)

    def ranked(self, query, mode=M.OR, use_tf=True):
        terms, phrases = query
        key = (tuple(int(t) for t in terms), tuple(tuple(int(t) for t in p) for p in phrases), mode, bool(use_tf))
        if key not in self._ranked:
            self._ranked[key] = self._rank_phrases(list(key[0]), [list(p) for p in key[1]], mode, use_tf)
        return self._ranked[key]

    def _rank_phrases(self, terms, phrases, mode, use_tf):
        nclauses = len(terms) + len(phrases)
        assert nclauses <= M.MAX_TERMS
        empty = (np.zeros(0, np.int64), np.zeros(0, np.float32), np.zeros(0, np.uint64), np.zeros(0), np.zeros(0, np.int64))
        w = self.weights(terms) + [self.phrase_weight(p) for p in phrases]
        s = M.query_shift(w) if nclauses else 24
        if not nclauses:
            return (*empty, s)
        scale = _f(2.0 ** s)
        docs, fx, c = [], [], []

        def add(d, tf, wt, basic):
            fn = self.fieldnorm_id[d]
            if basic:
                frac = self.basic[fn]
                exact = wt.astype(np.float64) / (1.0 + self.norm[fn].astype(np.float64))
            else:
                tff = tf.astype(np.float32)
                frac = (tff / (tff + self.norm[fn])).astype(np.float32)
                exact = wt.astype(np.float64) * tf / (tf + self.norm[fn].astype(np.float64))
            x = np.rint((_f(wt * scale) * frac).astype(np.float32)).astype(np.uint64)
            x[x == 0] = 1
            docs.append(d); fx.append(x); c.append(exact)

        for t, wt in zip(terms, w):
            if t >= self.n_terms or self.term_off[t] == self.term_off[t + 1]:
                if mode == M.AND:
                    return (*empty, s)
                continue
            b, e = self.term_off[t], self.term_off[t + 1]
            add(self.post_doc[b:e], self.post_tf[b:e], wt, not use_tf)
        for p, wt in zip(phrases, w[len(terms):]):
            d, f = self.phrase_postings(p)
            if not len(d):
                if mode == M.AND:
                    return (*empty, s)
                continue
            add(d, f, wt, False)
        if not docs:
            return (*empty, s)
        d, x, c = np.concatenate(docs), np.concatenate(fx), np.concatenate(c)
        order = np.argsort(d, kind="stable")
        d, x, c = d[order], x[order], c[order]
        uniq, start, npost = np.unique(d, return_index=True, return_counts=True)
        sums = np.add.reduceat(x, start)
        csum = np.add.reduceat(c, start)
        assert (sums < 1 << 32).all()
        keep = npost == nclauses if mode == M.AND else np.ones(len(uniq), bool)
        if self.alive is not None:
            keep &= self.alive[uniq]
        uniq, sums, csum, npost = uniq[keep], sums[keep], csum[keep], npost[keep]
        score = (sums.astype(np.float64).astype(np.float32) / scale).astype(np.float32)
        idx = np.lexsort((uniq, -score.astype(np.float64)))
        return uniq[idx], score[idx], sums[idx], csum[idx], npost[idx], s
