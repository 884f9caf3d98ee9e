"""TEST INFRASTRUCTURE: a host model of the BM25 kernel's score, bit for bit (nucliadb_b200/csrc/bm25.cuh, bm25_kernel and
bm25_finish_kernel, with the statistics of txt_upload_stats in api.cu).

It restates what the CUDA code computes, not what tantivy computes: tantivy sums f32 term scores (oracle/bm25.hpp), the kernel sums
fixed-point integers.  Per query, in f32 and in this order:
  w_t    = f32(idf_t) * f32(1 + K1)                        idf_t from oracle.bm25_idf (the same logf expression as api.cu)
  norm   = K1 * ((1 - B) + (B * value(fieldnorm id)) / avg),   avg = f32(total_tokens) / f32(total_docs)
  s      = the largest s in [4, 24] with max(1, f32(nt) * max_i w_i) * 2^s < 4.0e9   (unknown terms weigh 0)
  frac   = tf / (tf + norm)  with tf (clamped to 0xFFFFFF when packed);  Basic: 1 / (1 + norm)
  fx     = rint_half_even(f32(f32(w_t * 2^s) * frac)),  1 where that is 0
  score  = f32(sum of fx, exact) / 2^s
  order  = (score desc, doc asc); alive bits and search-after before the top-k, min_score after it.

Error against the real-valued score S = sum_t c_t, c_t = w_t * tf / (tf + norm) in float64 on the same f32 w_t and norm (u = 2^-24):
  frac carries two roundings and the product a third, so fx = c_t 2^s (1 + theta) + r with |theta| <= 3u + 3u^2 and |r| <= 1
  (rint moves by 1/2 at most; the fx = 1 floor replaces a value in [0, 1/2] by 1).  The integer sum is exact, and rounding it to
  f32 moves it by u * score at most; dividing by 2^s is exact.  So
      |score - S| <= u * |score| + sum_t (3.01 u c_t + 2^-s)                                                   (error_bound)
The shift rule keeps the sum below 2^32: fx <= w_t 2^s * frac + 1/2 with frac <= 1, so the sum is at most
nt * max_t w_t * 2^s + nt / 2 < 4.0e9 (1 + u) + 64 < 2^32."""
import numpy as np

import oracle as O

NIL = 0xFFFFFFFF
OR, AND = 0, 1
K1, B = np.float32(1.2), np.float32(0.75)
MAX_TERMS = 128
TF_MAX = 0xFFFFFF                   # bm25_pack_kernel stores tf in 24 bits
LIMIT = np.float32(4.0e9)
U = 2.0 ** -24
_f = np.float32


def f32_of_int(n) -> np.float32:
    """(float)n for an unsigned 64-bit integer, rounded to nearest even (as the C conversion does; no double rounding)."""
    n = int(n)
    if n < 1 << 24:
        return _f(n)
    e = n.bit_length() - 24
    m, r = divmod(n, 1 << e)
    half = 1 << (e - 1)
    if r > half or (r == half and m & 1):
        m += 1
    return _f(float(m) * 2.0 ** e)   # m <= 2^24: exact in float64 and in f32 (a carry to 2^24 stays exact)


_VALUES = None


def fieldnorm_values() -> np.ndarray:
    global _VALUES
    if _VALUES is None:
        _VALUES = np.array([O.fieldnorm_id_to_value(i) for i in range(256)], dtype=np.uint32)
    return _VALUES


def norm_cache(total_docs, total_tokens) -> np.ndarray:
    """txt_upload_stats: K1 * (1 - B + B * value / avg), every operation rounded to f32 (no contraction: -ffp-contract=off)."""
    avg = _f(f32_of_int(total_tokens) / f32_of_int(total_docs))
    vals = np.array([f32_of_int(v) for v in fieldnorm_values()], dtype=np.float32)
    return (K1 * ((_f(1.0) - B) + (B * vals) / avg)).astype(np.float32)


def term_weight(df, total_docs) -> np.float32:
    return _f(_f(O.bm25_idf(int(df), int(total_docs))) * (_f(1.0) + K1))


def query_shift(weights) -> int:
    """The fixed-point shift of one query from its terms' weights (unknown terms weigh 0)."""
    nt = len(weights)
    wmax = max([_f(w) for w in weights], default=_f(0.0))
    bound = max(_f(1.0), _f(_f(nt) * wmax))
    s = 24
    with np.errstate(over="ignore"):
        while s > 4 and _f(bound * _f(2.0 ** s)) >= LIMIT:
            s -= 1
    return s


def error_bound(score, csum, n_post, shift):
    """|score - S| <= u |score| + 3.01 u sum_t c_t + n_post 2^-s (see the module docstring)."""
    return U * np.abs(np.asarray(score, dtype=np.float64)) + 3.01 * U * np.asarray(csum, dtype=np.float64) + np.asarray(n_post) * 2.0 ** -shift


class Bm25Model:
    """One text segment as the library holds it.  Statistics default to the segment's own, as nidx_txt_create sets them (document
    count and the sum of the quantised lengths, at least 1 each); pass total_docs / total_tokens / doc_freq as set_stats does."""

    def __init__(self, n_docs, n_terms, term_off, post_doc, post_tf, fieldnorm_id, total_docs=None, total_tokens=None, doc_freq=None,
                 alive_bits=None):
        self.n_docs, self.n_terms = int(n_docs), int(n_terms)
        self.term_off = np.asarray(term_off, dtype=np.int64)
        self.post_doc = np.asarray(post_doc, dtype=np.int64)
        self.post_tf = np.minimum(np.asarray(post_tf, dtype=np.int64), TF_MAX)
        self.fieldnorm_id = np.asarray(fieldnorm_id, dtype=np.uint8)
        own_df = np.diff(self.term_off)
        if total_docs is None:
            total_docs = max(self.n_docs, 1)
            total_tokens = max(int(fieldnorm_values()[self.fieldnorm_id].astype(np.int64).sum()), 1)
        self.total_docs, self.total_tokens = int(total_docs), int(total_tokens)
        self.df = own_df if doc_freq is None else np.asarray(doc_freq, dtype=np.int64)
        self.norm = norm_cache(self.total_docs, self.total_tokens)
        self.basic = (_f(1.0) / (_f(1.0) + self.norm)).astype(np.float32)
        self._w, self._ranked = {}, {}
        self.alive = None
        if alive_bits is not None:
            bits = np.unpackbits(np.asarray(alive_bits, dtype=np.uint64).view(np.uint8), bitorder="little")
            self.alive = bits[: self.n_docs].astype(bool)

    @classmethod
    def of(cls, P, **kw):
        """From an oracle.Postings (statistics: the segment's own exact ones unless given, as the tests' set_stats calls pass)."""
        kw.setdefault("total_docs", P.n_docs)
        kw.setdefault("total_tokens", P.total_tokens)
        kw.setdefault("doc_freq", P.doc_freq)
        return cls(P.n_docs, P.n_terms, P.term_off, P.post_doc, P.post_tf, P.fieldnorm_id, **kw)

    def weight(self, t) -> np.float32:
        if t not in self._w:
            self._w[t] = term_weight(self.df[t], self.total_docs)
        return self._w[t]

    def weights(self, query):
        return [self.weight(int(t)) if int(t) < self.n_terms else _f(0.0) for t in query]

    def shift(self, query) -> int:
        return query_shift(self.weights(query))

    def ranked(self, query, mode=OR, use_tf=True):
        """Every matching alive document of one query, best first: (docs int64, scores f32, fixed-point sums, csum, n_post, shift).
        csum = sum of the postings' real-valued terms c_t (float64), n_post = postings summed (for error_bound)."""
        key = (tuple(int(t) for t in query), mode, bool(use_tf))
        if key not in self._ranked:
            self._ranked[key] = self._rank(list(key[0]), mode, use_tf)
        return self._ranked[key]

    def _rank(self, query, mode, use_tf):
        assert len(query) <= MAX_TERMS
        empty = (np.zeros(0, np.int64), np.zeros(0, np.float32), np.zeros(0, np.uint64), np.zeros(0), np.zeros(0, np.int64))
        s = self.shift(query) if query else 24
        if not query:
            return (*empty, s)
        w = self.weights(query)
        docs, fx, c = [], [], []
        scale = _f(2.0 ** s)
        for t, wt in zip(query, w):
            if t >= self.n_terms or self.term_off[t] == self.term_off[t + 1]:
                if mode == AND:
                    return (*empty, s)
                continue
            b, e = self.term_off[t], self.term_off[t + 1]
            d = self.post_doc[b:e]
            fn = self.fieldnorm_id[d]
            if use_tf:
                tff = self.post_tf[b:e].astype(np.float32)
                frac = (tff / (tff + self.norm[fn])).astype(np.float32)
                exact = wt.astype(np.float64) * self.post_tf[b:e] / (self.post_tf[b:e] + self.norm[fn].astype(np.float64))
            else:
                frac = self.basic[fn]
                exact = wt.astype(np.float64) / (1.0 + self.norm[fn].astype(np.float64))
            x = np.rint((_f(wt * scale) * frac).astype(np.float32)).astype(np.uint64)
            x[x == 0] = 1
            docs.append(d); fx.append(x); c.append(exact)
        if not docs:
            return (*empty, s)
        d, x, c = np.concatenate(docs), np.concatenate(fx), np.concatenate(c)
        order = np.argsort(d, kind="stable")
        d, x, c = d[order], x[order], c[order]
        uniq, start, npost = np.unique(d, return_index=True, return_counts=True)
        sums = np.add.reduceat(x, start)
        csum = np.add.reduceat(c, start)
        assert (sums < 1 << 32).all(), "the shift rule must keep every sum inside uint32"
        keep = npost == len(query) if mode == AND else np.ones(len(uniq), bool)
        if self.alive is not None:
            keep &= self.alive[uniq]
        uniq, sums, csum, npost = uniq[keep], sums[keep], csum[keep], npost[keep]
        score = (sums.astype(np.float64).astype(np.float32) / scale).astype(np.float32)   # sums < 2^32: exact in f64, one rounding to f32
        idx = np.lexsort((uniq, -score.astype(np.float64)))
        return uniq[idx], score[idx], sums[idx], csum[idx], npost[idx], s

    def search(self, queries, k, mode=OR, use_tf=True, min_score=0.0, after=None, docaddr_base=0):
        """TextSegment.search's outputs: (docs uint32 [nq][k] NIL-padded, scores f32 0-padded, counts int32, total uint64)."""
        nq = len(queries)
        docs = np.full((nq, k), NIL, dtype=np.uint32)
        scores = np.zeros((nq, k), dtype=np.float32)
        counts = np.zeros(nq, dtype=np.int32)
        total = np.zeros(nq, dtype=np.uint64)
        for q, query in enumerate(queries):
            d, sc = self.ranked(query, mode, use_tf)[:2]
            total[q] = len(d)
            if after is not None:   # is_after (nidx_paragraph reader.rs:379-392): 1 Drop, 2 KeepAfter, 3 Keep equal scores
                a_score, a_mode, a_addr = _f(after[0]), int(after[1]), int(after[2])
                eq = sc == a_score
                tie_ok = np.full(len(d), a_mode == 3) if a_mode != 2 else (docaddr_base + d > a_addr)
                ok = (sc < a_score) | (eq & tie_ok) if a_mode != 0 else np.ones(len(d), bool)
                d, sc = d[ok], sc[ok]
            d, sc = d[:k], sc[:k]
            ok = ~(sc < _f(min_score))
            d, sc = d[ok], sc[ok]
            docs[q, : len(d)] = d
            scores[q, : len(d)] = sc
            counts[q] = len(d)
        return docs, scores, counts, total
