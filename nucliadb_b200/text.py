"""Host-side mirror of the BM25 part of ``nidx_text`` / ``nidx_paragraph`` over the CUDA library.

Reference call shape (the scoring itself is tantivy's, restated in oracle/bm25.hpp and done on the GPU by
``bm25_kernel``):

* ``TextSearcher.search(DocumentSearchRequest)``      nidx_text/src/lib.rs:178-227 -> reader.rs:367-451
  body parsed with ``QueryParser::set_conjunction_by_default`` (AND of terms, real tf), ``TopDocs(k+1)``,
  ``next_page = len > k``, hits below ``min_score`` dropped (reader.rs:289-355).
* ``ParagraphSearcher.search(ParagraphSearchRequest)``  nidx_paragraph/src/lib.rs:117-147 -> reader.rs:244-392
  keyword query = OR of ``TermQuery(IndexRecordOption::Basic)`` (keyword_parser.rs:27-67): tf == 1.
* statistics over the union of all segments (nidx_tantivy/src/index_reader.rs:39-77); results ordered by
  (score desc, segment_ord asc, doc asc) with ``docaddr = (segment_ord << 32) + doc`` (reader.rs:310, Q13).

Tokenisation mirrors tantivy's "default" analyzer (SimpleTokenizer + RemoveLongFilter(40) + LowerCaser)
[recalled]; fuzzy fallback, filters and stop words are query-preparation, outside the hot path.

Facets (tantivy's ``FacetCollector``, run beside ``Count`` and ``TopDocs``: nidx_text/src/reader.rs:388-450,
nidx_paragraph/src/reader.rs:252-347) ARE on the hot path: a facet count visits every matched document, so it is counted inside
the BM25 pass (``bm25_facet_kernel``), and over every alive document for an empty body (``facet_count_all_kernel``).  The index
keeps ONE facet dictionary across its segments (like the term vocabulary), so per-segment bucket counts add up as arrays before the
top-50 cut of ``FacetCounts::top_k`` (nidx_text/src/reader.rs:43-62).  Each group lists its children by count descending, ties in
facet order (path segments compared bytewise); a group without a counted child is omitted.

Order by date (``SearchRequest.order``: ``TopDocs::order_by_fast_field("created" | "modified")`` in place of ``order_by_score``,
nidx_text/src/reader.rs:208-287, nidx_paragraph/src/reader.rs:229-243) is on the hot path too: every matched document is offered to
the top-k with its date (``bm25_order_kernel``), and an empty body lists every alive document (``date_topk_all_kernel``).  Dates are
seconds, results carry ``date`` instead of ``score``, ``min_score`` and search-after do not apply, and ``next_page = total > k``.
Segments are merged by (date in the requested direction, undated documents last, segment ord, doc): the tie order and the place of
undated documents are fixed here, not taken from the reference.

Security (``SearchRequest.security``: ``security_query``, nidx_text/src/search_query.rs:63-87) is a document mask: a resource's access
groups are indexed as a facet column (a group id gets a leading '/' when it lacks one; a resource without groups is public), the
request's groups compile to OR(public, each group's facet range) and run on the prefilter's evaluator, and the keyword passes run on
``nidx_txt_view``s of the segments under the resulting bits: totals, next page, facet counts and date listings all come from the masked
passes.  It filters only: BM25 scores are the body's (the reference also adds the security clause's own score).
"""
from __future__ import annotations

import re
import unicodedata
import uuid as _uuid_mod
from dataclasses import dataclass, field
from typing import Optional, Sequence

import numpy as np

from . import _lib
from .segment import TextSegment

_TOKEN = re.compile(r"[^\W_]+", re.UNICODE)


def tokenize(text: str) -> list:
    """tantivy's "default" analyzer [recalled]: SimpleTokenizer (alphanumeric runs) -> RemoveLongFilter::limit(40), which keeps a
    token iff `token.text.len() < 40` -- a length in UTF-8 BYTES, strictly below the limit -- -> LowerCaser."""
    return [t.lower() for t in _TOKEN.findall(text) if len(t.encode("utf-8")) < 40]


def tokenize_with_positions(text: str) -> list:
    """tokenize() with every token's position: its index in the SimpleTokenizer stream BEFORE RemoveLongFilter, so a dropped long
    token leaves a gap that a phrase does not match across [recalled].  -> [(position, token)]."""
    return [(i, t.lower()) for i, t in enumerate(_TOKEN.findall(text)) if len(t.encode("utf-8")) < 40]


# Rust's char::is_whitespace (Unicode White_Space) and nom's multispace0 (ASCII space, tab, CR, LF only)
_WHITE_SPACE = frozenset("\t\n\x0b\x0c\r \x85\xa0\u1680\u2000\u2001\u2002\u2003\u2004\u2005\u2006\u2007\u2008\u2009\u200a"
                         "\u2028\u2029\u202f\u205f\u3000")
_MULTISPACE = frozenset(" \t\r\n")


def _is_literal_char(c: str) -> bool:
    return c != '"' and c not in _WHITE_SPACE and unicodedata.category(c) != "Cc"


def _grammar(body: str):
    """nidx_paragraph's query grammar (query_parser/tokenizer.rs:68-127): [(kind, text)] with kind "L" literal, "Q" quoted,
    "E" excluded (-word), or None on a parse error (a character no rule takes, such as U+00A0 outside quotes)."""
    n = len(body)

    def ms(i):
        while i < n and body[i] in _MULTISPACE:
            i += 1
        return i

    def word(i):
        while i < n and _is_literal_char(body[i]):
            i += 1
        return i

    out, i = [], ms(0)
    while i < n:
        j = ms(i)
        if j < n and body[j] == '"' and (k := body.find('"', j + 1)) > j + 1:   # "..." (at least one character inside)
            text = body[j + 1:k]
            if any(c not in _WHITE_SPACE for c in text):                       # quotes around whitespace only are dropped
                out.append(("Q", text))
            i = ms(k + 1)
        elif body[i] == '"':                                                    # an unclosed quote (or "") is dropped
            while i < n and body[i] == '"':
                i += 1
        elif j < n and body[j] == "-" and word(j + 1) > j + 1:
            k = word(j + 1)
            out.append(("E", body[j + 1:k]))
            i = ms(k)
        elif word(j) > j:
            k = word(j)
            out.append(("L", body[j:k]))
            i = ms(k)
        else:
            return None
    return out


def paragraph_query_tokens(body: str) -> list:
    """tokenize_query_infallible (query_parser/tokenizer.rs:48-186): the grammar's tokens retokenized by SimpleTokenizer +
    LowerCaser -> [(kind, text)], a quoted group's words joined by one space; a parse error reads the whole body as one literal."""
    tokens = _grammar(body)
    out = []
    for kind, text in tokens if tokens is not None else [("L", body)]:
        words = [t.lower() for t in _TOKEN.findall(text)]
        if kind == "Q":
            if words:
                out.append(("Q", " ".join(words)))
        else:
            out += [(kind, w) for w in words]
    return out


def parse_paragraph_query(body: str):
    """paragraph_query_tokens + parse_keyword_query's clauses (keyword_parser.rs:27-91) -> (literal words, phrases as word lists).
    Literals (and excluded words, searched as literals here) are exactly tokenize()'s words; a quoted group of two or more words is
    a phrase (no word dropped: a long word is a term the index does not hold, so the phrase matches nothing), of one word a
    literal.  A parse error reads the whole body as literals."""
    tokens = _grammar(body)
    if tokens is None:
        return tokenize(body), []
    words, phrases = [], []
    for kind, text in tokens:
        if kind == "Q":
            ws = [t.lower() for t in _TOKEN.findall(text)]
            if len(ws) >= 2:
                phrases.append(ws)
                continue
        words += tokenize(text)
    return words, phrases


def fieldnorm_to_id(n: int) -> int:
    """tantivy's 1-byte fieldnorm code (Lucene SmallFloat.intToByte4) [recalled]."""
    if n < 24:
        return n
    x = n - 24
    nbits = x.bit_length()
    if nbits <= 3:
        return 24 + x
    shift = nbits - 4
    enc = ((x >> shift) & 7) | ((shift + 1) << 3)
    return min(255, 24 + enc)


@dataclass
class ResultScore:  # nodereader.proto:48-53
    bm25: float
    docaddr: int


@dataclass
class DocumentResult:
    uuid: str
    field: str
    score: Optional[ResultScore]
    labels: list
    date: Optional[int] = None   # seconds: the sort value under an order (nodereader.proto DocumentResult.date), None without a date


@dataclass
class OrderBy:  # nodereader.proto OrderBy
    sort_by: int = _lib.NIDX_ORDER_CREATED   # OrderField: CREATED 0, MODIFIED 1
    type: int = _lib.NIDX_ORDER_DESC          # OrderType: DESC 0, ASC 1


@dataclass
class DocumentSearchRequest:  # nidx_text/src/request_types.rs:17-28
    body: str = ""
    result_per_page: int = 20
    min_score: float = 0.0
    only_faceted: bool = False
    faceted: Sequence[str] = ()               # Faceted.labels: the facets to count children of (SearchRequest.faceted)
    search_after: Optional[SearchAfter] = None  # ParagraphSearchRequest.search_after (nidx_paragraph only)
    order: Optional[OrderBy] = None            # SearchRequest.order: results by date instead of score
    security: Optional[Sequence[str]] = None   # SearchRequest.security.access_groups: only public resources and those of these groups


@dataclass
class SearchAfter:  # nidx_paragraph/src/request_types.rs:20-31
    score: float
    tie_break: str = "drop"   # "drop" | "keep" | "keep_after"
    docaddr: int = 0          # payload of KeepAfter


@dataclass
class FacetResult:  # nodereader.proto:40-43
    tag: str
    total: int


@dataclass
class DocumentSearchResponse:
    results: list = field(default_factory=list)
    total: int = 0
    next_page: bool = False
    query: str = ""
    facets: dict = field(default_factory=dict)   # request facet -> [FacetResult], top 50 (nodereader.proto:74, 115)


FACET_TOP_K = 50   # FacetCounts::top_k(facet, 50): nidx_text/src/reader.rs:43-52, nidx_paragraph/src/search_response.rs:48-57


def facet_key(path: str) -> Optional[bytes]:
    """tantivy's encoded facet (segments joined by 0x00, no leading '/'; the root "/" is b""), or None when the string is not a
    valid facet (Facet::from_text fails [recalled]: it must start with '/')."""
    if not path.startswith("/"):
        return None
    return b"" if path == "/" else path[1:].encode("utf-8").replace(b"/", b"\0")


def group_key(group: str) -> bytes:
    """An access group id as the group column holds it: a facet, with a leading '/' added when the id lacks one
    (nidx_text/src/resource_indexer.rs:49-62, search_query.rs:63-87)."""
    return facet_key(group if group.startswith("/") else "/" + group)


def facet_path(key: bytes) -> str:
    return "/" + key.replace(b"\0", b"/").decode("utf-8")


def _facet_request(faceted: Sequence[str]):
    """Faceted.labels -> the valid facets, duplicates collapsed, in request order (is_valid_facet / Facet::from_text(..).ok())."""
    out = []
    for f in faceted:
        if facet_key(f) is not None and f not in out:
            out.append(f)
    return out


@dataclass
class TextDoc:
    uuid: str
    field: str
    text: str
    labels: Sequence[str] = ()
    created: Optional[int] = None    # IndexMetadata.created / .modified, seconds
    modified: Optional[int] = None
    groups: Sequence[str] = ()       # Resource.security.access_groups; none = public
    repeated: bool = False           # IndexParagraph.repeated_in_field (paragraph documents): Suggest skips it
    paragraph: Optional[tuple] = None   # (paragraph id, IndexParagraph) of a paragraph document, for Suggest's results


class TextIndexSegment:
    """One immutable segment: term dictionary + postings (host build, HBM resident)."""

    def __init__(self, docs: Sequence[TextDoc], vocab: dict, device=0):
        self.docs = list(docs)
        toks = [[vocab.setdefault(t, len(vocab)) for t in tokenize(d.text)] for d in self.docs]
        self.n_docs = len(self.docs)
        self.lens = np.asarray([len(t) for t in toks], dtype=np.int64)
        self.total_tokens = int(self.lens.sum())
        pairs = sorted({(t, i) for i, ts in enumerate(toks) for t in ts})
        tf = {}
        for i, ts in enumerate(toks):
            for t in ts:
                tf[(t, i)] = tf.get((t, i), 0) + 1
        self.n_terms = len(vocab)
        self.post_term = np.asarray([p[0] for p in pairs], dtype=np.int64)
        self.post_doc = np.asarray([p[1] for p in pairs], dtype=np.uint32)
        self.post_tf = np.asarray([tf[p] for p in pairs], dtype=np.uint32)
        self.fieldnorm_id = np.asarray([fieldnorm_to_id(int(x)) for x in self.lens], dtype=np.uint8)
        pos: dict = {}
        for i, d in enumerate(self.docs):
            for p, t in tokenize_with_positions(d.text):
                pos.setdefault((vocab[t], i), []).append(p)
        # every posting's positions, in posting order (nidx_txt_set_positions); uploaded on the first phrase query
        self.positions = np.asarray([p for pr in pairs for p in pos[pr]], dtype=np.uint32)
        self._gpu: Optional[TextSegment] = None
        self.device = device

    def doc_freq(self, n_terms: int) -> np.ndarray:
        return np.bincount(self.post_term, minlength=n_terms).astype(np.uint64)

    def upload(self, n_terms: int):
        term_off = np.zeros(n_terms + 1, dtype=np.uint64)
        term_off[1:] = np.cumsum(np.bincount(self.post_term, minlength=n_terms))
        self._gpu = TextSegment.create(self.n_docs, n_terms, term_off, self.post_doc, self.post_tf, self.fieldnorm_id, device=self.device)
        self.alive_count = self.n_docs
        return self._gpu

    def set_alive(self, alive: np.ndarray):
        """Deletions inside the segment: a bool per document (nidx_txt_set_alive).  The prefilter counts the alive documents for its
        All class."""
        alive = np.asarray(alive, dtype=bool)
        words = np.zeros((self.n_docs + 63) // 64 * 8, dtype=np.uint8)
        packed = np.packbits(alive, bitorder="little")
        words[: len(packed)] = packed
        self._gpu.set_alive(words.view(np.uint64))
        self.alive_count = int(alive.sum())


class TextSearcher:
    """nidx_text TextSearcher over one or more segments sharing one term dictionary (and one facet dictionary)."""

    conjunction = True   # QueryParser::set_conjunction_by_default (reader.rs:372-377)
    use_tf = True

    def __init__(self, segments: Sequence[TextIndexSegment], vocab: dict):
        _lib.require_device()
        self.segments, self.vocab = list(segments), vocab
        n_terms = len(vocab)
        total_docs = sum(s.n_docs for s in self.segments)
        total_tokens = sum(s.total_tokens for s in self.segments)
        df = np.zeros(n_terms, dtype=np.uint64)
        for s in self.segments:
            df += s.doc_freq(n_terms)
        for s in self.segments:  # union statistics on every segment (index_reader.rs:39-77)
            s.upload(n_terms).set_stats(max(total_docs, 1), max(total_tokens, 1), df)
        self.facet_keys: Optional[list] = None   # built on the first faceted request
        self.group_keys: Optional[list] = None   # built on the first request with security
        self._dates = False                        # uploaded on the first ordered request
        self._prefilter: Optional[_PrefilterIndex] = None   # built on the first prefilter
        self._positions = False                    # uploaded on the first phrase (query or keyword filter)

    def _ensure_facets(self):
        """The index's facet dictionary (every valid label of every document, in facet order) and each segment's per-document
        ords, uploaded once."""
        if self.facet_keys is not None:
            return
        keys = sorted({k for s in self.segments for d in s.docs for k in map(facet_key, d.labels) if k is not None})
        ord_of = {k: i for i, k in enumerate(keys)}
        for s in self.segments:
            rows = [sorted({ord_of[k] for k in map(facet_key, d.labels) if k is not None}) for d in s.docs]
            off = np.zeros(len(rows) + 1, dtype=np.uint64)
            off[1:] = np.cumsum([len(r) for r in rows])
            s._gpu.set_facets(keys, off, np.asarray([o for r in rows for o in r], dtype=np.uint32))
        self.facet_keys = keys

    def _ensure_groups(self):
        """The index's access group dictionary (group_key of every document's groups, in facet order) and each segment's
        per-document group ords, uploaded once."""
        if self.group_keys is not None:
            return
        keys = sorted({group_key(g) for s in self.segments for d in s.docs for g in d.groups})
        ord_of = {k: i for i, k in enumerate(keys)}
        for s in self.segments:
            rows = [sorted({ord_of[group_key(g)] for g in d.groups}) for d in s.docs]
            off = np.zeros(len(rows) + 1, dtype=np.uint64)
            off[1:] = np.cumsum([len(r) for r in rows])
            s._gpu.set_doc_groups(keys, off, np.asarray([o for r in rows for o in r], dtype=np.uint32))
        self.group_keys = keys

    def security_nodes(self, access_groups: Sequence[str]) -> list:
        """security_tree over this index's group dictionary."""
        self._ensure_groups()
        return security_tree(self.group_keys, access_groups)

    def _security_bits(self, access_groups: Sequence[str]) -> list:
        """Per segment, the security expression's bits (nidx_txt_prefilter), in HBM."""
        import torch

        nodes = _node_array(self.security_nodes(access_groups))
        out = []
        for s in self.segments:
            out.append(torch.empty(max((s.n_docs + 63) // 64, 1), dtype=torch.int64, device=torch.device("cuda", s.device)))
            s._gpu.prefilter(nodes, out=out[-1])
        return out

    def _security_views(self, access_groups: Sequence[str]) -> list:
        """Every segment as a view (nidx_txt_view) under the security expression's bits, which stay on the device."""
        views = []
        try:
            for s, bits in zip(self.segments, self._security_bits(access_groups)):
                views.append(s._gpu.view(bits))
        except BaseException:
            for v in views:
                v.close()
            raise
        return views

    def _ensure_dates(self):
        """Every segment's created / modified seconds, uploaded once."""
        if self._dates:
            return
        none = _lib.NIDX_DATE_NONE
        for s in self.segments:
            s._gpu.set_dates(np.asarray([none if d.created is None else int(d.created) for d in s.docs], dtype=np.int64),
                             np.asarray([none if d.modified is None else int(d.modified) for d in s.docs], dtype=np.int64))
        self._dates = True

    def _ensure_positions(self):
        if not self._positions:
            for s in self.segments:
                s._gpu.set_positions(s.positions)
            self._positions = True

    def prefilter(self, expr, security: Optional[Sequence[str]] = None):
        """TextReaderService::prefilter (nidx_text/src/reader.rs:147-180) for a nodereader.FilterExpression and / or the access groups
        of SearchRequest.security (both given: their intersection, in one program; expr may then be None): evaluated on the device
        over every segment -> vector.PrefilterResult: none (nothing matched), all (every alive document matched) or some, whose
        matched documents stay in HBM as a bitset (handed to VectorSearcher.search as they are; `fields` lists them on demand).
        A malformed expression, an invalid facet or resource UUID, or one the device cannot run (deeper than
        NIDX_PREFILTER_MAX_DEPTH, a keyword of more than 64 words) is a ValueError."""
        import torch

        from . import vector as V
        from ._lib import NidxError

        self._ensure_facets()
        self._ensure_dates()
        if self._prefilter is None:
            self._prefilter = _PrefilterIndex(self)
        ix = self._prefilter
        nodes, keep, phrases = ix.compile(expr, None if security is None else self.security_nodes(security))
        if phrases:
            self._ensure_positions()
        bits = torch.empty(ix.words_total, dtype=torch.int64, device=torch.device("cuda", self.segments[0].device))
        matching = 0
        try:
            for s, off in zip(self.segments, ix.word_off):
                matching += s._gpu.prefilter(nodes, out=bits[off: off + (s.n_docs + 63) // 64])[1]
        except NidxError as e:
            if e.code == -1:   # NIDX_EINVAL: the expression is not one the device runs
                raise ValueError(str(e)) from e
            raise
        if matching == 0:
            return V.PrefilterResult.none()
        if matching == sum(s.alive_count for s in self.segments):
            return V.PrefilterResult.all()
        return V.PrefilterResult.from_device(ix, bits, matching)

    def _facets(self, handles: list, faceted: Sequence[str], terms, k: int, params: dict, order: Optional[OrderBy] = None, phrases=()):
        """Counts of the request's facets over the matched set of every segment, summed, then grouped and cut to the top 50.
        With terms: the faceted BM25 search, ordered by date when `order` is given (returns its per-segment (docs, scores or
        dates, counts, total) too); without: every alive document (AllQuery)."""
        from ._lib import NidxError

        request = _facet_request(faceted)
        self._ensure_facets()
        keys = [facet_key(f) for f in request]
        try:
            b_req, b_ord = self.segments[0]._gpu.facet_buckets(keys)
        except NidxError as e:
            if e.code == -1:   # NIDX_EINVAL: one requested facet is an ancestor of another (tantivy asserts)
                raise ValueError(str(e)) from e
            raise
        counts = np.zeros(len(b_req), dtype=np.int64)
        hits = []
        for ord_, seg in enumerate(handles):
            if terms or phrases:
                qt, qo = np.asarray(terms, dtype=np.uint32), np.asarray([0, len(terms)], dtype=np.uint32)
                if phrases:
                    docs, scores, cnt, total, fc = seg.search_phrases(qt, qo, [(0, p) for p in phrases], k, docaddr_base=ord_ << 32, facets=keys,
                                                                           order=None if order is None else (order.sort_by, order.type), **params)
                elif order is not None:
                    docs, scores, cnt, total, fc = seg.search_ordered(qt, qo, k, order.sort_by, order.type, params["mode"], facets=keys)
                else:
                    docs, scores, cnt, total, fc = seg.search_faceted(qt, qo, k, keys, docaddr_base=ord_ << 32, **params)
                hits.append((docs, scores, cnt, total))
                counts += fc[0]
            else:
                counts += seg.facet_count_all(keys)
        groups: dict = {}
        for b, (r, o) in enumerate(zip(b_req, b_ord)):
            if counts[b]:
                depth = 0 if keys[r] == b"" else keys[r].count(b"\0") + 1
                child = b"\0".join(self.facet_keys[o].split(b"\0")[: depth + 1])
                groups.setdefault(int(r), []).append((-int(counts[b]), child))
        facets = {}
        for r in sorted(groups):
            facets[request[r]] = [FacetResult(facet_path(c), -n) for n, c in sorted(groups[r])[:FACET_TOP_K]]
        return facets, hits

    @classmethod
    def open(cls, docs_per_segment: Sequence[Sequence[TextDoc]], device=0):
        vocab: dict = {}
        segs = [TextIndexSegment(d, vocab, device) for d in docs_per_segment]
        return cls(segs, vocab)

    def _terms(self, body: str):
        terms = []
        for t in tokenize(body):
            terms.append(self.vocab.get(t, 0xFFFFFFF0))  # unknown term: matches nothing
        return terms

    def _clauses(self, body: str):
        """-> (term ids, phrases as term-id lists).  nidx_text's QueryParser grammar is not restated: no phrases."""
        return self._terms(body), []

    def _json_joins(self, text_index, json_index) -> list:
        """Per segment, on the device: (doc_join, res_join), each document's bit in the text prefilter's output (text_index: the
        shard's text _PrefilterIndex; NIL without a text document of its field) and its resource's ord in json_index.resource_ids
        (NIL: none).  Each half is built once per (this searcher, text_index / json_index), vectorised, and kept in HBM."""
        import torch

        def lookup(keys_sorted, values, queries):
            if len(keys_sorted) == 0:
                return np.full(len(queries), _lib.NIL, dtype=np.uint32)
            at = np.minimum(np.searchsorted(keys_sorted, queries), len(keys_sorted) - 1)
            return np.where(keys_sorted[at] == queries, values[at], _lib.NIL).astype(np.uint32)

        dev = torch.device("cuda", self.segments[0].device)
        up = lambda a: torch.from_numpy(a.view(np.int32)).to(dev)   # noqa: E731
        if getattr(self, "_res_join", None) is None or self._res_join[0] is not json_index:
            rids = np.asarray(json_index.resource_ids if json_index is not None else [], dtype=str)
            self._res_join = (json_index, [up(lookup(rids, np.arange(len(rids), dtype=np.uint32), np.asarray([d.uuid for d in s.docs], dtype=str)))
                                           for s in self.segments])
        if text_index is not None and (getattr(self, "_doc_join", None) is None or self._doc_join[0] is not text_index):
            keys = np.concatenate([np.asarray([d.uuid + "\x01" + d.field for d in ts.docs], dtype=str) for ts in text_index.searcher.segments])
            pos = np.concatenate([64 * off + np.arange(ts.n_docs, dtype=np.uint64) for ts, off in zip(text_index.searcher.segments, text_index.word_off)])
            keys, first = np.unique(keys, return_index=True)   # a field's first document, as a dict's setdefault would keep
            self._doc_join = (text_index, [up(lookup(keys, pos[first].astype(np.uint32), np.asarray([d.uuid + "\x01" + d.field for d in s.docs], dtype=str)))
                                           for s in self.segments])
        return [(self._doc_join[1][i] if text_index is not None else None, self._res_join[1][i]) for i in range(len(self.segments))]

    def json_masks(self, security: Optional[Sequence[str]], prefilter) -> list:
        """The per-segment masks of a search under SearchRequest.json_filter (nidx_txt_join_mask, on the device) for a Some on the
        device (vector.PrefilterResult): bit d = the security bits (when `security` is given) AND op(the text part's bit of the
        document's field (no text part: every field), the resource part's bit of its resource (no resource part: none)), op OR when
        the result's op_or or when it has no resource part."""
        import torch

        text_index, text_bits, _ = prefilter.device_bits or (None, None, 0)
        json_index, res_bits = prefilter.resources or (None, torch.zeros(1, dtype=torch.int64, device=torch.device("cuda", self.segments[0].device)))
        n_res = len(json_index.resource_ids) if json_index is not None else 0
        op = _lib.NIDX_F_OR if prefilter.op_or or prefilter.resources is None else _lib.NIDX_F_AND
        sec = self._security_bits(security) if security is not None else [None] * len(self.segments)
        masks = []
        for s, and_bits, (doc_join, res_join) in zip(self.segments, sec, self._json_joins(text_index, json_index)):
            mask, _ = s._gpu.join_mask(and_bits, text_bits, 0 if text_bits is None else text_bits.numel() * 64, doc_join, res_bits, n_res, res_join, op)
            masks.append(mask)
        return masks

    def search(self, request: DocumentSearchRequest, masks: Optional[list] = None) -> DocumentSearchResponse:
        """masks (one device bitset per segment, as json_masks makes them) replace the security mask: the search runs on views
        under them."""
        if request.security is None and masks is None:
            return self._search(request, [s._gpu for s in self.segments])
        views = self._security_views(request.security) if masks is None else [s._gpu.view(m) for s, m in zip(self.segments, masks)]
        try:
            return self._search(request, views)
        finally:
            for v in views:
                v.close()

    def _search(self, request: DocumentSearchRequest, handles: list) -> DocumentSearchResponse:
        """search() over one handle per segment: the segments themselves, or their views under a security mask."""
        terms, phrases = self._clauses(request.body)
        k = request.result_per_page
        resp = DocumentSearchResponse(query=request.body)
        after = None
        if request.search_after is not None:
            sa = request.search_after
            after = (sa.score, {"drop": 1, "keep_after": 2, "keep": 3}[sa.tie_break], sa.docaddr)
        params = dict(mode=_lib.NIDX_BM25_AND if self.conjunction else _lib.NIDX_BM25_OR, use_tf=self.use_tf, min_score=0.0, after=after)
        if request.order is not None and not request.only_faceted:   # only_faceted comes first (nidx_text/src/reader.rs:405-414)
            return self._search_ordered(request, handles, terms, params, phrases)
        hits = None
        if _facet_request(request.faceted):
            resp.facets, hits = self._facets(handles, request.faceted, terms, max(k, 0) + 1, params, phrases=phrases)
        if request.only_faceted:   # only the facets: no results, total 0 (nidx_text/src/reader.rs:407-414, search_response.rs:111-124)
            return DocumentSearchResponse(facets=resp.facets)
        if not (terms or phrases) or k <= 0:
            return resp
        qt = np.asarray(terms, dtype=np.uint32)
        qo = np.asarray([0, len(terms)], dtype=np.uint32)
        merged = []
        for ord_, seg in enumerate(handles):
            if hits is not None:   # the faceted pass already returned this segment's top-k and Count
                docs, scores, counts, total = hits[ord_]
            elif phrases:
                docs, scores, counts, total = seg.search_phrases(qt, qo, [(0, p) for p in phrases], k + 1, docaddr_base=ord_ << 32, **params)
            else:
                docs, scores, counts, total = seg.search(qt, qo, k + 1, docaddr_base=ord_ << 32, **params)
            resp.total += int(total[0])
            merged += [(-float(scores[0, i]), ord_, int(docs[0, i])) for i in range(int(counts[0]))]
        merged.sort()  # score desc, then segment_ord, then doc: lower docaddr first
        resp.next_page = len(merged) > k  # reader.rs:300-301
        for neg, ord_, doc in merged[:k]:
            score = -neg
            if score < request.min_score:  # reader.rs:302-305
                continue
            d = self.segments[ord_].docs[doc]
            resp.results.append(DocumentResult(d.uuid, d.field, ResultScore(score, (ord_ << 32) + doc), list(d.labels)))
        return resp


    def _search_ordered(self, request: DocumentSearchRequest, handles: list, terms, params: dict, phrases=()) -> DocumentSearchResponse:
        """TopDocs(k + 1) ordered by date beside Count (and the FacetCollector) in one pass per segment; an empty body lists every
        alive document.  convert_int_order (nidx_text/src/reader.rs:226-287): no min_score, next_page = total > k."""
        order, k = request.order, request.result_per_page
        resp = DocumentSearchResponse(query=request.body)
        self._ensure_dates()
        hits = None
        if _facet_request(request.faceted):
            resp.facets, hits = self._facets(handles, request.faceted, terms, max(k, 0) + 1, params, order=order, phrases=phrases)
        if k <= 0:
            return resp
        qt, qo = np.asarray(terms, dtype=np.uint32), np.asarray([0, len(terms)], dtype=np.uint32)
        rows = []
        for ord_, seg in enumerate(handles):
            if not (terms or phrases):
                docs, dates, count, total = seg.list_ordered(k + 1, order.sort_by, order.type)
            else:
                if hits is not None:
                    d2, t2, c2, tot2 = hits[ord_]
                elif phrases:
                    d2, t2, c2, tot2 = seg.search_phrases(qt, qo, [(0, p) for p in phrases], k + 1, mode=params["mode"], order=(order.sort_by, order.type))
                else:
                    d2, t2, c2, tot2 = seg.search_ordered(qt, qo, k + 1, order.sort_by, order.type, params["mode"])
                docs, dates, count, total = d2[0], t2[0], int(c2[0]), int(tot2[0])
            resp.total += int(total)
            rows += [(date_sort_key(int(dates[i]), order.type), ord_, int(docs[i]), int(dates[i])) for i in range(count)]
        rows.sort()   # date in the requested direction (undated last), then segment ord, then doc
        resp.next_page = resp.total > k
        for _, ord_, doc, date in rows[:k]:
            d = self.segments[ord_].docs[doc]
            resp.results.append(DocumentResult(d.uuid, d.field, None, list(d.labels), None if date == _lib.NIDX_DATE_NONE else date))
        return resp


_I64_MIN, _I64_MAX = -(1 << 63), (1 << 63) - 1


def _prefix_range(keys: list, prefix: bytes, facet: bool):
    """[lo, hi) of the sorted byte keys that start with `prefix`; facet=True: the facet `prefix` and its descendants (the key itself
    or prefix + 0x00 ...; the root b"" takes every key)."""
    import bisect

    lo = bisect.bisect_left(keys, prefix)
    if facet and prefix:
        return lo, bisect.bisect_left(keys, prefix + b"\x01")
    stem = prefix.rstrip(b"\xff")   # the least byte string above every key that starts with `prefix`
    return lo, bisect.bisect_left(keys, stem[:-1] + bytes([stem[-1] + 1])) if stem else len(keys)


def security_tree(group_keys: list, access_groups: Sequence[str]) -> list:
    """security_query (nidx_text/src/search_query.rs:63-87) as flat pre-order prefilter nodes (kind, n, lo, hi, terms) over a group
    dictionary (the sorted group_key of every group): OR of PUBLIC and, per requested group, the GROUP range of that group and its
    descendants.  No groups: public resources only."""
    flat = [(_lib.NIDX_P_OR, 1 + len(access_groups), 0, 0, None), (_lib.NIDX_P_PUBLIC, 0, 0, 0, None)]
    return flat + [(_lib.NIDX_P_GROUP, 0, *_prefix_range(group_keys, group_key(g), facet=True), None) for g in access_groups]


def _node_array(flat: list):
    """Flat pre-order nodes (kind, n, lo, hi, terms) -> the ctypes nidx_prefilter_node array."""
    nodes = (_lib.PrefilterNode * len(flat))()
    for i, (kind, n, lo, hi, terms) in enumerate(flat):
        nodes[i].kind, nodes[i].n, nodes[i].lo, nodes[i].hi, nodes[i].terms = kind, n, lo, hi, terms
    return nodes


class _PrefilterIndex:
    """What the prefilter of one TextSearcher keeps on the host (built on the first prefilter, once per searcher open): the
    dictionaries of resource ids and field paths -- field paths in facet order, so that a field filter (a facet term on
    `schema.field`) and a resource_field_prefix are ranges of ords -- every segment's columns (uploaded with
    nidx_txt_set_doc_columns), where each segment's documents start in the index-wide bitset (whole 64-bit words), and the join
    tables to vector segments (one u32 per document of that bitset, in HBM, built on the first hand-off to each)."""

    def __init__(self, searcher: "TextSearcher"):
        import weakref

        self.searcher = searcher
        docs = [d for s in searcher.segments for d in s.docs]
        self.resource_ids, res_ord = np.unique(np.asarray([d.uuid for d in docs], dtype=object).astype(str), return_inverse=True) if docs else ([], [])
        paths = sorted({d.field for d in docs}, key=lambda p: facet_key(p) if p.startswith("/") else b"\xff" + p.encode())
        self.field_paths = paths
        self.field_keys = [facet_key(p) if p.startswith("/") else b"\xff" + p.encode() for p in paths]   # a path without '/' is no facet: matches no filter
        field_of = {p: i for i, p in enumerate(paths)}
        fld_ord = np.asarray([field_of[d.field] for d in docs], dtype=np.uint32)
        res_ord = np.asarray(res_ord, dtype=np.uint32)
        self.word_off, at, words = [], 0, 0
        self.doc_base = np.zeros(len(searcher.segments) + 1, dtype=np.int64)
        for i, s in enumerate(searcher.segments):
            s._gpu.set_doc_columns(res_ord[at: at + s.n_docs], fld_ord[at: at + s.n_docs])
            self.word_off.append(words)
            words += (s.n_docs + 63) // 64
            at += s.n_docs
        self.words_total = words
        self.res_col, self.field_col = res_ord, fld_ord
        self.by_uuid: dict = {}   # parsed UUID bytes -> resource ords (several spellings of one UUID are several ids)
        for o, r in enumerate(self.resource_ids):
            try:
                self.by_uuid.setdefault(_uuid_mod.UUID(r).bytes, []).append(o)
            except ValueError:
                pass
        self._joins = weakref.WeakKeyDictionary()

    # ---- filter_to_query (nidx_text/src/search_query.rs:156-217) -> nidx_prefilter_node, pre-order ---------------------------------
    def compile(self, expr, security: Optional[list] = None):
        """-> (ctypes PrefilterNode array, keep-alive list, whether a phrase is used).  security: flat nodes
        (TextSearcher.security_nodes) ANDed with expr; expr may then be None."""
        flat, keep = [], []
        if security is not None:
            if expr is not None:
                flat.append((_lib.NIDX_P_AND, 2, 0, 0, None))
            flat += security
        phrases = False
        vocab = self.searcher.vocab

        def node(kind, n=0, lo=0, hi=0, terms=None):
            flat.append((kind, n, lo, hi, terms))

        def walk(e):
            nonlocal phrases
            kind = e.WhichOneof("expr")
            if kind in ("bool_and", "bool_or"):
                ops = getattr(e, kind).operands
                node(_lib.NIDX_P_AND if kind == "bool_and" else _lib.NIDX_P_OR, len(ops))
                for o in ops:
                    walk(o)
            elif kind == "bool_not":
                node(_lib.NIDX_P_NOT, 1)
                walk(e.bool_not)
            elif kind == "facet":
                key = facet_key(e.facet.facet)
                if key is None:   # Facet::from asserts a leading '/' [recalled]: the reference fails the request
                    raise ValueError(f"invalid facet {e.facet.facet!r}: a facet starts with '/'")
                node(_lib.NIDX_P_FACET, 0, *_prefix_range(self.searcher.facet_keys, key, facet=True))
            elif kind == "field":
                f = e.field
                path = f"/{f.field_type}/{f.field_id}" if f.HasField("field_id") else f"/{f.field_type}"
                node(_lib.NIDX_P_FIELD, 0, *_prefix_range(self.field_keys, facet_key(path), facet=True))
            elif kind == "resource":
                rid = e.resource.resource_id
                o = int(np.searchsorted(self.resource_ids, rid)) if len(self.resource_ids) else 0
                hit = o < len(self.resource_ids) and self.resource_ids[o] == rid
                node(_lib.NIDX_P_RESOURCE, 0, o, o + 1 if hit else o)
            elif kind == "resource_field_prefix":
                p = e.resource_field_prefix
                try:
                    rb = _uuid_mod.UUID(p.resource_id).bytes
                except ValueError as err:   # uuid::Uuid::parse_str(..).expect(..): the reference panics
                    raise ValueError(f"resource_field_prefix: invalid resource id {p.resource_id!r}") from err
                ords = self.by_uuid.get(rb, [])
                prefix = facet_key(f"/{p.field_type}/{p.field_id_prefix}")
                node(_lib.NIDX_P_AND, 2)
                node(_lib.NIDX_P_OR, len(ords))
                for o in ords:
                    node(_lib.NIDX_P_RESOURCE, 0, o, o + 1)
                node(_lib.NIDX_P_FIELD, 0, *_prefix_range(self.field_keys, prefix, facet=False))
            elif kind == "date":
                d = e.date
                since = d.since.seconds if d.HasField("since") else None
                until = d.until.seconds if d.HasField("until") else None
                if since is None and until is None:   # produce_date_range_query -> None: AllQuery
                    node(_lib.NIDX_P_ALL)
                else:
                    node(_lib.NIDX_P_DATE, int(d.field), _I64_MIN if since is None else since, _I64_MAX if until is None else until)
            elif kind == "keyword":   # translate_keyword_to_text_query (query_io.rs:22-42)
                words = tokenize(e.keyword.keyword) or [e.keyword.keyword]
                if len(words) > 64:
                    raise ValueError("a keyword filter of more than 64 words is not supported")
                phrases = phrases or len(words) > 1
                ids = np.asarray([vocab.get(w, 0xFFFFFFF0) for w in words], dtype=np.uint32)   # an unknown word matches nothing
                keep.append(ids)
                node(_lib.NIDX_P_KEYWORD, len(ids), terms=ids.ctypes.data)
            else:
                raise ValueError(f"filter expression without a known expression: {kind!r}")

        if expr is not None:
            walk(expr)
        return _node_array(flat), keep, phrases

    # ---- hand-off to the vector index ---------------------------------------------------------------------------------------
    def n_docs_total(self) -> int:
        return 64 * self.words_total

    def join(self, seg):
        """The join table to one vector OpenSegment (torch int32 [64 * words_total] on the device): for every document of the
        index-wide bitset, its key in the segment's field index -- the key that FieldId(resource, field) looks up there
        (searcher.rs:300-314: `{uuid.hex}{field}` through FieldKey) -- or NIL."""
        j = self._joins.get(seg)
        if j is not None:
            return j
        import torch

        from .vector import field_key

        # (resource ord, field ord) pairs of every field key of the segment: a loop over the segment's keys, not the documents
        suffix_of: dict = {}
        for o, path in enumerate(self.field_paths):
            fk = field_key(f"{_uuid_mod.UUID(int=0).hex}{path}")
            if fk is not None:
                suffix_of.setdefault(fk[16:], []).append(o)
        n_fields = max(len(self.field_paths), 1)
        codes, vals = [], []
        for kord, key in enumerate(sorted(seg._field_index)):
            for r in self.by_uuid.get(key[:16], ()):
                for f in suffix_of.get(key[16:], ()):
                    codes.append(r * n_fields + f)
                    vals.append(kord)
        codes, vals = np.asarray(codes, dtype=np.int64), np.asarray(vals, dtype=np.uint32)
        order = np.argsort(codes, kind="stable")
        codes, vals = codes[order], vals[order]
        doc_codes = self.res_col.astype(np.int64) * n_fields + self.field_col
        table = np.full(self.n_docs_total(), _lib.NIL, dtype=np.uint32)
        if len(codes) and len(doc_codes):
            at = np.minimum(np.searchsorted(codes, doc_codes), len(codes) - 1)
            hit = codes[at] == doc_codes
            docs = np.concatenate([64 * off + np.arange(s.n_docs) for s, off in zip(self.searcher.segments, self.word_off)])
            table[docs[hit]] = vals[at[hit]]
        j = torch.from_numpy(table.view(np.int32)).to(torch.device("cuda", self.searcher.segments[0].device))
        self._joins[seg] = j
        return j

    def fields(self, bits) -> list:
        """The matched documents of an index-wide bitset as FieldId(resource, field), segment by segment (FieldUuidCollector)."""
        from .vector import FieldId

        words = bits.cpu().numpy().view(np.uint64) if hasattr(bits, "cpu") else np.asarray(bits, dtype=np.uint64)
        out = []
        for s, off in zip(self.searcher.segments, self.word_off):
            mask = np.unpackbits(words[off: off + (s.n_docs + 63) // 64].view(np.uint8), bitorder="little")[: s.n_docs].astype(bool)
            out += [FieldId(_uuid_mod.UUID(s.docs[d].uuid), s.docs[d].field) for d in np.nonzero(mask)[0]]
        return out


def date_sort_key(seconds: Optional[int], order_type: int):
    """Sort key of a date under an order: the requested direction first, documents without a date (None or NIDX_DATE_NONE) last."""
    if seconds is None or seconds == _lib.NIDX_DATE_NONE:
        return (1, 0)
    return (0, seconds if order_type == _lib.NIDX_ORDER_ASC else -seconds)


class ParagraphSearcher(TextSearcher):
    """nidx_paragraph keyword search: OR of TermQuery(Basic) => tf == 1 (keyword_parser.rs:27-67), plus a PhraseQuery per quoted
    group of two or more words (scored with its real frequency): the body is parsed by parse_paragraph_query.  suggest() is the
    paragraph pass of NidxSearcher.Suggest (nucliadb_b200/suggest.py)."""

    conjunction = False
    use_tf = False
    _suggest_dict = None   # the vocabulary in HBM (segment.SuggestDict), built on the first fuzzy pass
    _repeated = False      # repeated_in_field bits uploaded (on the first suggest)

    def suggest_masks(self, security: Optional[Sequence[str]] = None, paragraph_filter=None, prefilter=None, op_or: bool = False) -> list:
        """Per segment, on the device, the suggest mask (nidx_txt_suggest_mask): NOT repeated_in_field AND the security bits (when
        `security` is given) AND op(paragraph_filter's bits, the prefilter's), op OR when op_or, an absent operand dropped.  The
        paragraph_filter (a nodereader.FilterExpression) runs on the prefilter's evaluator over the paragraphs; the prefilter is a
        vector.PrefilterResult whose Some is on the device (joined as json_masks joins it), None or All: no operand."""
        import torch

        if not self._repeated:
            for s in self.segments:
                s._gpu.set_repeated(np.asarray([d.repeated for d in s.docs], dtype=bool))
            self._repeated = True
        dev = torch.device("cuda", self.segments[0].device)
        n = len(self.segments)
        sec = self._security_bits(security) if security is not None else [None] * n
        pf = [None] * n
        if paragraph_filter is not None:
            self._ensure_facets()
            self._ensure_dates()
            if self._prefilter is None:
                self._prefilter = _PrefilterIndex(self)
            nodes, _keep, phrases = self._prefilter.compile(paragraph_filter)
            if phrases:
                self._ensure_positions()
            pf = []
            try:
                for s in self.segments:
                    pf.append(s._gpu.prefilter(nodes, out=torch.empty(max((s.n_docs + 63) // 64, 1), dtype=torch.int64, device=dev))[0])
            except _lib.NidxError as e:
                if e.code == -1:
                    raise ValueError(str(e)) from e
                raise
        joined = self.json_masks(None, prefilter) if prefilter is not None and prefilter.kind == "some" else [None] * n
        op = _lib.NIDX_F_OR if op_or else _lib.NIDX_F_AND
        return [s._gpu.suggest_mask(a, b, c, op)[0] for s, a, b, c in zip(self.segments, sec, pf, joined)]

    def suggest(self, body: str, top_k: int, masks: list):
        """The paragraph pass of Suggest over the segments under `masks` (suggest_masks): the keyword pass (the paragraph search's query,
        its BM25 bit for bit, TopDocs(top_k)), and when it finds nothing the fuzzy pass (suggest.fuzzy_clauses, nidx_txt_suggest_fuzzy)
        -> suggest.ParagraphSuggest, hits ordered by (score desc, segment, document), each of the first RESULTS_PER_PAGE fuzzy hits with
        its matches (the sorted expanded terms of more than 2 bytes that occur in it, one per (fuzzy clause, term))."""
        from . import suggest as S

        if not 1 <= top_k <= S.MAX_TOP_K:
            raise ValueError(f"top_k must be in 1..{S.MAX_TOP_K}")
        tokens = paragraph_query_tokens(body)
        out = S.ParagraphSuggest([], False, S.ematches(tokens))
        views = [s._gpu.view(m) for s, m in zip(self.segments, masks)]
        try:
            terms, phrases = self._clauses(body)
            if terms or phrases:
                qt, qo = np.asarray(terms, dtype=np.uint32), np.asarray([0, len(terms)], dtype=np.uint32)
                rows = []
                for ord_, v in enumerate(views):
                    params = dict(mode=_lib.NIDX_BM25_OR, use_tf=False, docaddr_base=ord_ << 32)
                    if phrases:
                        docs, scores, counts, _ = v.search_phrases(qt, qo, [(0, p) for p in phrases], top_k, **params)
                    else:
                        docs, scores, counts, _ = v.search(qt, qo, top_k, **params)
                    rows += [(-float(scores[0, i]), ord_, int(docs[0, i])) for i in range(int(counts[0]))]
                rows.sort()
                out.hits = [S.ParagraphHit(-neg, o, d) for neg, o, d in rows[:top_k]]
            if out.hits:
                return out
            clauses = S.fuzzy_clauses(tokens)
            if not clauses:
                return out
            if len(clauses) > _lib.NIDX_SG_MAX_CLAUSES:
                raise ValueError(f"a suggest body of more than {_lib.NIDX_SG_MAX_CLAUSES} clauses is not supported")
            out.fuzzy = True
            out.hits = self._suggest_fuzzy(clauses, top_k, views)
            return out
        finally:
            for v in views:
                v.close()

    def _suggest_fuzzy(self, clauses: list, top_k: int, views: list) -> list:
        from . import suggest as S
        from .segment import SuggestDict

        if self._suggest_dict is None:
            vocab_terms = [""] * len(self.vocab)
            for t, i in self.vocab.items():
                vocab_terms[i] = t
            self._suggest_dict = SuggestDict(vocab_terms, device=self.segments[0].device)
            self._vocab_terms = vocab_terms
        auto = [(v, S.FUZZY_DISTANCE, kind == S.FUZZY_PREFIX) for kind, v in clauses if kind in (S.FUZZY, S.FUZZY_PREFIX)]
        if sum(len(v) for v, _, _ in auto) > S.MAX_FUZZY_CODE_POINTS:
            raise ValueError(f"the fuzzy literals of a suggest body hold more than {S.MAX_FUZZY_CODE_POINTS} code points")
        bits = self._suggest_dict.expand(auto)[0] if auto else None
        spec, phrases, row = [], [], 0
        for kind, v in clauses:
            if kind in (S.FUZZY, S.FUZZY_PREFIX):
                spec.append((_lib.NIDX_SG_FUZZY, row))
                row += 1
            elif kind == S.TERM:
                spec.append((_lib.NIDX_SG_TERM, self.vocab.get(v, _lib.NIL)))
            else:
                spec.append((_lib.NIDX_SG_PHRASE, len(phrases)))
                phrases.append([self.vocab.get(t, 0xFFFFFFF0) for t in v])
        if phrases:
            self._ensure_positions()
        rows, found = [], {}
        for ord_, v in enumerate(views):
            ids, scores, count, trip = v.suggest_fuzzy(spec, bits, len(auto), len(self.vocab), phrases, top_k, min(S.RESULTS_PER_PAGE, top_k))
            rows += [(-float(scores[i]), ord_, int(ids[i])) for i in range(count)]
            for h, c, t in trip:
                found.setdefault((ord_, int(ids[h])), []).append(self._vocab_terms[t])
        rows.sort()
        hits = [S.ParagraphHit(-neg, o, d) for neg, o, d in rows[:top_k]]
        for h in hits[: S.RESULTS_PER_PAGE]:
            h.matches = sorted(t for t in found.get((h.segment, h.doc), []) if len(t.encode("utf-8")) > 2)
        return hits

    def _clauses(self, body: str):
        words, phrases = parse_paragraph_query(body)
        terms = [self.vocab.get(t, 0xFFFFFFF0) for t in words]   # unknown word: matches nothing
        phrase_terms = [[self.vocab.get(t, 0xFFFFFFF0) for t in p] for p in phrases]   # an unknown word: the phrase matches nothing
        if phrase_terms:
            self._ensure_positions()
        return terms, phrase_terms
