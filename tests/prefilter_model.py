"""A literal per-document restatement of the prefilter: nodereader.FilterExpression (SearchRequest.field_filter) over text documents,
as nidx_text's filter_to_query (nidx_text/src/search_query.rs:156-217) and TextReaderService::prefilter (reader.rs:147-180) define
it.  No dictionaries, no ranges, no bitsets: every node is evaluated on the document's own strings, dates and tokens.

    facet f                        the document carries f or a descendant of f (a facet term: tantivy indexes every ancestor; the
                                   root "/" is carried by a document with any label).  f without a leading '/': ValueError
                                   (Facet::from asserts [recalled]).  Labels without a leading '/' are no facets.
    field {type, id?}              the facet term "/type/id" (or "/type") on the field path: the path or a descendant of it
    resource r                     the resource id string equals r
    resource_field_prefix          the resource id parses to the UUID r (else ValueError: the reference panics) and the field name
                                   "type/name" starts with "type/prefix"
    date {field, since?, until?}   both bounds absent: every document (AllQuery); else since <= seconds <= until on that date,
                                   nanos dropped; an undated document never matches
    keyword k                      k's tokens (the default analyzer): 1 = a term, >= 2 = a phrase (slop 0, positions counted before
                                   long tokens are dropped), 0 = the raw literal as one term
    bool_and / bool_or             intersection / union; no operands: nothing
    bool_not e                     not e
Result over every alive document of every segment: 0 matched -> "none", every alive one -> "all", else "some".
"""
from __future__ import annotations

import functools
import uuid

from nucliadb_b200.text import tokenize, tokenize_with_positions


def _under(path: str, f: str) -> bool:
    """The facet `path` is the facet `f` or a descendant of it."""
    return f == "/" or path == f or path.startswith(f + "/")


def _uuid_or_none(s: str):
    try:
        return uuid.UUID(s)
    except ValueError:
        return None


@functools.lru_cache(maxsize=None)
def _positions(doc_text: str) -> dict:
    at = {}
    for p, t in tokenize_with_positions(doc_text):
        at.setdefault(t, set()).add(p)
    return at


def _phrase_in(doc_text: str, words: list) -> bool:
    at = _positions(doc_text)
    return any(all(s + i in at.get(w, ()) for i, w in enumerate(words)) for s in at.get(words[0], ()))


def matches(e, doc) -> bool:
    kind = e.WhichOneof("expr")
    if kind == "facet":
        f = e.facet.facet
        if not f.startswith("/"):
            raise ValueError(f"invalid facet {f!r}")
        return any(_under(l, f) for l in doc.labels if l.startswith("/"))
    if kind == "field":
        ff = e.field
        f = f"/{ff.field_type}/{ff.field_id}" if ff.HasField("field_id") else f"/{ff.field_type}"
        return _under(doc.field, f)
    if kind == "resource":
        return doc.uuid == e.resource.resource_id
    if kind == "resource_field_prefix":
        p = e.resource_field_prefix
        r = _uuid_or_none(p.resource_id)
        if r is None:
            raise ValueError(f"invalid resource id {p.resource_id!r}")
        return _uuid_or_none(doc.uuid) == r and doc.field.startswith(f"/{p.field_type}/{p.field_id_prefix}")
    if kind == "date":
        d = e.date
        if not d.HasField("since") and not d.HasField("until"):
            return True
        v = doc.modified if d.field == 1 else doc.created
        return v is not None and (not d.HasField("since") or v >= d.since.seconds) and (not d.HasField("until") or v <= d.until.seconds)
    if kind == "keyword":
        k = e.keyword.keyword
        words = tokenize(k)
        if len(words) <= 1:
            return (words[0] if words else k) in _positions(doc.text)
        return _phrase_in(doc.text, words)
    if kind == "bool_and":
        ops = e.bool_and.operands
        return len(ops) > 0 and all(matches(o, doc) for o in ops)
    if kind == "bool_or":
        return any(matches(o, doc) for o in e.bool_or.operands)
    if kind == "bool_not":
        return not matches(e.bool_not, doc)
    raise ValueError(f"unknown filter expression {kind!r}")


def prefilter(expr, segments, alive=None):
    """segments: [[TextDoc]], alive: [[bool]] or None (all alive) -> (per segment [bool] matched-and-alive, class)."""
    alive = alive if alive is not None else [[True] * len(s) for s in segments]
    # every node is validated even where a document does not reach it (the reference builds the whole query first)
    _validate(expr)
    bits = [[a and matches(expr, d) for d, a in zip(docs, al)] for docs, al in zip(segments, alive)]
    n = sum(sum(b) for b in bits)
    total = sum(sum(a) for a in alive)
    return bits, ("none" if n == 0 else "all" if n == total else "some")


def _validate(e):
    kind = e.WhichOneof("expr")
    if kind == "facet" and not e.facet.facet.startswith("/"):
        raise ValueError(f"invalid facet {e.facet.facet!r}")
    if kind == "resource_field_prefix" and _uuid_or_none(e.resource_field_prefix.resource_id) is None:
        raise ValueError("invalid resource id")
    if kind in ("bool_and", "bool_or"):
        for o in getattr(e, kind).operands:
            _validate(o)
    if kind == "bool_not":
        _validate(e.bool_not)
    if kind is None:
        raise ValueError("empty filter expression")


def depth(e) -> int:
    """Levels of nesting as the device counts them (NIDX_PREFILTER_MAX_DEPTH): a resource_field_prefix runs as AND(OR(resource
    ords), field range), two levels more than another leaf."""
    kind = e.WhichOneof("expr")
    if kind == "resource_field_prefix":
        return 3
    if kind in ("bool_and", "bool_or"):
        return 1 + max((depth(o) for o in getattr(e, kind).operands), default=0)
    if kind == "bool_not":
        return 1 + depth(e.bool_not)
    return 1
