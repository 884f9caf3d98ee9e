"""The JSON index (reference: nidx/nidx_json) and ``SearchRequest.json_filter`` on the device.

Flattening (nidx_json/src/resource_indexer.rs): every resource with non-empty ``json_fields`` and ``skip_json`` false is ONE document,
the object ``{field_id: json.loads(value)}``; invalid JSON fails the index message.  Values are flattened as tantivy flattens a JSON
field: the path is ``field_id`` + ``.`` + the nested keys joined by ``.``; each element of an array (nested arrays too) is a value of
the array's path; ``null`` is not indexed.  A value is typed (path, kind, value) with kind ``text``, ``bool``, ``num`` or ``date``.

Rules that cannot be checked against tantivy here, each *recalled, unverifiable here* (DESIGN 7 lists them too):
  * numbers: integers and floats share one kind and compare by their numeric value, exactly (150 and 150.0 are the same number), so
    an Int / IntRange predicate matches a float value and a Float / FloatRange predicate matches an integer value;
  * integers above i64::MAX up to u64::MAX keep their exact value (tantivy stores them as u64); larger ones, and smaller than
    i64::MIN, are the float serde_json parses them to;
  * a number whose float is not finite (``1e400``, an integer beyond the f64 range) is invalid JSON and fails the index message, as
    serde_json's "number out of range" does, and so are NaN and Infinity;
  * a string in RFC 3339 form (``2024-01-01T00:00:00Z``, offset or ``Z`` required, fraction allowed) is a text value AND a date value,
    in seconds since the epoch (the fraction dropped towards -inf), as the Date / DateRange predicates compare at second precision;
  * a key that contains ``.`` is one path segment: the filter's path is split at every ``.`` that is not escaped as ``\\.``, so
    ``{"a.b": 1}`` answers ``a\\.b``, and ``a.b`` answers ``{"a": {"b": 1}}`` only.

Query (nidx_json/src/search.rs, query_planner/prefilter.rs:175-233): Text is an exact, case-sensitive match; Boolean, Int, Float, Date
and their ranges compare values of that kind with inclusive bounds, a missing bound unbounded; AND / OR are Must / Should (without
operands: nothing), NOT is Must(AllQuery) + MustNot, i.e. it ranges over the JSON documents, not over every resource.  An expression
without ``expr`` or a path without a predicate is a ValueError (InvalidRequest).

On the device the JSON documents are a text segment without terms (include/nidx_b200.h, "JSON filters"): the dictionary of every
(path, kind, value), sorted, lives on the host; a document's values are facet ords in HBM, so a leaf is one ord range found by binary
search and the expression runs in nidx_txt_prefilter's single pass, then nidx_txt_resource_bits turns the matched documents into a
bitset over this index's resources.
"""
from __future__ import annotations

import bisect
import datetime as _dt
import json
import math
import re
from typing import Optional, Sequence

import numpy as np

from . import _lib

I64_MIN, I64_MAX, U64_MAX = -(1 << 63), (1 << 63) - 1, (1 << 64) - 1
_RFC3339 = re.compile(r"^\d{4}-\d{2}-\d{2}[Tt ]\d{2}:\d{2}:\d{2}(\.\d+)?([Zz]|[+-]\d{2}:\d{2})$")
SEP = "\x01"   # joins path segments in a path key (no JSON key can contain it unescaped in a filter path)


def _reject_constant(name):
    raise ValueError(f"invalid JSON: {name} is not a JSON number")


def rfc3339_seconds(s: str) -> Optional[int]:
    """Seconds since the epoch of an RFC 3339 date-time string, else None."""
    if not _RFC3339.match(s):
        return None
    body = s[:-1] + "+00:00" if s[-1] in "Zz" else s
    try:
        t = _dt.datetime.fromisoformat(body.replace("t", "T").replace(" ", "T", 1))
    except ValueError:
        return None
    delta = t - _dt.datetime(1970, 1, 1, tzinfo=_dt.timezone.utc)
    return delta.days * 86400 + delta.seconds   # microseconds dropped: floor towards -inf


def _finite(x: float) -> float:
    if not math.isfinite(x):
        raise ValueError("invalid JSON: number out of range")
    return x


def _number(v):
    if isinstance(v, int) and not (I64_MIN <= v <= U64_MAX):
        try:
            return _finite(float(v))
        except OverflowError:
            raise ValueError("invalid JSON: number out of range") from None
    return v


def flatten(json_fields) -> list:
    """{field_id: JSON text} -> [(path key, kind, value)]: the typed values of one JSON document (path segments joined by SEP)."""
    out = []

    def walk(segs, v):
        if v is None:
            return
        if isinstance(v, dict):
            for k, x in v.items():
                walk(segs + (k,), x)
        elif isinstance(v, list):
            for x in v:
                walk(segs, x)
        elif isinstance(v, bool):
            out.append((SEP.join(segs), "bool", v))
        elif isinstance(v, (int, float)):
            out.append((SEP.join(segs), "num", _number(v)))
        elif isinstance(v, str):
            out.append((SEP.join(segs), "text", v))
            secs = rfc3339_seconds(v)
            if secs is not None:
                out.append((SEP.join(segs), "date", secs))

    for field_id, text in json_fields.items():
        walk((field_id,), json.loads(text, parse_constant=_reject_constant, parse_float=lambda t: _finite(float(t))))
    return out


def path_key(field_id: str, json_path: str) -> str:
    """The path of a JsonFieldPathFilter: ``field_id.json_path`` split at every unescaped ``.``."""
    segs, cur, s, i = [], [], f"{field_id}.{json_path}", 0
    while i < len(s):
        if s[i] == "\\" and i + 1 < len(s) and s[i + 1] == ".":
            cur.append(".")
            i += 2
            continue
        if s[i] == ".":
            segs.append("".join(cur))
            cur = []
        else:
            cur.append(s[i])
        i += 1
    segs.append("".join(cur))
    return SEP.join(segs)


def leaf_range(path_filter):
    """JsonFieldPathFilter -> (path key, kind, lo, hi) with inclusive bounds, None = unbounded."""
    pred = path_filter.WhichOneof("predicate")
    if pred is None:
        raise ValueError("Missing predicate")
    p = path_key(path_filter.field_id, path_filter.json_path)
    opt = lambda m, f, g=lambda x: x: g(getattr(m, f)) if m.HasField(f) else None   # noqa: E731
    if pred == "text":
        return p, "text", path_filter.text, path_filter.text
    if pred == "boolean":
        return p, "bool", path_filter.boolean, path_filter.boolean
    if pred in ("int", "float"):
        v = getattr(path_filter, pred)
        return p, "num", v, v
    if pred in ("int_range", "float_range"):
        r = getattr(path_filter, pred)
        return p, "num", opt(r, "lower"), opt(r, "upper")
    if pred == "date":
        return p, "date", path_filter.date.seconds, path_filter.date.seconds
    r = path_filter.date_range
    return p, "date", opt(r, "lower", lambda t: t.seconds), opt(r, "upper", lambda t: t.seconds)


def validate(expr):
    """Raise ValueError where the reference's proto_to_json_filter returns InvalidRequest."""
    kind = expr.WhichOneof("expr")
    if kind is None:
        raise ValueError("Empty JsonFilterExpression")
    if kind == "path":
        leaf_range(expr.path)
    elif kind == "bool_not":
        validate(expr.bool_not)
    else:
        for o in getattr(expr, kind).operands:
            validate(o)


class JsonIndex:
    """The alive JSON documents of a shard on one device: docs = [(resource id, [(path key, kind, value)], access groups)]."""

    def __init__(self, docs: Sequence[tuple], device=0):
        from .segment import TextSegment
        from .text import group_key

        self.device, self.n_docs = device, len(docs)
        self.resource_ids = sorted({d[0] for d in docs})
        res_of = {r: i for i, r in enumerate(self.resource_ids)}
        lists: dict = {}
        for _, entries, _ in docs:
            for p, k, v in entries:
                lists.setdefault((p, k), set()).add(v)
        self.values, self.base, n = {}, {}, 0
        for key in sorted(lists):
            self.values[key] = sorted(lists[key])
            self.base[key] = n
            n += len(self.values[key])
        self.n_values = n
        rows = [sorted({self.base[(p, k)] + bisect.bisect_left(self.values[(p, k)], v) for p, k, v in entries}) for _, entries, _ in docs]
        self.group_keys = sorted({group_key(g) for _, _, gs in docs for g in gs})
        gord = {g: i for i, g in enumerate(self.group_keys)}
        grows = [sorted({gord[group_key(g)] for g in gs}) for _, _, gs in docs]
        self.segment = TextSegment.create(self.n_docs, 0, np.zeros(1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32),
                                          np.zeros(self.n_docs, dtype=np.uint8), device=device)
        # the value dictionary stays here: the library gets one 8-byte big-endian key per ord, which keeps the keys ascending
        kb = np.arange(n, dtype=">u8").view(np.uint8)
        ko = np.arange(n + 1, dtype=np.uint64) * 8
        off = np.zeros(self.n_docs + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(r) for r in rows])
        ords = np.asarray([o for r in rows for o in r], dtype=np.uint32)
        _lib.check(_lib.load().nidx_txt_set_facets(self.segment._h, n, _lib.ptr(kb), _lib.ptr(ko), _lib.ptr(off), _lib.ptr(ords)))
        self.segment.set_doc_columns(np.asarray([res_of[d[0]] for d in docs], dtype=np.uint32), np.zeros(self.n_docs, dtype=np.uint32))
        goff = np.zeros(self.n_docs + 1, dtype=np.uint64)
        goff[1:] = np.cumsum([len(r) for r in grows])
        self.segment.set_doc_groups(self.group_keys, goff, np.asarray([o for r in grows for o in r], dtype=np.uint32))

    def close(self):
        self.segment.close()

    # ---- JsonFilterExpression -> flat pre-order prefilter nodes (kind, n, lo, hi, terms) ---------------------------------------
    def ord_range(self, path: str, kind: str, lo, hi):
        """The ords [b, e) of the values of (path, kind) within [lo, hi] (None: unbounded)."""
        vals = self.values.get((path, kind))
        if vals is None or (lo is not None and lo != lo) or (hi is not None and hi != hi):   # absent path, NaN bound
            return 0, 0
        b = 0 if lo is None else bisect.bisect_left(vals, lo)
        e = len(vals) if hi is None else bisect.bisect_right(vals, hi)
        base = self.base[(path, kind)]
        return base + b, base + max(b, e)

    def compile(self, expr, security: Optional[Sequence[str]] = None) -> list:
        flat = []

        def walk(e):
            kind = e.WhichOneof("expr")
            if kind is None:
                raise ValueError("Empty JsonFilterExpression")
            if kind == "path":
                b, e_ = self.ord_range(*leaf_range(e.path))
                flat.append((_lib.NIDX_P_FACET, 0, b, e_, None) if e_ > b else (_lib.NIDX_P_OR, 0, 0, 0, None))
            elif kind == "bool_not":
                flat.append((_lib.NIDX_P_NOT, 1, 0, 0, None))
                walk(e.bool_not)
            else:
                ops = getattr(e, kind).operands
                flat.append((_lib.NIDX_P_AND if kind == "bool_and" else _lib.NIDX_P_OR, len(ops), 0, 0, None))
                for o in ops:
                    walk(o)

        if security is not None:   # the resource's access groups, over this index's dictionary
            from .text import security_tree

            flat.append((_lib.NIDX_P_AND, 2, 0, 0, None))
            flat += security_tree(self.group_keys, security)
        walk(expr)
        return flat

    def prefilter(self, expr, security: Optional[Sequence[str]] = None, on_device: bool = True):
        """The expression (AND the access groups of `security`) over the alive documents -> (document bits, matching documents,
        resource bits over resource_ids).  on_device: torch CUDA int64 tensors, else numpy uint64 words."""
        from ._lib import NidxError
        from .text import _node_array

        nodes = _node_array(self.compile(expr, security))
        out = None
        if on_device:
            import torch

            out = torch.empty(max((self.n_docs + 63) // 64, 1), dtype=torch.int64, device=torch.device("cuda", self.device))
        try:
            bits, matching = self.segment.prefilter(nodes, out=out)
        except NidxError as e:
            if e.code == -1:   # NIDX_EINVAL: deeper than NIDX_PREFILTER_MAX_DEPTH or a longer program
                raise ValueError(str(e)) from e
            raise
        return bits, matching, self.segment.resource_bits(bits, len(self.resource_ids))
