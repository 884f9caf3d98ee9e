"""A per-document host model of the JSON prefilter (nidx_json) and of its combination with the text prefilter, written against parsed
JSON objects directly (no ord dictionary, no device): what nucliadb_b200/json_index.py and the device hand-offs are checked against.

  matches(doc, expr)        one JSON document ({field_id: parsed JSON}) against a nodereader.JsonFilterExpression
  resources(docs, expr)     the resource set: every alive document that matches, by resource id (NOT ranges over the documents)
  combine(text, res, op)    PrefilterResult::combine (nidx_types/src/prefilter.rs:49-92) on ("all" | "none" | set of (rid, field))
  with_security(...)        the rule here: AND(security, op(field_filter, json)) -- a security filter is never widened
"""
import datetime
import re

_RFC3339 = re.compile(r"^\d{4}-\d{2}-\d{2}[Tt ]\d{2}:\d{2}:\d{2}(\.\d+)?([Zz]|[+-]\d{2}:\d{2})$")


def _date(s):
    if not isinstance(s, str) or not _RFC3339.match(s):
        return None
    t = datetime.datetime.fromisoformat(s.upper().replace(" ", "T").replace("Z", "+00:00"))
    return int((t - datetime.datetime(1970, 1, 1, tzinfo=datetime.timezone.utc)).total_seconds() // 1)


def _segments(field_id, json_path):
    return [p.replace("\0", ".") for p in f"{field_id}.{json_path}".replace("\\.", "\0").split(".")]


def values(doc, segs):
    """Every non-null scalar at the path `segs` of a document (arrays flattened)."""
    def walk(v, rest):
        if isinstance(v, list):
            for x in v:
                yield from walk(x, rest)
        elif not rest:
            if v is not None and not isinstance(v, dict):
                yield v
        elif isinstance(v, dict) and rest[0] in v:
            yield from walk(v[rest[0]], rest[1:])
    return list(walk(doc, segs))


def _num(v):
    if isinstance(v, bool) or not isinstance(v, (int, float)):
        return None
    return float(v) if isinstance(v, int) and not (-(1 << 63) <= v <= (1 << 64) - 1) else v


def _in(x, lo, hi):
    return x is not None and (lo is None or x >= lo) and (hi is None or x <= hi)


def leaf(doc, f):
    vals = values(doc, _segments(f.field_id, f.json_path))
    p = f.WhichOneof("predicate")
    opt = lambda m, n: getattr(m, n) if m.HasField(n) else None   # noqa: E731
    if p == "text":
        return any(isinstance(v, str) and v == f.text for v in vals)
    if p == "boolean":
        return any(isinstance(v, bool) and v == f.boolean for v in vals)
    if p in ("int", "float"):
        x = getattr(f, p)
        return any(_num(v) is not None and _num(v) == x for v in vals)
    if p in ("int_range", "float_range"):
        r = getattr(f, p)
        lo, hi = opt(r, "lower"), opt(r, "upper")
        return any(_in(_num(v), lo, hi) for v in vals)
    if p == "date":
        return any(_date(v) == f.date.seconds for v in vals)
    if p == "date_range":
        r = f.date_range
        lo = r.lower.seconds if r.HasField("lower") else None
        hi = r.upper.seconds if r.HasField("upper") else None
        return any(_in(_date(v), lo, hi) for v in vals)
    raise ValueError("Missing predicate")


def matches(doc, e) -> bool:
    kind = e.WhichOneof("expr")
    if kind is None:
        raise ValueError("Empty JsonFilterExpression")
    if kind == "path":
        return leaf(doc, e.path)
    if kind == "bool_not":
        return not matches(doc, e.bool_not)
    ops = [matches(doc, o) for o in e.bool_and.operands] if kind == "bool_and" else [matches(doc, o) for o in e.bool_or.operands]
    return (all(ops) if kind == "bool_and" else any(ops)) if ops else False


def resources(docs, e) -> set:
    """docs: [(resource id, {field_id: parsed JSON})] (the alive JSON documents)."""
    return {rid for rid, doc in docs if matches(doc, e)}


def combine(text, res: set, op_or: bool):
    """text: "all" | "none" | set of (rid, field); fields at resource level are (rid, None)."""
    if not res:
        return text if op_or else "none"
    res_level = {(r, None) for r in res}
    if op_or:
        if text == "all":
            return "all"
        if text == "none":
            return res_level
        return res_level | {f for f in text if f[0] not in res}
    if text == "none":
        return "none"
    if text == "all":
        return res_level
    kept = {f for f in text if f[0] in res}
    return kept or "none"


def admits(result, rid, field) -> bool:
    """Whether a combined result lets a paragraph of (rid, field) through (a resource-level entry admits every field)."""
    if result == "all":
        return True
    if result == "none":
        return False
    return (rid, None) in result or (rid, field) in result


def with_security(visible: set, text, res: set, op_or: bool):
    """AND(security, op(field_filter, json)): text and res already ANDed with the visible resources, then combined."""
    t = text if text in ("all", "none") else {f for f in text if f[0] in visible}
    return combine(t, res & visible, op_or), visible
