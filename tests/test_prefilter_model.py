"""The prefilter's per-document model (tests/prefilter_model.py) without a GPU: equal to the binding's former host loop on the nodes
that loop evaluates, and hand-checked on the rest (dates, keywords, resource_field_prefix) and on the cases where the loop and the
reference disagree (an empty bool_and, a facet without a leading '/', a field id containing '/')."""
import random
import uuid

import pytest

from nucliadb_b200 import nidx_protos as P
from nucliadb_b200.binding import _doc_matches
from nucliadb_b200.text import TextDoc, _prefix_range

import prefilter_model as M

RIDS = [uuid.UUID(int=i + 1).hex for i in range(6)]
LABELS = ["/l/a", "/l/a/b", "/l/c", "/k/x", "/k/x/y/z", "/e"]
FIELDS = ["/a/title", "/a/summary", "/f/file1", "/t/text", "/a/titles"]


def _docs(rng, n):
    return [TextDoc(rng.choice(RIDS), rng.choice(FIELDS), "alpha beta", tuple(rng.sample(LABELS, rng.randint(0, 3)))) for _ in range(n)]


def _random_expr(rng, depth):
    e = P.FilterExpression()
    kind = rng.choice(["facet", "field", "resource", "and", "or", "not"] if depth > 1 else ["facet", "field", "resource"])
    if kind == "facet":
        e.facet.facet = rng.choice(LABELS + ["/l", "/k/x/y", "/nope"])
    elif kind == "field":
        e.field.field_type = rng.choice(["a", "f", "t", "x"])
        if rng.random() < 0.6:
            e.field.field_id = rng.choice(["title", "summary", "file1", "text", "titl"])
    elif kind == "resource":
        e.resource.resource_id = rng.choice(RIDS + ["other"])
    elif kind == "not":
        e.bool_not.CopyFrom(_random_expr(rng, depth - 1))
    else:
        ops = getattr(e, "bool_and" if kind == "and" else "bool_or").operands
        for _ in range(rng.randint(1, 4)):   # at least one operand: an empty bool_and is a degenerate case
            ops.add().CopyFrom(_random_expr(rng, depth - 1))
    return e


def test_model_equals_the_host_loop_on_its_nodes():
    rng = random.Random(11)
    docs = _docs(rng, 300)
    for _ in range(300):
        e = _random_expr(rng, rng.randint(1, 6))
        assert [M.matches(e, d) for d in docs] == [_doc_matches(e, d) for d in docs], e


def _set(ts, seconds):
    ts.seconds, ts.nanos = seconds, 999_999_999


def test_date_bounds():
    docs = [TextDoc(RIDS[0], "/a/t", "", (), 100, 200), TextDoc(RIDS[0], "/a/t", "", (), None, None), TextDoc(RIDS[0], "/a/t", "", (), 99, 201)]
    e = P.FilterExpression()
    e.date.field = 0
    _set(e.date.since, 100)          # inclusive, nanos ignored
    assert [M.matches(e, d) for d in docs] == [True, False, False]
    _set(e.date.until, 99)
    assert [M.matches(e, d) for d in docs] == [False, False, False]
    e.date.ClearField("since")
    assert [M.matches(e, d) for d in docs] == [False, False, True]
    e.date.field = 1                          # modified
    _set(e.date.until, 200)
    assert [M.matches(e, d) for d in docs] == [True, False, False]
    _set(e.date.until, 201)
    assert [M.matches(e, d) for d in docs] == [True, False, True]
    both_absent = P.FilterExpression()
    both_absent.date.field = 1
    assert [M.matches(both_absent, d) for d in docs] == [True, True, True]   # AllQuery: undated documents too


def test_keywords():
    long = "x" * 45
    docs = [TextDoc(RIDS[0], "/a/t", "Alpha beta gamma", ()), TextDoc(RIDS[0], "/a/t", f"alpha {long} beta gamma", ()),
            TextDoc(RIDS[0], "/a/t", "gamma beta alpha", ())]

    def kw(k):
        e = P.FilterExpression()
        e.keyword.keyword = k
        return [M.matches(e, d) for d in docs]

    assert kw("BETA") == [True, True, True]                        # 1 token: a term
    assert kw("alpha beta gamma") == [True, False, False]          # 3 tokens: a phrase; the dropped long token leaves a gap
    assert kw(f"alpha {long} beta") == [True, False, False]        # the query's long token is dropped: "alpha beta"
    assert kw("beta gamma") == [True, True, False]
    assert kw("!!") == [False, False, False] and kw("") == [False, False, False]   # 0 tokens: the raw literal, never a token


def test_resource_field_prefix():
    rid = uuid.UUID(int=7)
    docs = [TextDoc(rid.hex, "/a/title", "", ()), TextDoc(str(rid), "/a/summary", "", ()), TextDoc(rid.hex, "/f/title", "", ()),
            TextDoc(RIDS[0], "/a/title", "", ())]
    e = P.FilterExpression()
    e.resource_field_prefix.resource_id = str(rid)                 # the hyphenated spelling parses to the same UUID
    e.resource_field_prefix.field_type = "a"
    assert [M.matches(e, d) for d in docs] == [True, True, False, False]   # empty prefix: every field of the type
    e.resource_field_prefix.field_id_prefix = "ti"
    assert [M.matches(e, d) for d in docs] == [True, False, False, False]
    e.resource_field_prefix.resource_id = "not-a-uuid"
    with pytest.raises(ValueError):
        M.prefilter(e, [docs])


def test_degenerate_cases_follow_the_reference():
    docs = [TextDoc(RIDS[0], "/a/x/y", "", ("/l/a", "bare")), TextDoc(RIDS[0], "/a/x", "", ())]
    empty_and = P.FilterExpression()
    empty_and.bool_and.SetInParent()
    assert [M.matches(empty_and, d) for d in docs] == [False, False]          # the host loop: all([]) matched everything
    assert [_doc_matches(empty_and, d) for d in docs] == [True, True]
    bare = P.FilterExpression()
    bare.facet.facet = "bare"                                                  # no leading '/': the reference fails the request
    with pytest.raises(ValueError):
        M.prefilter(bare, [docs])
    assert _doc_matches(bare, docs[0])
    fid = P.FilterExpression()
    fid.field.field_type, fid.field.field_id = "a", "x"                      # a facet term: "/a/x/y" is a descendant of "/a/x"
    assert [M.matches(fid, d) for d in docs] == [True, True]
    assert [_doc_matches(fid, d) for d in docs] == [False, True]
    slash = P.FilterExpression()
    slash.field.field_type, slash.field.field_id = "a", "x/y"                # a field id containing '/'
    assert [M.matches(slash, d) for d in docs] == [True, False]


def test_result_classes():
    docs = [TextDoc(RIDS[0], "/a/t", "", ("/l/a",)), TextDoc(RIDS[1], "/a/t", "", ())]
    e = P.FilterExpression()
    e.facet.facet = "/l/a"
    assert M.prefilter(e, [docs])[1] == "some"
    assert M.prefilter(e, [docs], [[True, False]])[1] == "all"     # every ALIVE document matched
    assert M.prefilter(e, [docs], [[False, True]])[1] == "none"


def test_prefix_ranges_of_the_host_dictionaries():
    """The ord ranges the host resolves strings into (text._prefix_range), against a scan of the sorted keys."""
    rng = random.Random(3)
    alphabet = [b"a", b"b", b"\0", b"\xff", b"ab"]
    keys = sorted({b"".join(rng.choice(alphabet) for _ in range(rng.randint(0, 4))) for _ in range(200)})
    for _ in range(300):
        p = b"".join(rng.choice(alphabet) for _ in range(rng.randint(0, 3)))
        lo, hi = _prefix_range(keys, p, facet=False)
        assert keys[lo:hi] == [k for k in keys if k.startswith(p)], p
        lo, hi = _prefix_range(keys, p, facet=True)
        assert keys[lo:hi] == [k for k in keys if not p or k == p or k.startswith(p + b"\0")], p
