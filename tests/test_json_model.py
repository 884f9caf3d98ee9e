"""tests/json_model.py pinned to the reference's known answers: the 17 unit tests of nidx_json/src/search.rs and the 8 searches of
tests/integration/search_json_filter.rs (fixtures restated by hand), PrefilterResult::combine, and the flattening rules chosen in
nucliadb_b200/json_index.py."""
import json

import pytest

from nucliadb_b200 import json_index as J
from nucliadb_b200 import nidx_protos as P

import json_model as M


def path(field_id, json_path, **pred):
    e = P.JsonFilterExpression()
    e.path.field_id, e.path.json_path = field_id, json_path
    (k, v), = pred.items()
    if k in ("int_range", "float_range", "date_range"):
        for b, x in zip(("lower", "upper"), v):
            if x is not None:
                if k == "date_range":
                    getattr(getattr(e.path, k), b).seconds = x
                else:
                    setattr(getattr(e.path, k), b, x)
        getattr(e.path, k).SetInParent()
    elif k == "date":
        e.path.date.seconds = v
    else:
        setattr(e.path, k, v)
    return e


def op(kind, *operands):
    e = P.JsonFilterExpression()
    if kind == "not":
        e.bool_not.CopyFrom(operands[0])
    else:
        getattr(e, "bool_" + kind).operands.extend(operands)
        getattr(e, "bool_" + kind).SetInParent()
    return e


# nidx_json/src/search.rs build_test_index / build_date_index (uuids 1, 2, 3 and 0x11, 0x12, 0x13)
PRODUCTS = [("apple", {"t/product": {"name": "red apple", "price": 150, "score": 4.5, "available": True}}),
            ("banana", {"t/product": {"name": "green banana", "price": 80, "score": 3.2, "available": False}}),
            ("cherry", {"t/product": {"name": "red cherry", "price": 200, "score": 4.8, "available": True}})]
EVENTS = [("old", {"t/event": {"ts": "2020-01-01T00:00:00Z"}}), ("mid", {"t/event": {"ts": "2022-06-15T00:00:00Z"}}),
          ("new", {"t/event": {"ts": "2024-01-01T00:00:00Z"}})]

UNIT = [   # (name, docs, expr, must contain, must not contain, exact set or None)
    ("test_exact_match", PRODUCTS, path("t/product", "name", text="red apple"), {"apple"}, set(), None),
    ("test_exact_match_partial", PRODUCTS, path("t/product", "name", text="apple"), set(), {"apple"}, None),
    ("test_int_exact", PRODUCTS, path("t/product", "price", int=150), {"apple"}, {"banana", "cherry"}, None),
    ("test_int_range", PRODUCTS, path("t/product", "price", int_range=(80, 150)), {"apple", "banana"}, {"cherry"}, None),
    ("test_int_range_unbounded_upper", PRODUCTS, path("t/product", "price", int_range=(150, None)), {"apple", "cherry"}, set(), None),
    ("test_float_exact", PRODUCTS, path("t/product", "score", float=3.2), {"banana"}, {"apple", "cherry"}, None),
    ("test_float_range", PRODUCTS, path("t/product", "score", float_range=(4.0, 5.0)), {"apple", "cherry"}, set(), None),
    ("test_bool_match_true", PRODUCTS, path("t/product", "available", boolean=True), {"apple", "cherry"}, set(), None),
    ("test_bool_match_false", PRODUCTS, path("t/product", "available", boolean=False), set(), set(), {"banana"}),
    ("test_and_combination", PRODUCTS, op("and", path("t/product", "available", boolean=True), path("t/product", "price", int_range=(None, 150))),
     set(), set(), {"apple"}),
    ("test_or_combination", PRODUCTS, op("or", path("t/product", "available", boolean=False)), {"banana"}, set(), None),
    ("test_not_combination", PRODUCTS, op("not", path("t/product", "available", boolean=False)), {"apple", "cherry"}, {"banana"}, None),
    ("test_nested_and_or", PRODUCTS, op("or", op("and", path("t/product", "available", boolean=True), path("t/product", "price", int_range=(None, 150))),
                                        path("t/product", "available", boolean=False)), {"apple", "banana"}, {"cherry"}, None),
    ("test_exact_match_text_field", [("x", {"k/product": {"color": "Red Apple"}})], path("k/product", "color", text="Red Apple"), {"x"}, set(), None),
    ("test_exact_match_text_field_partial", [("x", {"k/product": {"color": "Red Apple"}})], path("k/product", "color", text="red"), set(), {"x"}, None),
    ("test_exact_match_text_field_case", [("x", {"k/product": {"color": "Red Apple"}})], path("k/product", "color", text="red apple"), set(), {"x"}, None),
    ("test_date_exact", EVENTS, path("t/event", "ts", date=1655251200), set(), set(), {"mid"}),
    ("test_date_range_bounded", EVENTS, path("t/event", "ts", date_range=(1609459200, 1672531200)), set(), set(), {"mid"}),
    ("test_date_range_unbounded_upper", EVENTS, path("t/event", "ts", date_range=(1640995200, None)), {"mid", "new"}, {"old"}, None),
    ("test_date_range_unbounded_lower", EVENTS, path("t/event", "ts", date_range=(None, 1609459200)), set(), set(), {"old"}),
]


@pytest.mark.parametrize("name,docs,expr,yes,no,exact", UNIT, ids=[u[0] for u in UNIT])
def test_reference_unit_cases(name, docs, expr, yes, no, exact):
    got = M.resources(docs, expr)
    assert yes <= got and not (no & got)
    if exact is not None:
        assert got == exact


# tests/integration/search_json_filter.rs setup_fixture: {"price", "category", "available"} under t/product, one paragraph each
FIXTURE = [("apple", 150, "fruit", True), ("banana", 80, "fruit", False), ("hammer", 200, "tool", True)]
INTEGRATION = [
    ("test_json_exact_match", path("t/product", "category", text="fruit"), {"apple", "banana"}),
    ("test_json_no_match", path("t/product", "category", text="vegetable"), set()),
    ("test_json_int_range", path("t/product", "price", int_range=(80, 150)), {"apple", "banana"}),
    ("test_json_bool_match", path("t/product", "available", boolean=True), {"apple", "hammer"}),
    ("test_json_and_filter", op("and", path("t/product", "category", text="fruit"), path("t/product", "available", boolean=True)), {"apple"}),
    ("test_json_or_filter", op("or", path("t/product", "available", boolean=False), path("t/product", "category", text="tool")), {"banana", "hammer"}),
    ("test_json_not_filter", op("not", path("t/product", "category", text="tool")), {"apple", "banana"}),
]


def fixture_docs():
    return [(r, {"t/product": json.loads(json.dumps({"price": p, "category": c, "available": a}))}) for r, p, c, a in FIXTURE]


@pytest.mark.parametrize("name,expr,want", INTEGRATION, ids=[i[0] for i in INTEGRATION])
def test_reference_integration_searches(name, expr, want):
    res = M.resources(fixture_docs(), expr)
    result = M.combine("all", res, op_or=False)   # no field_filter: the text result is All
    got = {r for r, _, _, _ in FIXTURE if M.admits(result, r, "/a/title")}
    assert got == want


def test_reference_integration_with_security():
    """test_json_filter_combined_with_security: apple {engineering, fruit}, banana {other, fruit}, hammer {engineering, tool}."""
    visible = {"apple", "hammer"}
    res = M.resources(fixture_docs(), path("t/product", "category", text="fruit"))
    result, vis = M.with_security(visible, "all", res, op_or=False)
    assert {r for r in ("apple", "banana", "hammer") if r in vis and M.admits(result, r, "/a/title")} == {"apple"}


def test_security_is_not_widened_under_or():
    res = {"banana"}                                   # matches the JSON filter, outside the caller's groups
    text = {("apple", "/a/title")}                     # the field filter's fields, already ANDed with security
    result, vis = M.with_security({"apple"}, text, res, op_or=True)
    assert not (M.admits(result, "banana", "/a/title") and "banana" in vis)
    assert M.combine(text, res, op_or=True) != "none" and M.admits(M.combine(text, res, True), "banana", "/a/title")   # the reference would


def test_combine_cases():
    t = {("a", "/t/x"), ("b", "/t/y")}
    assert M.combine(t, set(), True) == t and M.combine(t, set(), False) == "none"
    assert M.combine("all", {"a"}, True) == "all" and M.combine("all", {"a"}, False) == {("a", None)}
    assert M.combine("none", {"a"}, True) == {("a", None)} and M.combine("none", {"a"}, False) == "none"
    assert M.combine(t, {"a"}, True) == {("a", None), ("b", "/t/y")}
    assert M.combine(t, {"a"}, False) == {("a", "/t/x")} and M.combine(t, {"c"}, False) == "none"
    # PrefilterResult.combine gives the model's All and None; a Some keeps the text part and the non-empty resource set as parts
    from nucliadb_b200 import vector as V

    text = V.PrefilterResult.from_device("text index", "text bits", len(t))
    for model, pf in (("all", V.PrefilterResult.all()), ("none", V.PrefilterResult.none()), (t, text)):
        for res in (set(), {"a"}):
            for op_or in (False, True):
                got, want = pf.combine("json index", "res bits" if res else None, len(res), op_or), M.combine(model, res, op_or)
                assert got.kind == (want if want in ("all", "none") else "some"), (model, res, op_or)
                if got.kind == "some":
                    assert got.device_bits == pf.device_bits and got.resources == (("json index", "res bits") if res else None)
                    assert got.op_or == (op_or and pf is text and bool(res))


def test_empty_expression_and_missing_predicate_are_invalid():
    with pytest.raises(ValueError):
        J.validate(P.JsonFilterExpression())
    e = P.JsonFilterExpression()
    e.path.field_id, e.path.json_path = "t/x", "a"
    with pytest.raises(ValueError):
        J.validate(e)
    J.validate(op("and"))   # no operands: valid, matches nothing
    assert M.resources(PRODUCTS, op("and")) == set() and M.resources(PRODUCTS, op("or")) == set()


def test_flattening_nested_arrays_mixed_types():
    doc = {"t/p": json.dumps({"a": {"b": [1, [2.5, None], {"c": "x"}], "d": None}, "e": [True, "2024-01-01T00:00:00+01:00"], "a.b": 7})}
    got = sorted(J.flatten(doc), key=repr)
    want = sorted([("t/p\x01a\x01b", "num", 1), ("t/p\x01a\x01b", "num", 2.5), ("t/p\x01a\x01b\x01c", "text", "x"), ("t/p\x01e", "bool", True),
                   ("t/p\x01e", "text", "2024-01-01T00:00:00+01:00"), ("t/p\x01e", "date", 1704063600), ("t/p\x01a.b", "num", 7)], key=repr)
    assert got == want
    assert J.path_key("t/p", "a.b") == "t/p\x01a\x01b" and J.path_key("t/p", "a\\.b") == "t/p\x01a.b"
    # the model reads the same values through the same rules
    parsed = {"t/p": json.loads(doc["t/p"])}
    assert M.resources([("r", parsed)], path("t/p", "a.b", int=1)) == {"r"}
    assert M.resources([("r", parsed)], path("t/p", "a\\.b", int=7)) == {"r"}
    assert M.resources([("r", parsed)], path("t/p", "a.b", int=7)) == set()
    assert M.resources([("r", parsed)], path("t/p", "e", date=1704063600)) == {"r"}
    assert M.resources([("r", parsed)], path("t/p", "a.d", text="")) == set()   # null is not indexed


def test_numbers_compare_by_value_whatever_their_type():
    docs = [("i", {"f": {"v": 150}}), ("f", {"f": {"v": 150.0}}), ("h", {"f": {"v": 2 ** 63}}), ("g", {"f": {"v": 10 ** 30}})]
    assert M.resources(docs, path("f", "v", int=150)) == {"i", "f"}
    assert M.resources(docs, path("f", "v", float=150.0)) == {"i", "f"}
    assert M.resources(docs, path("f", "v", int_range=(2 ** 62, None))) == {"h", "g"}
    assert M.resources(docs, path("f", "v", float_range=(1e30, 1e30))) == {"g"}
    assert J.flatten({"f": json.dumps({"v": 2 ** 63})}) == [("f\x01v", "num", 2 ** 63)]
    assert J.flatten({"f": json.dumps({"v": 10 ** 30})}) == [("f\x01v", "num", 1e30)]


def test_invalid_json_fails():
    with pytest.raises(ValueError):
        J.flatten({"f": "{not json"})
    with pytest.raises(ValueError):
        J.flatten({"f": '{"v": NaN}'})


def test_rfc3339_rule():
    assert J.rfc3339_seconds("2022-06-15T00:00:00Z") == 1655251200
    assert J.rfc3339_seconds("2022-06-15T00:00:00.9Z") == 1655251200
    assert J.rfc3339_seconds("1969-12-31T23:59:59.5Z") == -1
    assert J.rfc3339_seconds("2022-06-15") is None and J.rfc3339_seconds("red apple") is None
    assert J.rfc3339_seconds("2022-06-15T02:00:00+02:00") == 1655251200
    assert J.rfc3339_seconds("2022-06-14T22:00:00-02:00") == 1655251200


def test_numbers_out_of_range_fail():
    for text in ('{"v": 1e400}', '{"v": -1e400}', '{"v": ' + "9" * 400 + "}"):
        with pytest.raises(ValueError):
            J.flatten({"f": text})
