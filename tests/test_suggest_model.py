"""Suggest's plan and the host model (tests/suggest_model.py) against the reference's own tests: suggest.rs's split test, fuzzy_parser.rs's
clause tests and every assertion of tests/integration/suggest.rs, over the golden shard (tests/golden/suggest_shard.json).  CPU only."""
import numpy as np
import pytest

import graph_model as GM
import suggest_model as SM
from nucliadb_b200 import graph as G
from nucliadb_b200 import suggest as S
from nucliadb_b200.text import TextDoc, paragraph_query_tokens


def test_split_suggest_query_as_suggest_rs():
    query = "what are the best use cases for Apache Cassandra"
    assert S.split_suggest_query(query, 3) == ["for Apache Cassandra", "Apache Cassandra", "Cassandra"]
    assert S.split_suggest_query(query, 2) == ["Apache Cassandra", "Cassandra"]
    assert S.split_suggest_query("Ann", 3) == ["Ann", "", ""]
    assert S.entity_groups("Solomon Isa") == ["Solomon Isa", "Isa"]
    assert S.entity_groups("a") == []
    assert S.split_suggest_query("x  y", 3) == ["x  y", "y", "y"]   # split on ' ' exactly: the empty word between the spaces counts
    assert S.entity_groups("x  y") == ["x  y"]


def test_clause_kinds_as_fuzzy_parser_rs():
    def kinds(body):
        return [k for k, _ in S.fuzzy_clauses(paragraph_query_tokens(body))]

    assert kinds("ab") == [S.TERM]                      # shorter than MIN_FUZZY_LEN: an exact term
    assert kinds("abc") == [S.FUZZY]                    # not a prefix: shorter than MIN_FUZZY_PREFIX_LEN
    assert kinds("abcd") == [S.FUZZY_PREFIX]            # the last literal
    assert kinds("abcd abcd") == [S.FUZZY, S.FUZZY_PREFIX]   # only the last literal is a prefix
    assert kinds("é") == [S.TERM] and kinds("éa") == [S.FUZZY] and kinds("éé") == [S.FUZZY_PREFIX]   # lengths in UTF-8 bytes
    assert S.fuzzy_clauses(paragraph_query_tokens('"little prince" -story "one" abcd')) == [
        (S.PHRASE, ["little", "prince"]), (S.TERM, "story"), (S.TERM, "one"), (S.FUZZY_PREFIX, "abcd")]
    assert kinds('abcd -story') == [S.FUZZY_PREFIX, S.TERM]   # an excluded word is no literal: abcd stays the last one
    assert S.ematches(paragraph_query_tokens('"little prince" -story abcd abcd')) == ["little prince", "abcd"]


def shard_docs(resources=None):
    """The golden shard's paragraphs, one segment per resource (as the binding indexes them)."""
    segs = []
    for r in resources or SM.golden_resources():
        docs = [TextDoc(r["uuid"], "/" + f, r["texts"][f][s:e], tuple(r["labels"])) for f, s, e in r["paragraphs"]]
        if docs:
            segs.append(docs)
    return segs


def ids(model, segs, hits):
    return sorted((segs[o][d].uuid, segs[o][d].field) for _, o, d in hits)


@pytest.fixture(scope="module")
def shard():
    segs = shard_docs()
    return segs, SM.SuggestModel(segs)


LP, ZA = SM.golden_resources()[0]["uuid"], SM.golden_resources()[1]["uuid"]


def run(shard, body, keep=lambda d: True, k=20):
    segs, model = shard
    masks = [np.asarray([keep(d) for d in s], dtype=bool) for s in segs]
    hits, fuzzy, matches = model.suggest(body, k, masks)
    return ids(model, segs, hits), fuzzy, matches, hits


def test_suggest_rs_paragraphs(shard):
    assert run(shard, "Nietzche")[:2] == ([(ZA, "/a/summary")], False)
    assert run(shard, "story")[:2] == ([(LP, "/a/summary")], False)
    got, fuzzy, matches, hits = run(shard, "princes")   # typo tolerant: the fuzzy prefix pass
    assert got == [(LP, "/a/summary"), (LP, "/a/title")] and fuzzy
    assert all(matches[(o, d)] == ["prince"] for _, o, d in hits)
    assert run(shard, "z")[0] == []                    # too short to be fuzzy, and no exact match
    assert run(shard, "a")[0] == [(LP, "/a/summary")]  # exact
    assert run(shard, "Hanna Adrent")[0] == []
    got, fuzzy, matches, hits = run(shard, "ann")       # suggest_features: "ann" reaches "and" at distance 1
    assert got == [(LP, "/a/summary")] and fuzzy and matches[(hits[0][1], hits[0][2])] == ["and"]


def test_suggest_rs_filters(shard):
    assert run(shard, "prince", keep=lambda d: d.field == "/a/title")[0] == [(LP, "/a/title")]
    en = lambda d: "/s/p/en" in d.labels   # noqa: E731
    assert run(shard, "prince", keep=en)[0] == [(LP, "/a/summary"), (LP, "/a/title")]
    assert run(shard, "prince", keep=lambda d: "/s/p/de" in d.labels)[0] == []
    assert run(shard, "prince", keep=lambda d: "/s/p/de" not in d.labels)[0] == [(LP, "/a/summary"), (LP, "/a/title")]
    assert run(shard, "prince", keep=lambda d: not en(d))[0] == []


def entity_model():
    docs = []
    for r in SM.golden_resources():
        for field, src, rel, dst in r["relations"]:
            docs.append(G.GraphDoc(r["uuid"], field, tuple(src), tuple(dst), rel, ""))
    return GM.Model(docs)


@pytest.mark.parametrize("body,expected", [
    ("Ann", {"Anna", "Anthony"}), ("joh", {"John"}), ("anyth", {"Anthony"}), ("anything", set()),
    ("barc", {"Barcelona", "Bárcenas"}), ("Barc", {"Barcelona", "Bárcenas"}), ("BARC", {"Barcelona", "Bárcenas"}),
    ("BÄRĈ", {"Barcelona", "Bárcenas"}), ("BáRc", {"Barcelona", "Bárcenas"}), ("Solomon Isa", {"Solomon Islands", "Israel"}),
    ("ann", {"Anna", "Anthony"}), (SM.golden_resources()[2]["uuid"][:6], set())])
def test_suggest_rs_entities(body, expected):
    req = S.entity_request(body, 20)
    got = entity_model().request(req) if req is not None else []
    assert {key[0] for key, _ in got} == expected and len(got) == len(expected)


def test_merge_suggest():
    from nucliadb_b200 import nidx_protos as P

    a = P.SuggestResponse(shard_ids=["a"], total=2, query="q", ematches=["x", "y"])
    a.results.add(uuid="u1").score.bm25 = 1.0
    a.results.add(uuid="u2").score.bm25 = 0.5
    a.entity_results.nodes.add(value="Anna")
    b = P.SuggestResponse(shard_ids=["b"], total=1, query="q", ematches=["y", "z"])
    b.results.add(uuid="u3").score.bm25 = 0.7
    b.entity_results.nodes.add(value="Anna")
    b.entity_results.nodes.add(value="John")
    m = S.merge_suggest([("a", a), ("b", b)], 2)
    assert list(m.shard_ids) == ["a", "b"] and m.total == 3 and list(m.ematches) == ["x", "y", "z"]
    assert [r.uuid for r in m.results] == ["u1", "u3"] and [r.shard_id for r in m.results] == [b"a", b"b"]
    assert [n.value for n in m.entity_results.nodes] == ["Anna", "John"]
    m = S.merge_suggest([("a", P.SuggestResponse(shard_ids=["a"])), ("b", P.SuggestResponse(shard_ids=["b"]))], 2)
    assert not m.HasField("entity_results")
    one = P.SuggestResponse(shard_ids=["a"])
    one.entity_results.SetInParent()
    assert S.merge_suggest([("a", one)], 2) is one   # one shard: its answer as it is (an empty entity_results stays present)


def test_suggest_clause_struct_has_the_header_layout(tmp_path):
    import ctypes as C
    import os
    import subprocess

    from nucliadb_b200 import _lib as L
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "l.c"
    src.write_text(f'#include <stdio.h>\n#include <stddef.h>\n#include "{root}/include/nidx_b200.h"\nint main(void) {{ printf("%zu %zu %zu", '
                   "sizeof(nidx_suggest_clause), offsetof(nidx_suggest_clause, kind), offsetof(nidx_suggest_clause, arg)); return 0; }\n")
    subprocess.run(["gcc", "-o", str(tmp_path / "l"), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(tmp_path / "l")], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(L.SuggestClause)] + [getattr(L.SuggestClause, f).offset for f, _ in L.SuggestClause._fields_]
