"""The graph search's host model (tests/graph_model.py) against the reference's own assertions (nidx_relation/tests/
test_graph_search.rs and test_graph_query_parser_search.rs) over its knowledge graph (nidx_tests/src/graph.rs, transcribed in tests/golden/graph_knowledge.json), and the
normalisation and tokenisation the index uses."""
import json
import os

import pytest

from graph_model import Model, fuzzy_match, some_mask
from nucliadb_b200 import graph as G
from nucliadb_b200 import nidx_protos as P

KG = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "graph_knowledge.json")))
RID = "0123456789abcdef0123456789abcdef"
FULL, PREFIX, WORDS, PREFIX_WORDS = 0, 1, 2, 3
ENTITY = 0


def knowledge_docs():
    return [G.GraphDoc(RID, "a/metadata", (s, ENTITY, KG["entities"][s]), (t, ENTITY, KG["entities"][t]), KG["labels"][lab], lab)
            for s, lab, t in KG["triples"]]


def node(value=None, subtype=None, ntype=None, exact=None, fuzzy=None):
    n = P.GraphQuery.Node()
    if value is not None:
        n.value = value
    if subtype is not None:
        n.node_subtype = subtype
    if ntype is not None:
        n.node_type = ntype
    if exact is not None:
        n.exact.kind = exact
    if fuzzy is not None:
        n.fuzzy.kind, n.fuzzy.distance = fuzzy
    return n


def request(kind=G.PATH, source=None, relation=None, destination=None, undirected=False, top_k=100):
    r = P.GraphSearchRequest(kind=kind, top_k=top_k)
    p = r.query.path.path
    if source is not None:
        p.source.CopyFrom(source)
    if relation is not None:
        p.relation.CopyFrom(relation)
    if destination is not None:
        p.destination.CopyFrom(destination)
    p.undirected = undirected
    return r


@pytest.fixture(scope="module")
def model():
    return Model(knowledge_docs())


def triples(m, req):
    return {(m.docs[i].source[0], m.docs[i].label, m.docs[i].target[0]) for i, _ in m.request(req)}


def test_node_search(model):
    hits = model.request(request(G.NODES, source=node(subtype="PLACE"), undirected=True))
    assert {k[0] for k, _ in hits} == {"New York", "UK"}


def test_relation_search(model):
    rel = P.GraphQuery.Relation(relation_type=4)   # SYNONYM
    hits = model.request(request(G.RELATIONS, relation=rel))
    assert [k[1] for k, _ in hits] == ["ALIAS"]


def test_graph_node_query(model):
    anna = {("Anna", "FOLLOW", "Erin"), ("Anna", "LIVE_IN", "New York"), ("Anna", "LOVE", "Cat"), ("Anna", "WORK_IN", "New York")}
    assert triples(model, request(source=node("Anna"))) == anna
    assert len(model.request(request(source=node(subtype="PERSON")))) == 12
    assert triples(model, request(destination=node("Anna", "PERSON", ENTITY))) == {("Anastasia", "IS_FRIEND", "Anna")}
    assert triples(model, request(source=node("Anna", "PERSON", ENTITY), undirected=True)) == anna | {("Anastasia", "IS_FRIEND", "Anna")}


@pytest.mark.parametrize("value,kind", [("Computer science", FULL), ("Computer sci", PREFIX), ("Compu", PREFIX), ("Computer", WORDS),
                                        ("science", WORDS), ("sci", PREFIX_WORDS)])
def test_graph_node_exact_matches(model, value, kind):
    assert triples(model, request(destination=node(value, exact=kind))) == {("Margaret", "WORK_IN", "Computer science")}


def test_graph_fuzzy_node_query(model):
    friend = {("Anastasia", "IS_FRIEND", "Anna")}
    assert triples(model, request(source=node("Anastas", "PERSON", fuzzy=(PREFIX, 1)))) == friend
    assert triples(model, request(source=node("AnXstXsia", "PERSON", fuzzy=(FULL, 1)))) == set()
    assert triples(model, request(source=node("AnXstasia", "PERSON", fuzzy=(FULL, 1)))) == friend
    assert len(model.request(request(source=node("Ana", "PERSON", fuzzy=(PREFIX, 1))))) == 5


@pytest.mark.parametrize("value,kind", [("Computer scXence", FULL), ("CompuXer sci", PREFIX), ("CoXpu", PREFIX), ("ComXuter", WORDS),
                                        ("sciXnce", WORDS), ("scXen", PREFIX_WORDS)])
def test_graph_node_fuzzy_matches(model, value, kind):
    assert triples(model, request(destination=node(value, fuzzy=(kind, 1)))) == {("Margaret", "WORK_IN", "Computer science")}


def test_not_and_or_and_the_all_query(model):
    r = request()
    r.query.path.bool_not.path.source.value = "Anna"
    assert len(model.request(r)) == len(KG["triples"]) - 4
    r = P.GraphSearchRequest(kind=G.PATH, top_k=100)
    for v in ("Tom", "Jerry"):
        r.query.path.bool_or.operands.add().path.source.value = v
    assert triples(model, r) == {("Tom", "CHASE", "Jerry"), ("Tom", "IS", "Cat"), ("Jerry", "IS", "Mouse")}
    assert len(model.request(P.GraphSearchRequest(kind=G.PATH, top_k=100, query=P.GraphQuery(path=P.GraphQuery.PathQuery())))) == len(KG["triples"])


def test_scores_and_ties(model):
    hits = model.request(request(source=node("Anna"), top_k=2))
    assert len(hits) == 2 and hits[0][1] == hits[1][1] and hits[0][0] < hits[1][0]   # equal BM25 scores: lower document first
    assert hits[0][1] == G.leaf_score(len(KG["triples"]), 4)
    # a Some prefilter adds 1.0 ahead of the query
    some = model.request(request(source=node("Anna"), top_k=2), some_mask=[True] * len(KG["triples"]))
    assert some[0][1] == G.leaf_score(len(KG["triples"]), 4) + 1


@pytest.mark.parametrize("raw,norm", [("New  York", "new york"), ("Café Olé", "cafe ole"), ("ÀÉÎÕÜ ñ", "aeiou n"), ("MR. P", "mr. p"),
                                      ("Straße", "straße"), ("日本 東京", "日本 東京"), ("  tab\tsep\n", "tab sep")])
def test_normalize(raw, norm):
    assert G.normalize(raw) == norm


def test_tokens_are_the_default_analyzer():
    from nucliadb_b200.text import tokenize

    assert tokenize("Computer science") == ["computer", "science"]
    assert tokenize("Mr. P") == ["mr", "p"]
    assert tokenize("Ünïcode-wörds") == ["ünïcode", "wörds"]


@pytest.mark.parametrize("term,entry,d,prefix,want", [("abc", "abc", 0, False, True), ("abc", "acb", 1, False, True), ("abc", "ca", 1, False, False),
                                                      ("abc", "abcdef", 0, True, True), ("abd", "abcdef", 1, True, True), ("abc", "xbcdef", 0, True, False),
                                                      ("ab", "", 2, False, True), ("ab", "", 2, True, True), ("über", "uber", 1, False, True)])
def test_restricted_damerau_levenshtein(term, entry, d, prefix, want):
    assert fuzzy_match(term, entry, d, prefix) is want


def test_parser_rejections():
    with pytest.raises(ValueError):
        G.node_query(request(G.NODES, source=node("x")).query.path, "src")   # a NODES path must be undirected
    with pytest.raises(ValueError):
        G.path_query(request(source=node("x", fuzzy=(FULL, 3))).query.path)
    v = node("x")
    v.vector.vector.append(1.0)
    with pytest.raises(NotImplementedError):
        G.path_query(request(source=v).query.path)


# ---- the rest of test_graph_search.rs and test_graph_query_parser_search.rs -------------------------------------------------------
# The parser tests build Expression::Not / Expression::Or of relations and nodes directly; a GraphSearchRequest cannot express those
# forms, so their assertions are restated through the request forms that give the same queries' sets (bool_not, bool_or).
def _rel(value=None, rtype=None):
    r = P.GraphQuery.Relation()
    if value is not None:
        r.value = value
    if rtype is not None:
        r.relation_type = rtype
    return r


def _pq(source=None, relation=None, destination=None, undirected=False):
    return request(G.PATH, source, relation, destination, undirected).query.path


def _run(m, pq, prefilter="all", kind=G.PATH):
    """A PATH request under a prefilter: "all", "none" or a Some's [(resource hex, field path)]."""
    r = P.GraphSearchRequest(kind=kind, top_k=100)
    r.query.path.CopyFrom(pq)
    if prefilter == "none":
        return []
    mask = None if prefilter == "all" else some_mask(m.docs, prefilter)
    return m.request(r, some_mask=mask)


def _triples(m, hits):
    return {(m.docs[i].source[0], m.docs[i].label, m.docs[i].target[0]) for i, _ in hits}


def test_graph_relation_query(model):
    assert _triples(model, _run(model, _pq(relation=_rel("LIVE_IN")))) == {("Anna", "LIVE_IN", "New York"), ("Peter", "LIVE_IN", "New York")}
    assert _triples(model, _run(model, _pq(relation=_rel(rtype=4)))) == {("Mr. P", "ALIAS", "Peter")}
    assert _run(model, _pq(relation=_rel("FAKE", 4))) == []
    q = P.GraphQuery.PathQuery()
    q.bool_or.operands.add().CopyFrom(_pq(relation=_rel("LIVE_IN")))
    q.bool_or.operands.add().CopyFrom(_pq(relation=_rel("BORN_IN")))
    assert _triples(model, _run(model, q)) == {("Anna", "LIVE_IN", "New York"), ("Erin", "BORN_IN", "UK"), ("Peter", "LIVE_IN", "New York")}
    q = P.GraphQuery.PathQuery()
    q.bool_not.CopyFrom(_pq(relation=_rel("LIVE_IN")))
    assert len(_run(model, q)) == 15


def test_graph_directed_path_query(model):
    assert len(_run(model, _pq())) == 17
    assert _triples(model, _run(model, _pq(source=node("Erin", "PERSON", ENTITY), destination=node("UK", "PLACE", ENTITY)))) == {("Erin", "BORN_IN", "UK")}
    person_place = {("Anna", "LIVE_IN", "New York"), ("Anna", "WORK_IN", "New York"), ("Erin", "BORN_IN", "UK"), ("Peter", "LIVE_IN", "New York")}
    assert _triples(model, _run(model, _pq(source=node(subtype="PERSON", ntype=ENTITY), destination=node(subtype="PLACE", ntype=ENTITY)))) == person_place
    assert _triples(model, _run(model, _pq(source=node(subtype="PERSON"), destination=node(subtype="PLACE")))) == person_place   # parser test
    live = {("Anna", "LIVE_IN", "New York"), ("Peter", "LIVE_IN", "New York")}
    assert _triples(model, _run(model, _pq(source=node(subtype="PERSON", ntype=ENTITY), relation=_rel("LIVE_IN"),
                                           destination=node(subtype="PLACE", ntype=ENTITY)))) == live
    q = P.GraphQuery.PathQuery()
    either = q.bool_and.operands.add()
    either.bool_or.operands.add().CopyFrom(_pq(relation=_rel("LIVE_IN")))
    either.bool_or.operands.add().CopyFrom(_pq(relation=_rel("LOVE")))
    q.bool_and.operands.add().bool_not.CopyFrom(_pq(source=node("Anna")))
    assert _triples(model, _run(model, q)) == {("Erin", "LOVE", "Climbing"), ("Dimitri", "LOVE", "Anastasia"), ("Peter", "LIVE_IN", "New York")}


def test_graph_undirected_path_query(model):
    assert _triples(model, _run(model, _pq(source=node("Anna", "PERSON", ENTITY), relation=_rel("IS_FRIEND"), undirected=True))) == \
        {("Anastasia", "IS_FRIEND", "Anna")}


def test_graph_response(model):
    import types

    q = P.GraphQuery.PathQuery()
    q.bool_or.operands.add().CopyFrom(_pq(relation=_rel("LIVE_IN")))
    q.bool_or.operands.add().CopyFrom(_pq(relation=_rel("WORK_IN")))
    resp = G.GraphSearcher(types.SimpleNamespace(docs=model.docs)).response(G.PATH, _run(model, q))
    paths = {(resp.nodes[p.source].value, resp.relations[p.relation].label, resp.nodes[p.destination].value) for p in resp.graph}
    assert paths == {("Anna", "LIVE_IN", "New York"), ("Anna", "WORK_IN", "New York"), ("Margaret", "WORK_IN", "Computer science"),
                     ("Peter", "LIVE_IN", "New York")}
    assert len(resp.graph) == 4 and len(resp.nodes) == 8 and len(resp.relations) == 4   # no dedup, as the reference
    assert all(p.resource_field_id == f"{RID}/a/metadata" for p in resp.graph)


def test_prefilter(model):
    nil = "00000000000000000000000000000000"
    assert len(_run(model, _pq(), "all")) == 17
    assert _run(model, _pq(), "none") == []
    assert _run(model, _pq(), [(nil, "/f/fake")]) == []
    assert len(_run(model, _pq(), [(RID, "/a/metadata")])) == 17
    assert len(_run(model, _pq(), [(RID, "/f/fake")])) == 17   # a listed resource admits its a/metadata relations
    assert all(s == 2.0 for _, s in _run(model, _pq(), [(RID, "/f/fake")]))   # the all query 1.0 + the prefilter 1.0


def test_prefilter_file_field():
    docs = [G.GraphDoc(d.rid, "f/my_file", d.source, d.target, d.rel_type, d.label) for d in knowledge_docs()]
    m = Model(docs)
    assert len(_run(m, _pq(), "all")) == 17
    assert _run(m, _pq(), "none") == []
    assert _run(m, _pq(), [(RID, "/f/fake")]) == []   # another field of the resource admits only a/metadata relations
    assert len(_run(m, _pq(), [(RID, "/f/my_file")])) == 17


def test_facet_filter():
    docs = [G.GraphDoc(RID, "a/metadata", ("Peter Processor", ENTITY, "PERSON"), ("Pedro Procesador", ENTITY, "PERSON"), 2, "SAME"),
            G.GraphDoc(RID, "a/metadata", ("Ursula User", ENTITY, "PERSON"), ("Úrsula Usuaria", ENTITY, "PERSON"), 2, "SAME", None, ("/g/u",)),
            G.GraphDoc(RID, "a/metadata", ("Alfred Agent", ENTITY, "PERSON"), ("Alfred Agente", ENTITY, "PERSON"), 2, "SAME", None, ("/g/da/mytask",))]
    m = Model(docs)
    for facet, want in [("/g/u", ["Ursula User"]), ("/g/da", ["Alfred Agent"]), ("/g/da/mytask", ["Alfred Agent"]), ("/g/da/faketask", [])]:
        q = P.GraphQuery.PathQuery()
        q.facet.facet = facet
        assert [m.docs[i].source[0] for i, _ in _run(m, q)] == want


def test_parser_node_queries(model):
    assert len(_run(model, _pq(source=node()))) == 17
    assert len(_run(model, _pq(source=node(subtype="PERSON", ntype=ENTITY)))) == 12
    assert len(_run(model, _pq(source=node("Anna", "PERSON", ENTITY)))) == 4
    assert len(_run(model, _pq(destination=node("Anna", "PERSON", ENTITY)))) == 1
    assert len(_run(model, _pq(source=node("Anna", "PERSON", ENTITY), undirected=True))) == 5


@pytest.mark.parametrize("value,fuzzy,want", [("Anastas", (FULL, 2), 1), ("AnXstXsia", (FULL, 1), 0), ("AnXstXsia", (FULL, 2), 1),
                                              ("Anas", (PREFIX, 0), 1), ("Anas", (PREFIX, 2), 5)])
def test_parser_fuzzy_node_queries(model, value, fuzzy, want):
    assert len(_run(model, _pq(source=node(value, fuzzy=fuzzy)))) == want
