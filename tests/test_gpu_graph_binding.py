"""NidxSearcher.GraphSearch and SearchRequest.graph_search through the binding: two shards merged by concatenation equal the host
model's per-shard answers, security hides the relations of resources outside the caller's groups, a deletion hides a resource's
relations and a semantic (VectorMatch) leaf answers UNIMPLEMENTED."""
import uuid

import numpy as np
import pytest

from graph_model import Model
from test_graph_model import KG, node, request

pytestmark = pytest.mark.gpu


def _resource(P, rid, shard, triples, groups=None):
    res = P.Resource()
    res.resource.uuid, res.shard_id = rid, shard
    res.texts["a/title"].text = "a title"
    if groups is not None:
        res.security.SetInParent()
        res.security.access_groups.extend(groups)
    for s, lab, t in triples:
        ir = res.field_relations["a/metadata"].relations.add()
        r = ir.relation
        r.source.value, r.source.ntype, r.source.subtype = s, 0, KG["entities"][s]
        r.to.value, r.to.ntype, r.to.subtype = t, 0, KG["entities"][t]
        r.relation, r.relation_label = KG["labels"][lab], lab
        r.metadata.paragraph_id = f"{rid}/a/metadata/0-1"
        ir.facets.append("/kg")
    return res


def test_graph_search_over_two_shards(tmp_path):
    import grpc

    from nucliadb_b200 import graph as G
    from nucliadb_b200 import nidx_protos as P
    from nucliadb_b200.binding import NidxBinding

    b = NidxBinding({"INDEXER__OBJECT_STORE": "file", "INDEXER__FILE_PATH": str(tmp_path)})
    try:
        shards = [b.new_shard("kb", {}), b.new_shard("kb", {})]
        (tmp_path / "index").mkdir()
        triples = KG["triples"]
        rids = [uuid.UUID(int=i + 1).hex for i in range(4)]
        layout = [(0, rids[0], triples[:6], ["g1"]), (0, rids[1], triples[6:9], ["g2"]), (1, rids[2], triples[9:], None), (1, rids[3], triples[:2], None)]
        for n, (s, rid, ts, groups) in enumerate(layout):
            (tmp_path / f"index/{n}").write_bytes(_resource(P, rid, shards[s], ts, groups).SerializeToString())
            b.index(P.IndexMessage(shard=shards[s], resource=rid, typemessage=0, storage_key=f"index/{n}", kbid="kb").SerializeToString())
        b.index(P.IndexMessage(shard=shards[1], resource=rids[3], typemessage=1, kbid="kb").SerializeToString())   # deleted
        b.wait_for_sync()
        models = [Model([G.GraphDoc(rid, "a/metadata", (x, 0, KG["entities"][x]), (y, 0, KG["entities"][y]), KG["labels"][lab], lab, None, ("/kg",))
                         for s2, rid, ts, _ in layout[:3] if s2 == s for x, lab, y in ts]) for s in (0, 1)]
        reqs = [request(0, source=node(subtype="PERSON")), request(1, source=node("Ana", fuzzy=(1, 1)), undirected=True), request(2),
                request(0, source=node("Anna"), undirected=True)]
        channel = grpc.insecure_channel(f"127.0.0.1:{b.searcher_port}")
        call = channel.unary_unary(P.GRAPH_SEARCH_METHOD, request_serializer=lambda m: m.SerializeToString(), response_deserializer=P.GraphSearchResponse.FromString)
        for req in reqs:
            req.shard_ids.extend(shards)
            got = call(req)
            want = [h for m in models for h in m.request(req)]
            assert list(np.float32(got.scores)) == [np.float32(s) for _, s in want]
            if req.kind == 0:
                assert [(got.nodes[p.source].value, got.relations[p.relation].label, got.nodes[p.destination].value) for p in got.graph] == \
                    [(m.docs[i].source[0], m.docs[i].label, m.docs[i].target[0]) for m in models for i, _ in m.request(req)]
                assert all(p.resource_field_id.endswith("/a/metadata") and list(p.facets) == ["/kg"] and p.metadata.paragraph_id for p in got.graph)
            elif req.kind == 1:
                assert [(n.value, n.ntype, n.subtype) for n in got.nodes] == [k for k, _ in want]
            else:
                assert [(r.relation_type, r.label) for r in got.relations] == [k for k, _ in want]
        # security: only the resources of the caller's groups (and public ones) answer
        req = request(0, top_k=100)
        req.shard_ids.extend(shards)
        req.security.access_groups.append("g1")
        got = call(req)
        assert {p.resource_field_id.split("/")[0] for p in got.graph} == {rids[0], rids[2]}
        # shard 0 is a Some (the g2 resource is hidden): the all query plus the prefilter's 1.0; shard 1 is All: the all query alone
        assert [(p.resource_field_id.split("/")[0], s) for p, s in zip(got.graph, got.scores)] == \
            [(rids[0], 2.0)] * len(layout[0][2]) + [(rids[2], 1.0)] * len(layout[2][2])
        # SearchRequest.graph_search fills SearchResponse.graph
        sreq = P.SearchRequest(shard_ids=shards, result_per_page=5)
        sreq.graph_search.query.CopyFrom(reqs[0].query)
        sresp = b.search(sreq)
        assert len(sresp.graph.graph) == sum(len(m.request(request(0, source=node(subtype="PERSON"), top_k=20))) for m in models)
        # ... under the same prefilter as GraphSearch: field_filter and security (json_filter does not apply to relations)
        sreq.security.access_groups.append("g1")
        greq = P.GraphSearchRequest(kind=0, top_k=20, shard_ids=shards, query=reqs[0].query, security=sreq.security)
        assert b.search(sreq).graph.SerializeToString() == P.GraphSearchResponse(nodes=(g := call(greq)).nodes, relations=g.relations,
                                                                                  graph=g.graph, scores=g.scores).SerializeToString()
        # a field filter on a shard without text documents answers nothing, in both
        ff = P.FilterExpression()
        ff.facet.facet = "/l/x"
        lone = b.new_shard("kb", {})
        res = _resource(P, rids[3], lone, triples[:3])
        res.texts.clear()
        (tmp_path / "index/lone").write_bytes(res.SerializeToString())
        b.index(P.IndexMessage(shard=lone, resource=rids[3], typemessage=0, storage_key="index/lone", kbid="kb").SerializeToString())
        b.wait_for_sync()
        assert len(call(P.GraphSearchRequest(kind=0, top_k=20, shard_ids=[lone], query=reqs[0].query, field_filter=ff)).graph) == 0
        assert len(call(P.GraphSearchRequest(kind=0, top_k=20, shard_ids=[lone], query=reqs[0].query)).graph) == 3
        sreq = P.SearchRequest(shard_ids=[lone], result_per_page=5, field_filter=ff)
        sreq.graph_search.query.CopyFrom(reqs[0].query)
        assert len(b.search(sreq).graph.graph) == 0
        # a semantic leaf is UNIMPLEMENTED
        v = request(0, source=node("x"))
        v.query.path.path.source.vector.vector.append(1.0)
        v.shard_ids.extend(shards)
        with pytest.raises(grpc.RpcError) as e:
            call(v)
        assert e.value.code() == grpc.StatusCode.UNIMPLEMENTED
        channel.close()
    finally:
        b.close()
