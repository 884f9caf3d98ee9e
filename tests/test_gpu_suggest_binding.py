"""NidxSearcher.Suggest through NidxBinding and gRPC on localhost, over the golden shard (the resources of the reference's
tests/integration/suggest.rs): every assertion of that file, a two-shard merge, the empty plans and an unknown shard."""
import pytest

import suggest_model as SM

pytestmark = pytest.mark.gpu


def _resource(P, r, shard, groups=None, json_fields=None):
    import json

    res = P.Resource()
    res.resource.uuid, res.shard_id = r["uuid"], shard
    if groups is not None:
        res.security.SetInParent()
        res.security.access_groups.extend(groups)
    for f, v in (json_fields or {}).items():
        res.json_fields[f].value = json.dumps(v)
    res.labels.extend(r["labels"])
    for f, text in r["texts"].items():
        res.texts[f].text = text
    for f, s, e in r["paragraphs"]:
        p = res.paragraphs[f].paragraphs[f"{r['uuid']}/{f}/{s}-{e}"]
        p.start, p.end, p.field = s, e, f
    for field, src, rel, dst in r["relations"]:
        x = res.field_relations[field].relations.add().relation
        x.source.value, x.source.ntype, x.source.subtype = src
        x.to.value, x.to.ntype, x.to.subtype = dst
        x.relation = rel
    return res


@pytest.fixture(scope="module")
def binding(tmp_path_factory):
    from nucliadb_b200 import nidx_protos as P
    from nucliadb_b200.binding import NidxBinding

    tmp = tmp_path_factory.mktemp("suggest")
    b = NidxBinding({"INDEXER__OBJECT_STORE": "file", "INDEXER__FILE_PATH": str(tmp)})
    shards = [b.new_shard("kb", {}), b.new_shard("kb", {}), b.new_shard("kb", {})]
    rs = SM.golden_resources()
    # shard 2: the little prince in access group g1 with a JSON document, the people and places resource public without one
    layout = [(0, rs[0], {}), (0, rs[1], {}), (0, rs[2], {}), (1, rs[0], {}), (2, rs[0], dict(groups=["g1"], json_fields={"t/p": {"lang": "en"}})),
              (2, rs[2], {})]
    for n, (s, r, kw) in enumerate(layout):
        (tmp / f"r{n}").write_bytes(_resource(P, r, shards[s], **kw).SerializeToString())
        b.index(P.IndexMessage(shard=shards[s], resource=r["uuid"], typemessage=0, storage_key=f"r{n}", kbid="kb").SerializeToString())
    b.wait_for_sync()
    yield b, shards
    b.close()


def _call(b, P):
    import grpc

    channel = grpc.insecure_channel(f"127.0.0.1:{b.searcher_port}")
    return channel.unary_unary(P.SUGGEST_METHOD, request_serializer=lambda m: m.SerializeToString(), response_deserializer=P.SuggestResponse.FromString)


def _fields(resp):
    return sorted((r.uuid, r.field) for r in resp.results)


LP, ZA, PAP = (r["uuid"] for r in SM.golden_resources())


def test_suggest_rs_paragraphs_and_entities(binding):
    from nucliadb_b200 import nidx_protos as P

    b, shards = binding
    call = _call(b, P)

    def par(body, **kw):
        req = P.SuggestRequest(shard_ids=[shards[0]], body=body, top_k=20, features=[P.SUGGEST_PARAGRAPHS], **kw)
        got = b.suggest(req)
        assert got == call(req)
        assert got.total == len(got.results) and not got.HasField("entity_results") and got.query == body
        return _fields(got)

    assert par("Nietzche") == [(ZA, "/a/summary")]
    assert par("story") == [(LP, "/a/summary")]
    assert par("princes") == [(LP, "/a/summary"), (LP, "/a/title")]
    assert par("z") == [] and par("Hanna Adrent") == []
    assert par("a") == [(LP, "/a/summary")] and par("ann") == [(LP, "/a/summary")]
    field = P.FilterExpression()
    field.field.field_type, field.field.field_id = "a", "title"
    assert par("prince", field_filter=field) == [(LP, "/a/title")]
    en, de = P.FilterExpression(), P.FilterExpression()
    en.facet.facet, de.facet.facet = "/s/p/en", "/s/p/de"
    not_en, not_de = P.FilterExpression(), P.FilterExpression()
    not_en.bool_not.CopyFrom(en)
    not_de.bool_not.CopyFrom(de)
    assert par("prince", field_filter=en) == [(LP, "/a/summary"), (LP, "/a/title")] and par("prince", field_filter=de) == []
    assert par("prince", field_filter=not_de) == [(LP, "/a/summary"), (LP, "/a/title")] and par("prince", field_filter=not_en) == []
    assert par("prince", paragraph_filter=de) == [] and par("prince", paragraph_filter=en) == [(LP, "/a/summary"), (LP, "/a/title")]
    assert par("prince", paragraph_filter=de, field_filter=en, filter_operator=P.FILTER_OR) == [(LP, "/a/summary"), (LP, "/a/title")]
    assert par("prince", paragraph_filter=de, field_filter=en) == []
    got = b.suggest(P.SuggestRequest(shard_ids=[shards[0]], body="princes", top_k=20, features=[P.SUGGEST_PARAGRAPHS]))
    assert all(list(r.matches) == ["prince"] and r.paragraph.startswith(LP) for r in got.results) and list(got.ematches) == ["princes"]

    def ent(body):
        req = P.SuggestRequest(shard_ids=[shards[0]], body=body, top_k=20, features=[P.SUGGEST_ENTITIES])
        got = b.suggest(req)
        assert got == call(req) and got.HasField("entity_results") and got.total == 0 and not got.results
        return sorted(n.value for n in got.entity_results.nodes)

    assert ent("Ann") == ["Anna", "Anthony"] and ent("joh") == ["John"] and ent("anyth") == ["Anthony"] and ent("anything") == []
    for body in ("barc", "Barc", "BARC", "BÄRĈ", "BáRc"):
        assert ent(body) == ["Barcelona", "Bárcenas"]
    assert ent("Solomon Isa") == ["Israel", "Solomon Islands"] and ent("ann") == ["Anna", "Anthony"] and ent(PAP[:6]) == []


def test_two_shards_empty_plans_and_unknown_shard(binding):
    import grpc

    from nucliadb_b200 import nidx_protos as P

    b, shards = binding
    call = _call(b, P)
    shards = shards[:2]
    req = P.SuggestRequest(shard_ids=shards, body="prince", top_k=20, features=[P.SUGGEST_PARAGRAPHS, P.SUGGEST_ENTITIES])
    got = call(req)
    one = [b.suggest(P.SuggestRequest(shard_ids=[s], body="prince", top_k=20, features=[P.SUGGEST_PARAGRAPHS, P.SUGGEST_ENTITIES])) for s in shards]
    assert list(got.shard_ids) == shards and got.total == 4 and len(got.results) == 4
    assert sorted((r.shard_id, r.uuid, r.field) for r in got.results) == sorted((s.encode(), r.uuid, r.field) for s, o in zip(shards, one) for r in o.results)
    scores = [r.score.bm25 for r in got.results]
    assert scores == sorted(scores, reverse=True)
    assert not got.HasField("entity_results")   # no shard found a node
    got = call(P.SuggestRequest(shard_ids=shards, body="prince", top_k=1, features=[P.SUGGEST_PARAGRAPHS]))
    assert len(got.results) == 1 and got.total == 2
    for req in (P.SuggestRequest(shard_ids=shards, body="prince", top_k=0, features=[P.SUGGEST_PARAGRAPHS, P.SUGGEST_ENTITIES]),
                P.SuggestRequest(shard_ids=shards, body="prince", top_k=20)):
        got = call(req)
        assert got.total == 0 and not got.results and not got.HasField("entity_results") and got.query == ""
    with pytest.raises(grpc.RpcError) as e:
        call(P.SuggestRequest(shard_ids=["nope"], body="prince", top_k=20, features=[P.SUGGEST_PARAGRAPHS]))
    assert e.value.code() == grpc.StatusCode.NOT_FOUND
    with pytest.raises(grpc.RpcError) as e:
        call(P.SuggestRequest(shard_ids=shards, body="prince", top_k=2000, features=[P.SUGGEST_PARAGRAPHS]))
    assert e.value.code() == grpc.StatusCode.INVALID_ARGUMENT


def test_security_and_json_filter(binding):
    from nucliadb_b200 import nidx_protos as P
    from test_json_model import path

    b, shards = binding
    call = _call(b, P)
    both = [P.SUGGEST_PARAGRAPHS, P.SUGGEST_ENTITIES]

    def ask(body="prince", security=None, json_filter=None, field_filter=None, op_or=False, features=both):
        req = P.SuggestRequest(shard_ids=[shards[2]], body=body, top_k=20, features=features, filter_operator=P.FILTER_OR if op_or else P.FILTER_AND)
        if security is not None:
            req.security.SetInParent()
            req.security.access_groups.extend(security)
        if json_filter is not None:
            req.json_filter.CopyFrom(json_filter)
        if field_filter is not None:
            req.field_filter.CopyFrom(field_filter)
        got = b.suggest(req)
        assert got == call(req)
        return got

    both_fields = [(LP, "/a/summary"), (LP, "/a/title")]
    assert _fields(ask()) == both_fields
    assert _fields(ask(security=["g1"])) == both_fields and _fields(ask(security=["g1/sub"])) == []
    assert _fields(ask(security=[])) == [] and _fields(ask(body="princes", security=["other"])) == []
    # entities follow the text prefilter: the public resource's relations stay visible, the grouped one has none
    assert sorted(n.value for n in ask(body="Ann", security=[]).entity_results.nodes) == ["Anna", "Anthony"]
    en, de = path("t/p", "lang", text="en"), path("t/p", "lang", text="de")
    assert _fields(ask(json_filter=en)) == both_fields and _fields(ask(body="princes", json_filter=en)) == both_fields
    got = ask(json_filter=de)   # a None prefilter empties everything, entities included
    assert got == P.SuggestResponse(shard_ids=[shards[2]])
    got = ask(body="Ann", json_filter=de, features=[P.SUGGEST_ENTITIES])
    assert not got.HasField("entity_results")
    # json_filter does not apply to entities: a Some from JSON alone leaves them all
    assert sorted(n.value for n in ask(body="Ann", json_filter=en).entity_results.nodes) == ["Anna", "Anthony"]
    title = P.FilterExpression()
    title.field.field_type, title.field.field_id = "a", "title"
    assert _fields(ask(json_filter=de, field_filter=title, op_or=True)) == [(LP, "/a/title")]
    assert _fields(ask(json_filter=en, field_filter=title)) == [(LP, "/a/title")]
    assert _fields(ask(json_filter=en, field_filter=title, security=["g2"])) == []
    assert _fields(ask(json_filter=en, field_filter=title, security=["g1"], op_or=True)) == both_fields
