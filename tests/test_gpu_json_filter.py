"""SearchRequest.json_filter on the device: the JSON prefilter's document and resource bits against tests/json_model.py bit for bit
(padding words included) on random nested JSON, the vector hand-off and the paragraph mask against host restatements, and the whole
path over gRPC through NidxBinding."""
import json
import random
import uuid

import numpy as np
import pytest

import json_model as M
from test_json_model import INTEGRATION, op, path

pytestmark = pytest.mark.gpu

KEYS = ["a", "b", "c", "d.e"]
WORDS = ["red", "Red", "apple", "2024-01-01T00:00:00Z", "2020-05-05T10:00:00+02:00", ""]


def _value(rng, depth):
    r = rng.random()
    if depth < 2 and r < 0.2:
        return {k: _value(rng, depth + 1) for k in rng.sample(KEYS, rng.randint(0, 3))}
    if depth < 2 and r < 0.3:
        return [_value(rng, depth + 1) for _ in range(rng.randint(0, 3))]
    if r < 0.45:
        return rng.randint(-5, 5)
    if r < 0.6:
        return rng.choice([-2.5, 0.0, 1.0, 3.25, 1e30])
    if r < 0.7:
        return rng.random() < 0.5
    if r < 0.75:
        return None
    return rng.choice(WORDS)


def _corpus(seed, n):
    rng = random.Random(seed)
    docs = []
    for i in range(n):
        rid = uuid.UUID(int=rng.randrange(max(n // 2, 1)) + 1).hex    # some resources have several documents
        doc = {f: {k: _value(rng, 1) for k in rng.sample(KEYS, rng.randint(0, 4))} for f in rng.sample(["t/p", "t/q"], rng.randint(1, 2))}
        docs.append((rid, doc))
    return docs


def _exprs():
    leaves = [path("t/p", "a", int=1), path("t/p", "a", float=1.0), path("t/p", "b", int_range=(-2, 3)), path("t/p", "b", int_range=(None, 0)),
              path("t/q", "c", float_range=(0.5, None)), path("t/p", "a", boolean=True), path("t/p", "c", text="red"),
              path("t/q", "a", text="Red"), path("t/p", "d\\.e", date=1704067200), path("t/p", "a", date_range=(1588665600, None)),
              path("t/p", "nothere", int=1), path("t/p", "b.a", int_range=(None, None))]
    return leaves + [op("and", leaves[0], leaves[2]), op("or", leaves[4], leaves[6], leaves[8]), op("not", leaves[5]),
                     op("not", op("or", leaves[1], op("and", leaves[3], op("not", leaves[7])))), op("and"), op("or")]


def _index(docs, alive, device=0):
    from nucliadb_b200 import json_index as J

    keep = [d for d, a in zip(docs, alive) if a]
    return J.JsonIndex([(r, J.flatten({f: json.dumps(v) for f, v in doc.items()}), ()) for r, doc in keep], device=device), keep


def _words(mask):
    w = np.zeros((len(mask) + 63) // 64 * 8, dtype=np.uint8)
    b = np.packbits(np.asarray(mask, dtype=bool), bitorder="little")
    w[: len(b)] = b
    return w.view(np.uint64)


@pytest.mark.parametrize("n", [1, 1000, 200_003])
def test_json_prefilter_matches_the_model(n):
    docs = _corpus(n, n)
    alive = [random.Random(n + 1).random() > 0.1 for _ in docs] if n > 1 else [True]
    ix, keep = _index(docs, alive)
    exprs = _exprs() if n <= 1000 else _exprs()[12:16]
    for e in exprs:
        want = [M.matches(doc, e) for _, doc in keep]
        want_res = {r for (r, _), m in zip(keep, want) if m}
        for on_device in (True, False):
            bits, matching, res = ix.prefilter(e, on_device=on_device)
            bits = bits.cpu().numpy().view(np.uint64) if on_device else bits
            res = res.cpu().numpy().view(np.uint64) if on_device else res
            assert np.array_equal(bits, _words(want)), (n, e)
            assert matching == sum(want)
            assert np.array_equal(res[: (len(ix.resource_ids) + 63) // 64], _words([r in want_res for r in ix.resource_ids])[: (len(ix.resource_ids) + 63) // 64])
    ix.close()


def test_combined_result_hand_off_and_paragraph_mask_match_host_restatements():
    """A resource whose vectors belong to a field with no text document still passes at resource level."""
    import torch

    from nucliadb_b200 import text as T
    from nucliadb_b200 import vector as V

    rng = np.random.default_rng(3)
    rids = [uuid.UUID(int=i + 7).hex for i in range(40)]
    elems, tdocs, pdocs = [], [], []
    for i, r in enumerate(rids):
        for f in ("a/title", "t/extra"):
            elems += [V.Elem(f"{r}/{f}/{j}-{j + 5}", [rng.standard_normal(8).astype(np.float32)], labels=[f"/l/x{i % 3}"]) for j in range(2)]
            pdocs.append(T.TextDoc(r, "/" + f, "fox words" + " fox" * (i % 3), labels=(f"/l/x{i % 3}", f"/l/y{i % 2}")))
        tdocs.append(T.TextDoc(r, "/a/title", f"fox {i}", labels=(f"/l/x{i % 3}",)))   # no text document for t/extra
    seg = V.OpenSegment.create(elems, V.VectorConfig(dimension=8))
    ts = T.TextSearcher.open([tdocs])
    ps = T.ParagraphSearcher.open([pdocs])
    copy = T.ParagraphSearcher.open([pdocs])
    jdocs = [(r, {"t/p": {"v": i % 4}}) for i, r in enumerate(rids) if i % 5]
    ix, keep = _index(jdocs, [True] * len(jdocs))
    for e in (path("t/p", "v", int_range=(1, 2)), op("not", path("t/p", "v", int=1))):
        res = M.resources(keep, e)
        _, found, res_bits = ix.prefilter(e)
        for ff, op_or in (("/l/x1", False), ("/l/x1", True), (None, False), ("/l/none", True)):
            expr = None
            if ff is not None:
                from nucliadb_b200 import nidx_protos as P
                expr = P.FilterExpression()
                expr.facet.facet = ff
            text = ts.prefilter(expr) if expr is not None else V.PrefilterResult.all()
            tset = text.kind if text.kind in ("all", "none") else {(uuid.UUID(str(f.resource_id)).hex, f.field_id) for f in text.fields}
            want = M.combine(tset, res, op_or)
            assert want not in ("all", "none")
            pf = text.combine(ix, res_bits, found, op_or)
            got = V.VectorSearcher(seg.config, [seg]).search(V.VectorSearchRequest(vector=[0.1] * 8, result_per_page=len(elems), min_score=-1e9,
                                                                                    with_duplicates=True), pf)
            got_keys = {d.doc_id for d in got.documents}
            want_keys = {k.key for k in elems if M.admits(want, k.key.split("/")[0], "/" + "/".join(k.key.split("/")[1:3]))}
            assert got_keys == want_keys, (e, ff, op_or)
            masks = ps.json_masks(None, pf)
            m = masks[0].cpu().numpy().view(np.uint64)
            want_m = [M.admits(want, d.uuid, d.field) for d in ps.segments[0].docs]
            assert np.array_equal(m, _words(want_m)), (e, ff, op_or)
            # the view equals a copy of the segment whose alive bits are alive AND mask: ids, score bits, totals, facet counts
            copy.segments[0].set_alive(np.asarray(want_m, dtype=bool))
            req = T.DocumentSearchRequest(body="fox words", result_per_page=100, faceted=["/l"])
            vr = ps.search(req, masks=masks)
            cr = copy.search(req)
            assert vr.total == cr.total == sum(want_m) and vr.next_page == cr.next_page
            assert [(r.uuid, r.field, np.float32(r.score.bm25).tobytes(), r.score.docaddr) for r in vr.results] == \
                   [(r.uuid, r.field, np.float32(r.score.bm25).tobytes(), r.score.docaddr) for r in cr.results]
            assert vr.facets == cr.facets
    ix.close()
    torch.cuda.synchronize()


def test_binding_honours_json_filter_end_to_end(tmp_path):
    import grpc

    from nidx_binding import NidxBinding
    from nucliadb_b200 import nidx_protos as P
    from nucliadb_b200.vector import VectorConfig

    dim = 3
    binding = NidxBinding({"INDEXER__OBJECT_STORE": "file", "INDEXER__FILE_PATH": str(tmp_path)})
    shard = binding.new_shard("kb", {"english": VectorConfig(dimension=dim)})
    (tmp_path / "index").mkdir()
    rids = [uuid.UUID(int=i + 501).hex for i in range(4)]
    names = {"apple": 0, "banana": 1, "hammer": 2}

    def index(i, price, category, available, key, groups=None, skip=False, delete=()):
        res = P.Resource()
        res.resource.uuid, res.shard_id = rids[i], shard
        if groups:
            res.security.SetInParent()
            res.security.access_groups.extend(groups)
        if price is not None:
            res.json_fields["t/product"].value = json.dumps({"price": price, "category": category, "available": available})
        res.skip_json = skip
        res.json_fields_to_delete.extend(delete)
        res.texts["a/title"].text = f"{category} item"
        pid = f"{rids[i]}/a/title/0-20"
        par = res.paragraphs["a/title"].paragraphs[pid]
        par.start, par.end = 0, 20
        par.sentences[pid].vector.extend([0.1 * (i + 1), 0.2, 0.3])
        (tmp_path / f"index/{key}").write_bytes(res.SerializeToString())
        binding.index(P.IndexMessage(shard=shard, resource=rids[i], typemessage=0, storage_key=f"index/{key}", kbid="kb").SerializeToString())

    index(0, 150, "fruit", True, "0", ["engineering"])
    index(1, 80, "fruit", False, "1", ["other"])
    index(2, 200, "tool", True, "2", ["engineering"])
    binding.wait_for_sync()
    chan = grpc.insecure_channel(f"127.0.0.1:{binding.searcher_port}")
    search = chan.unary_unary(P.SEARCH_METHOD, request_serializer=lambda m: m.SerializeToString(), response_deserializer=P.SearchResponse.FromString)

    def request(e=None, security=None, op_or=False, field_filter=None):
        req = P.SearchRequest(shard_ids=[shard], body="item", paragraph=True, document=True, result_per_page=10, vector=[0.1, 0.2, 0.3], vectorset="english",
                              min_score_semantic=-1e9, with_duplicates=True, filter_operator=P.FILTER_OR if op_or else P.FILTER_AND)
        if e is not None:
            req.json_filter.CopyFrom(e)
        if security is not None:
            req.security.SetInParent()
            req.security.access_groups.extend(security)
        if field_filter is not None:
            req.field_filter.resource.resource_id = field_filter
        return req

    def got(resp):
        return {r.uuid for r in resp.paragraph.results}, {d.doc_id.id.split("/")[0] for d in resp.vector.documents}

    for name, e, want in INTEGRATION:
        resp = search(request(e))
        want_ids = {rids[names[w]] for w in want}
        if not want:   # the None case: the vector, paragraph and document sections are absent
            assert not resp.HasField("paragraph") and not resp.HasField("vector") and not resp.HasField("document"), name
            continue
        assert got(resp) == (want_ids, want_ids), name
    fruit = path("t/product", "category", text="fruit")
    assert got(search(request(fruit, ["engineering"]))) == ({rids[0]}, {rids[0]})
    # a request without json_filter answers as on a shard without JSON data, byte for byte (shard ids aside)
    plain = NidxBinding({"INDEXER__OBJECT_STORE": "file", "INDEXER__FILE_PATH": str(tmp_path)})
    plain_shard = plain.new_shard("kb", {"english": VectorConfig(dimension=dim)})
    for i, grp in enumerate((["engineering"], ["other"], ["engineering"])):
        res = P.Resource.FromString((tmp_path / f"index/{i}").read_bytes())
        res.shard_id = plain_shard
        res.ClearField("json_fields")
        (tmp_path / f"index/plain{i}").write_bytes(res.SerializeToString())
        plain.index(P.IndexMessage(shard=plain_shard, resource=rids[i], typemessage=0, storage_key=f"index/plain{i}", kbid="kb").SerializeToString())
    plain.wait_for_sync()

    def normalised(resp):
        resp.ClearField("shard_ids")
        for r in list(resp.document.results) + list(resp.paragraph.results):
            r.ClearField("shard_id")
        return resp.SerializeToString()

    for sec, ff, op_or in ((None, None, False), (["engineering"], None, False), (None, rids[2], True), (["other"], rids[1], False)):
        a, b = request(None, sec, op_or, ff), request(None, sec, op_or, ff)
        b.shard_ids[:] = [plain_shard]
        b.faceted.labels.append("/l")
        a.faceted.labels.append("/l")
        assert normalised(search(a)) == normalised(plain.search(b)), (sec, ff, op_or)
    plain.close()
    # security is never widened under OR: banana matches the JSON filter but is outside the groups
    p, v = got(search(request(fruit, ["engineering"], op_or=True, field_filter=rids[2])))
    assert rids[1] not in p and rids[1] not in v and rids[0] in v and rids[2] in v
    # an empty JSON set under OR keeps the text result, for the paragraph search too: only the field_filter's resource
    assert got(search(request(path("t/product", "category", text="vegetable"), op_or=True, field_filter=rids[2]))) == ({rids[2]}, {rids[2]})
    with pytest.raises(grpc.RpcError) as err:
        search(request(P.JsonFilterExpression()))
    assert err.value.code() == grpc.StatusCode.INVALID_ARGUMENT
    # skip_json keeps the old document; json_fields_to_delete drops it, and a re-index brings the new one
    index(0, 999, "tool", True, "0b", ["engineering"], skip=True)
    binding.wait_for_sync()
    assert rids[0] in got(search(request(fruit)))[0]
    index(0, 999, "tool", True, "0c", ["engineering"], delete=[rids[0]])
    binding.wait_for_sync()
    assert got(search(request(fruit)))[0] == {rids[1]}
    assert rids[0] in got(search(request(path("t/product", "price", int=999))))[0]
    # a message that changes the resource's groups with skip_json: the JSON document answers with the new groups
    index(0, 999, "tool", True, "0d", ["admin"], skip=True)
    binding.wait_for_sync()
    p, v = got(search(request(path("t/product", "price", int=999), ["engineering"], op_or=True, field_filter=rids[2])))
    assert rids[0] not in p and rids[0] not in v and rids[2] in p and rids[2] in v
    assert rids[0] in got(search(request(path("t/product", "price", int=999), ["admin"], op_or=True, field_filter=rids[2])))[1]
    # a resource deletion removes its JSON document
    binding.index(P.IndexMessage(shard=shard, resource=rids[1], typemessage=1, kbid="kb").SerializeToString())
    binding.wait_for_sync()
    assert not search(request(fruit)).HasField("paragraph")
    binding.close()
