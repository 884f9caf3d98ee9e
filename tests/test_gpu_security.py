"""SearchRequest.security on the device: the PUBLIC / GROUP prefilter leaves against tests/security_model.py bit for bit, the keyword
passes on a masked view (nidx_txt_view) against the same calls on a copy of the segment whose alive bits are alive AND mask, two
views on two streams, and the whole path over gRPC through NidxBinding."""
import dataclasses
import random
import uuid

import numpy as np
import pytest

import security_model as M
import test_gpu_prefilter as G

pytestmark = pytest.mark.gpu


def _groups(rng, n):
    """n nested group ids (up to 4 levels), some spelled without the leading '/'."""
    out = set()
    while len(out) < n:
        path = "/".join(f"{rng.choice('abcg')}{rng.randint(0, 9)}" for _ in range(rng.randint(1, 4)))
        out.add(path)
    return [g if i % 3 else "/" + g for i, g in enumerate(sorted(out))]


def _secure_corpus(seed, n, n_groups=1000):
    docs, rids = G._corpus(seed, n)
    rng = random.Random(seed)
    groups = _groups(rng, n_groups)
    by_rid = {r: (() if rng.random() < 0.3 else tuple(rng.sample(groups, rng.randint(1, 5)))) for r in rids}
    return [dataclasses.replace(d, groups=by_rid[d.uuid]) for d in docs], rids, groups


def _requests(rng, groups):
    tops = sorted({g.lstrip("/").split("/")[0] for g in groups})
    return [[], [rng.choice(tops)], ["/" + rng.choice(tops)], [rng.choice(groups)], [rng.choice(groups) for _ in range(8)],
            ["/nothere", rng.choice(groups).lstrip("/")], [rng.choice(tops)[:1]]]


def _check_bits(ts, segments, alive, req, expr):
    """The device bits of ts.prefilter(expr, security=req) and, per segment, of the host path, against the model."""
    from nucliadb_b200 import _lib

    try:
        want = M.bits(segments, req, expr, alive)
    except ValueError:
        return
    total = sum(map(sum, want))
    res = ts.prefilter(expr, security=req)
    assert res.kind == ("none" if total == 0 else "all" if total == sum(map(sum, alive)) else "some"), (req, expr)
    if res.kind == "some":
        bits = res.device_bits[1].cpu().numpy().view(np.uint64)
        assert np.array_equal(bits, np.concatenate([G._words(w, s.n_docs) for s, w in zip(ts.segments, want)])), (req, expr)
    nodes, _keep, _ = ts._prefilter.compile(expr, ts.security_nodes(req))
    for s, w in zip(ts.segments, want):
        words, count = s._gpu.prefilter(nodes)
        assert np.array_equal(words, G._words(w, s.n_docs)) and count == sum(w), (req, expr)
    if expr is None:   # the security tree under NOT and, with a keyword leaf, under OR
        from nucliadb_b200.text import _node_array

        sec = ts.security_nodes(req)
        flat_not = [(_lib.NIDX_P_NOT, 1, 0, 0, None)] + sec
        kw = np.asarray([ts.vocab.get("alpha", 0xFFFFFFF0), ts.vocab.get("beta", 0xFFFFFFF0)], dtype=np.uint32)
        flat_or = [(_lib.NIDX_P_OR, 2, 0, 0, None)] + sec + [(_lib.NIDX_P_KEYWORD, 2, 0, 0, kw.ctypes.data)]
        for flat, rule in ((flat_not, lambda d: not M.granted(d.groups, req)), (flat_or, lambda d: M.granted(d.groups, req) or _alpha_beta(d))):
            nodes = _node_array(flat)
            for s, docs, al in zip(ts.segments, segments, alive):
                words, count = s._gpu.prefilter(nodes)
                w = [a and rule(d) for d, a in zip(docs, al)]
                assert np.array_equal(words, G._words(w, s.n_docs)) and count == sum(w), req


def _alpha_beta(doc):
    import prefilter_model

    return prefilter_model._phrase_in(doc.text, ["alpha", "beta"])


@pytest.mark.parametrize("n", [1, 4097, 200_003])
def test_security_prefilter_matches_the_model(n):
    docs, rids, groups = _secure_corpus(n, n)
    rng = random.Random(n + 1)
    segments = G._split(docs, 2 if n > 1 else 1)
    ts, alive = G._searcher(segments, "random", n)
    ts._ensure_positions()
    exprs = [None] + [G._expr(rng, rids, rng.randint(1, 5)) for _ in range(3 if n > 100_000 else 12)]
    for req in _requests(rng, groups):
        for expr in exprs:
            _check_bits(ts, segments, alive, req, expr)


def _variants(seg, facets, qsets):
    """Every keyword pass of one handle -> a list of numpy outputs (scores as uint32 views, only the filled entries)."""
    from nucliadb_b200 import _lib

    out = []
    for qt, qo, phrases in qsets:
        for mode in (_lib.NIDX_BM25_OR, _lib.NIDX_BM25_AND):
            runs = [seg.search(qt, qo, 50, mode=mode), seg.search_faceted(qt, qo, 50, facets, mode=mode, use_tf=False),
                    seg.search_ordered(qt, qo, 50, _lib.NIDX_ORDER_MODIFIED, _lib.NIDX_ORDER_ASC, mode),
                    seg.search_ordered(qt, qo, 50, _lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_DESC, mode, facets=facets)]
            if phrases:
                runs += [seg.search_phrases(qt, qo, phrases, 50, mode=mode), seg.search_phrases(qt, qo, phrases, 50, mode=mode, facets=facets),
                         seg.search_phrases(qt, qo, phrases, 50, mode=mode, order=(_lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_ASC))]
            for r in runs:
                counts = np.asarray(r[2])
                out.append([np.asarray(r[0])[i, : counts[i]] for i in range(len(counts))])
                out.append([np.asarray(r[1])[i, : counts[i]].view(np.uint32 if r[1].dtype == np.float32 else np.uint64) for i in range(len(counts))])
                out += [counts, np.asarray(r[3])] + ([np.asarray(r[4])] if len(r) > 4 else [])
    docs, dates, count, total = seg.list_ordered(300, _lib.NIDX_ORDER_MODIFIED, _lib.NIDX_ORDER_DESC)
    out += [docs[:count], dates[:count], count, total, seg.facet_count_all(facets)]
    return out


def _same(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        if isinstance(x, list):
            _same(x, y)
        else:
            assert np.array_equal(np.asarray(x), np.asarray(y))


def test_masked_keyword_passes_equal_a_copy_with_alive_and_mask():
    """Each keyword pass on a view equals, id for id, score bit for bit and count for count, the same call on a second copy of the
    index whose alive bits were set to alive AND mask with nidx_txt_set_alive (same statistics on both)."""
    import torch

    from nucliadb_b200.text import TextSearcher, _node_array, facet_key

    docs, rids, groups = _secure_corpus(11, 150_001, 200)
    segments = G._split(docs, 2)
    ts, alive = G._searcher(segments, "random", 11)
    copy = TextSearcher.open(segments)
    for t in (ts, copy):
        t._ensure_facets(); t._ensure_dates(); t._ensure_positions()
    facets = [facet_key(f) for f in ("/l", "/k/x")]
    v = ts.vocab
    qsets = [(np.asarray([v["alpha"], v["beta"]], np.uint32), np.asarray([0, 2], np.uint32), []),
             (np.asarray([v["gamma"], v["delta"], v["eps"], 0xFFFFFFF0], np.uint32), np.asarray([0, 1, 4], np.uint32), [(0, [v["alpha"], v["beta"]]), (1, [v["beta"], v["alpha"]])])]
    rng = np.random.default_rng(3)
    for req in (["/" + groups[0].lstrip("/").split("/")[0]], [], None):
        for s, c, al in zip(ts.segments, copy.segments, alive):
            words = (s.n_docs + 63) // 64
            if req is not None:   # the device path: the prefilter's bits, never on the host until the check below
                mask = torch.empty(words, dtype=torch.int64, device="cuda")
                s._gpu.prefilter(_node_array(ts.security_nodes(req)), out=mask)
                view = s._gpu.view(mask)
                keep = mask.cpu().numpy().view(np.uint64)
            else:                 # the host path: a random mask that ignores alive, with its padding bits set
                keep = rng.integers(0, 2**63, size=words, dtype=np.int64).view(np.uint64) | np.uint64(1 << 63)
                view = s._gpu.view(keep)
                keep = keep & G._words(al, s.n_docs)
            c._gpu.set_alive(keep)
            try:
                _same(_variants(view, facets, qsets), _variants(c._gpu, facets, qsets))
            finally:
                view.close()
    # a view refuses the setters and leaves its parent as it was
    from nucliadb_b200._lib import NidxError

    s = ts.segments[0]
    view = s._gpu.view(np.zeros((s.n_docs + 63) // 64, np.uint64))
    for call in (lambda: view.set_alive(None), lambda: view.set_facets([], np.zeros(s.n_docs + 1), np.zeros(0)),
                 lambda: view.set_doc_groups([], np.zeros(s.n_docs + 1), np.zeros(0)), lambda: view.set_stats(1, 1)):
        with pytest.raises(NidxError):
            call()
    assert view.list_ordered(10)[3] == 0 and s._gpu.list_ordered(10)[3] == sum(alive[0])
    view.close()


def test_two_masks_on_two_streams():
    import torch

    from nucliadb_b200 import _lib
    from nucliadb_b200.text import TextSearcher

    docs, rids, groups = _secure_corpus(21, 60_000, 100)
    ts = TextSearcher.open([docs])
    seg = ts.segments[0]._gpu
    words = (seg.n_docs + 63) // 64
    rng = np.random.default_rng(21)
    masks = [torch.from_numpy(rng.integers(-2**63, 2**63 - 1, size=words, dtype=np.int64)).cuda() for _ in range(2)]
    v = ts.vocab
    qt = torch.tensor([v["alpha"], v["beta"], v["gamma"]], dtype=torch.int32, device="cuda")
    qo = torch.tensor([0, 3], dtype=torch.int32, device="cuda")
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    views, outs = [], []
    for m, st in zip(masks, streams):
        st.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(st):
            views.append(seg.view(m))
            outs.append(views[-1].search(qt, qo, 100, mode=_lib.NIDX_BM25_OR))
    torch.cuda.synchronize()
    got = [[t.cpu().numpy() for t in o] for o in outs]
    for i, m in enumerate(masks):   # each against its own mask alone, on the host path
        want = seg.view(m.cpu().numpy().view(np.uint64))
        d, s, c, tot = want.search(qt.cpu().numpy().view(np.uint32), qo.cpu().numpy().view(np.uint32), 100, mode=_lib.NIDX_BM25_OR)
        assert np.array_equal(got[i][0].view(np.uint32)[0, : c[0]], d[0, : c[0]]) and np.array_equal(got[i][1].view(np.uint32)[0, : c[0]], s.view(np.uint32)[0, : c[0]])
        assert got[i][2][0] == c[0] and got[i][3].view(np.uint64)[0] == tot[0]
        want.close()
    assert got[0][3][0] != got[1][3][0] or not np.array_equal(got[0][0], got[1][0])
    for vw in views:
        vw.close()


def test_binding_honours_security_end_to_end(tmp_path):
    import grpc

    from nidx_binding import NidxBinding
    from nucliadb_b200 import nidx_protos as P
    from nucliadb_b200.vector import VectorConfig

    dim = 8
    binding = NidxBinding({"INDEXER__OBJECT_STORE": "file", "INDEXER__FILE_PATH": str(tmp_path)})
    shard = binding.new_shard("kb", {"en": VectorConfig(dimension=dim)})
    rng = np.random.default_rng(4)
    rids = [uuid.UUID(int=i + 101).hex for i in range(6)]
    groups = [(), ("g1",), ("/g1/sub",), ("/g2",), ("g10",), None]   # None: no security message at all
    (tmp_path / "index").mkdir()

    def index(i, grp, seq_key):
        res = P.Resource()
        res.resource.uuid, res.shard_id = rids[i], shard
        res.metadata.created.seconds = res.metadata.modified.seconds = 1000 + i
        res.labels.append(f"/l/r{i % 2}")
        if grp is not None:
            res.security.SetInParent()
            res.security.access_groups.extend(grp)
        for fid, text in (("a/title", f"fox number {i}"), ("a/summary", "the quick fox and the dog")):
            res.texts[fid].text = text
            pid = f"{rids[i]}/{fid}/0-{len(text)}"
            par = res.paragraphs[fid].paragraphs[pid]
            par.start, par.end = 0, len(text)
            par.sentences[pid].vector.extend(rng.standard_normal(dim).astype(np.float32).tolist())
        (tmp_path / f"index/{seq_key}").write_bytes(res.SerializeToString())
        binding.index(P.IndexMessage(shard=shard, resource=rids[i], typemessage=0, storage_key=f"index/{seq_key}", kbid="kb").SerializeToString())

    for i, g in enumerate(groups):
        index(i, g, f"{i}")
    binding.wait_for_sync()
    chan = grpc.insecure_channel(f"127.0.0.1:{binding.searcher_port}")
    search = chan.unary_unary(P.SEARCH_METHOD, request_serializer=lambda m: m.SerializeToString(), response_deserializer=P.SearchResponse.FromString)

    def request(sec, order=False):
        req = P.SearchRequest(shard_ids=[shard], body="fox", vector=[0.1] * dim, vectorset="en", result_per_page=50, min_score_semantic=-1e9,
                              with_duplicates=True, document=True, paragraph=True)
        req.faceted.labels.append("/l")
        if order:
            req.order.sort_by, req.order.type = 0, 1
        if sec is not None:
            req.security.SetInParent()
            req.security.access_groups.extend(sec)
        return req

    def check(sec, want):
        want_ids = {rids[i] for i in want}
        for order in (False, True):
            resp = search(request(sec, order))
            got = {"document": {r.uuid for r in resp.document.results}, "paragraph": {r.uuid for r in resp.paragraph.results},
                   "vector": {d.doc_id.id.split("/")[0] for d in resp.vector.documents}}
            assert got == {"document": want_ids, "paragraph": want_ids, "vector": want_ids}, (sec, order, got)
            assert resp.document.total == resp.paragraph.total == 2 * len(want)
            n_r0 = sum(1 for i in want if i % 2 == 0)
            want_facets = sorted([(f"/l/r{j}", 2 * n) for j, n in ((0, n_r0), (1, len(want) - n_r0)) if n], key=lambda t: (-t[1], t[0]))
            for target in (resp.document, resp.paragraph):
                assert [(f.tag, f.total) for f in target.facets["/l"].facetresults] == want_facets

    check(["g1"], [0, 1, 2, 5])                  # /g1 grants /g1/sub, not /g10
    check(["/g1/sub"], [0, 2, 5])
    check([], [0, 5])                            # public resources only
    check(["/g2", "g10"], [0, 3, 4, 5])
    check(["g1/sub", "nothere"], [0, 2, 5])
    # every group granted: the same bytes as no security at all (security filters, it never scores)
    for order in (False, True):
        assert search(request(["g1", "g2", "g10"], order)).SerializeToString() == search(request(None, order)).SerializeToString()
    # a field_filter intersects with security for the vector search
    req = request(["g1"])
    req.field_filter.facet.facet = "/l/r1"
    assert {d.doc_id.id.split("/")[0] for d in search(req).vector.documents} == {rids[1], rids[5]}
    # a deletion, and a re-index that moves a resource to another group
    binding.index(P.IndexMessage(shard=shard, resource=rids[1], typemessage=1, kbid="kb").SerializeToString())
    index(3, ("g1",), "3b")
    binding.wait_for_sync()
    check(["g1"], [0, 2, 3, 5])
    check(["/g2"], [0, 5])
    binding.close()
