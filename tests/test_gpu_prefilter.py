"""The prefilter on the device (TextSearcher.prefilter -> nidx_txt_prefilter, VectorSearcher.search -> nidx_vec_prefilter_bits)
against the per-document model of tests/prefilter_model.py, bit for bit, and the hand-off to the vector search against the same search
given the model's fields as PrefilterResult.some."""
import random
import uuid

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

I64_MIN, I64_MAX = -(1 << 63), (1 << 63) - 1
WORDS = ["alpha", "beta", "gamma", "delta", "eps", "zeta"]
LONG = "q" * 44
LABELS = ["/l/a", "/l/a/b", "/l/c", "/k/x", "/k/x/y/z", "/e", "bare"]
FIELDS = ["/a/title", "/a/summary", "/a/titles", "/f/file1", "/t/x/y", "/u"]
DATES = [None, -5, -1, 0, 1, 5, 100, I64_MIN + 1, I64_MAX]


def _rids(rng, n):
    out = []
    for i in range(n):
        u = uuid.UUID(int=rng.getrandbits(128))
        out.append(str(u) if i % 7 == 3 else u.hex)   # some resources spell their UUID with hyphens
    return out


def _corpus(seed, n):
    from nucliadb_b200.text import TextDoc

    rng = random.Random(seed)
    rids = _rids(rng, max(n // 3, 1))
    docs = []
    for _ in range(n):
        words = [rng.choice(WORDS[:2]) if rng.random() < 0.5 else rng.choice(WORDS) for _ in range(rng.randint(1, 8))]
        if rng.random() < 0.1:
            words.insert(rng.randint(0, len(words)), LONG)
        docs.append(TextDoc(rng.choice(rids), rng.choice(FIELDS), " ".join(words), tuple(rng.sample(LABELS, rng.randint(0, 3))),
                            rng.choice(DATES), rng.choice(DATES)))
    return docs, rids


def _split(docs, n_segments):
    cuts = [len(docs) * i // n_segments for i in range(n_segments + 1)]
    return [docs[a:b] for a, b in zip(cuts, cuts[1:])]


def _leaf(rng, rids):
    from nucliadb_b200 import nidx_protos as P

    e = P.FilterExpression()
    kind = rng.choice(["facet", "field", "resource", "rfp", "date", "keyword"])
    if kind == "facet":
        e.facet.facet = rng.choice(["/l/a", "/l/a/b", "/l", "/k/x/y", "/k", "/e", "/", "/nope", "/l/a/"])
    elif kind == "field":
        e.field.field_type = rng.choice(["a", "f", "t", "u", "zz", ""])
        if rng.random() < 0.6:
            e.field.field_id = rng.choice(["title", "summary", "file1", "x", "x/y", "titl"])
    elif kind == "resource":
        e.resource.resource_id = rng.choice(rids + ["other"])
    elif kind == "rfp":
        r = rng.choice(rids)
        e.resource_field_prefix.resource_id = str(uuid.UUID(r)) if rng.random() < 0.5 else uuid.UUID(r).hex
        e.resource_field_prefix.field_type = rng.choice(["a", "t", "f"])
        e.resource_field_prefix.field_id_prefix = rng.choice(["", "ti", "title", "x/", "file"])
    elif kind == "date":
        e.date.field = rng.randint(0, 1)
        for bound in ("since", "until"):
            if rng.random() < 0.6:
                getattr(e.date, bound).seconds = rng.choice([d for d in DATES if d is not None] + [I64_MIN, -2, 2])
                getattr(e.date, bound).nanos = rng.randint(0, 999_999_999)
    else:
        e.keyword.keyword = rng.choice(["alpha", "BETA", "alpha beta", "beta alpha gamma", f"alpha {LONG} beta", "nothere", "alpha nothere", "", "!!",
                                        "gamma delta eps"])
    return e


def _expr(rng, rids, depth):
    from nucliadb_b200 import nidx_protos as P

    if depth <= 1 or rng.random() < 0.3:
        return _leaf(rng, rids)
    e = P.FilterExpression()
    kind = rng.choice(["and", "or", "not"])
    if kind == "not":
        e.bool_not.CopyFrom(_expr(rng, rids, depth - 1))
    else:
        ops = getattr(e, "bool_and" if kind == "and" else "bool_or").operands
        for _ in range(rng.choice([0, 1, 2, 2, 3, 4])):
            ops.add().CopyFrom(_expr(rng, rids, depth - 1))
    return e


def _chain(rng, rids, depth):
    """An expression exactly `depth` levels deep (NOT / AND / OR wrapped around a leaf)."""
    from nucliadb_b200 import nidx_protos as P

    def plain():   # a leaf one level deep (a resource_field_prefix runs as three)
        while True:
            e = _leaf(rng, rids)
            if e.WhichOneof("expr") != "resource_field_prefix":
                return e

    e = plain()
    for level in range(depth - 1):
        w = P.FilterExpression()
        if level % 3 == 0:
            w.bool_not.CopyFrom(e)
        else:
            ops = (w.bool_and if level % 3 == 1 else w.bool_or).operands
            ops.add().CopyFrom(e)
            ops.add().CopyFrom(plain())
        e = w
    return e


def _words(mask, n_docs):
    out = np.zeros((n_docs + 63) // 64 * 8, dtype=np.uint8)
    packed = np.packbits(np.asarray(mask, dtype=bool), bitorder="little")
    out[: len(packed)] = packed
    return out.view(np.uint64)


def _searcher(segments, alive_kind, seed):
    from nucliadb_b200.text import TextSearcher

    ts = TextSearcher.open(segments)
    rng = np.random.default_rng(seed)
    alive = []
    for s in ts.segments:
        if alive_kind == "all":
            alive.append([True] * s.n_docs)
            continue
        a = np.zeros(s.n_docs, dtype=bool) if alive_kind == "none" else rng.random(s.n_docs) < 0.7
        words = _words(a, s.n_docs)
        if s.n_docs % 64:
            words[-1] |= np.uint64(~((1 << (s.n_docs % 64)) - 1) & 0xFFFFFFFFFFFFFFFF)   # padding bits set: they must not count
        s._gpu.set_alive(words)
        s.alive_count = int(a.sum())
        alive.append(a.tolist())
    return ts, alive


def _check(ts, segments, alive, expr):
    import prefilter_model as M

    try:
        want_bits, want_class = M.prefilter(expr, segments, alive)
    except ValueError:
        with pytest.raises(ValueError):
            ts.prefilter(expr)
        return None
    res = ts.prefilter(expr)
    assert res.kind == want_class, expr
    nodes, _keep, _ = ts._prefilter.compile(expr)
    for s, mb in zip(ts.segments, want_bits):   # the host path, segment by segment: the words and the count
        words, count = s._gpu.prefilter(nodes)
        assert np.array_equal(words, _words(mb, s.n_docs)), expr
        assert count == sum(mb)
    if res.kind == "some":   # the device path: one index-wide bitset, each segment from a whole word
        bits = res.device_bits[1].cpu().numpy().view(np.uint64)
        want = np.concatenate([_words(mb, s.n_docs) for s, mb in zip(ts.segments, want_bits)] or [np.zeros(0, np.uint64)])
        assert np.array_equal(bits, want), expr
        assert res.device_bits[2] == sum(map(sum, want_bits))
        fields = [(f.resource_id, f.field_id) for f in res.fields]
        assert fields == [(uuid.UUID(d.uuid), d.field) for docs, mb in zip(segments, want_bits) for d, m in zip(docs, mb) if m]
    return res


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 4097, 262145])
def test_bits_match_the_model(n):
    docs, rids = _corpus(n, n)
    rng = random.Random(n)
    n_exprs = 4 if n > 100_000 else 40
    for n_segments in ((1, 3) if n <= 4097 else (2,)):
        segments = _split(docs, n_segments)
        for alive_kind in (("all", "none", "random") if n <= 4097 else ("random",)):
            ts, alive = _searcher(segments, alive_kind, n + n_segments)
            for _ in range(n_exprs if alive_kind == "random" else max(n_exprs // 4, 2)):
                _check(ts, segments, alive, _expr(rng, rids, rng.randint(1, 6)))
            if n > 100_000:   # phrase leaves whose virtual lists have skip rows (their drivers have >= 256 postings)
                from nucliadb_b200 import nidx_protos as P

                for k in ("alpha beta", "beta alpha alpha", "alpha gamma"):
                    e = P.FilterExpression()
                    e.keyword.keyword = k
                    _check(ts, segments, alive, e)


def test_every_leaf_kind_and_the_depth_limit():
    from nucliadb_b200 import _lib
    from nucliadb_b200 import nidx_protos as P

    import prefilter_model as M

    docs, rids = _corpus(7, 700)
    segments = _split(docs, 3)
    ts, alive = _searcher(segments, "random", 7)
    rng = random.Random(7)
    for _ in range(150):
        _check(ts, segments, alive, _leaf(rng, rids))
    for d in (1, 2, 17, 63, _lib.NIDX_PREFILTER_MAX_DEPTH):
        e = _chain(rng, rids, d)
        assert M.depth(e) == d
        _check(ts, segments, alive, e)
    for _ in range(30):   # seeded random trees up to the limit
        e = _expr(rng, rids, rng.randint(1, 12))
        if M.depth(e) <= _lib.NIDX_PREFILTER_MAX_DEPTH:
            _check(ts, segments, alive, e)
    with pytest.raises(ValueError):   # one level past the limit
        ts.prefilter(_chain(rng, rids, _lib.NIDX_PREFILTER_MAX_DEPTH + 1))
    bad = P.FilterExpression()
    bad.resource_field_prefix.resource_id = "not-a-uuid"
    with pytest.raises(ValueError):
        ts.prefilter(bad)


def _vector_index(docs, dim, seed):
    from nucliadb_b200 import vector as V

    rng = np.random.default_rng(seed)
    elems = []
    for i, d in enumerate(docs):
        if i % 5 == 4:
            continue   # a field without paragraphs
        for j in range(1 + i % 3):
            v = rng.standard_normal(dim).astype(np.float32)
            elems.append(V.Elem(f"{d.uuid}/{d.field[1:]}/{j}", [v], labels=[rng.choice(["/p/a", "/p/b"])]))
    cfg = V.VectorConfig(dimension=dim, similarity=V.Similarity.Dot)
    half = len(elems) // 2
    segs = [(V.VectorIndexer.index_elems(elems[:half], cfg), 1), (V.VectorIndexer.index_elems(elems[half:], cfg), 2)]
    return V.VectorSearcher.open(cfg, segs), rng


def test_hand_off_equals_the_search_given_the_model_fields():
    from nucliadb_b200 import _lib
    from nucliadb_b200 import vector as V

    import prefilter_model as M

    docs, rids = _corpus(3, 4097)
    segments = _split(docs, 2)
    ts, alive = _searcher(segments, "all", 3)
    vs, vrng = _vector_index(docs, 16, 3)
    rng = random.Random(3)
    checked = 0
    while checked < 12:
        expr = _expr(rng, rids, rng.randint(1, 4))
        try:
            bits, cls = M.prefilter(expr, segments, alive)
        except ValueError:
            continue
        if cls != "some":
            continue
        res = ts.prefilter(expr)
        fields = [V.FieldId(uuid.UUID(d.uuid), d.field) for docs_, mb in zip(segments, bits) for d, m in zip(docs_, mb) if m]
        for op in (V.FilterOperator.And, V.FilterOperator.Or):
            for formula in (None, V.Literal("/p/a"), V.Not(V.Literal("/p/b"))):
                for method in (_lib.NIDX_METHOD_BRUTE, _lib.NIDX_METHOD_HNSW):
                    req = V.VectorSearchRequest(vector=vrng.standard_normal(16).astype(np.float32).tolist(), result_per_page=20, min_score=-1e9,
                                                filtering_formula=formula, filter_operator=op)
                    got = vs.search(req, res, method=method, ef=64).documents
                    want = vs.search(req, V.PrefilterResult.some(fields), method=method, ef=64).documents
                    assert [(d.doc_id, d.score) for d in got] == [(d.doc_id, d.score) for d in want], (expr, op, formula, method)
        checked += 1


def test_binding_date_keyword_and_field_prefix_filters(tmp_path):
    from nidx_binding import NidxBinding
    from nucliadb_b200 import nidx_protos as P
    from nucliadb_b200.vector import VectorConfig

    dim = 8
    binding = NidxBinding({"INDEXER__OBJECT_STORE": "file", "INDEXER__FILE_PATH": str(tmp_path)})
    shard = binding.new_shard("kb", {"en": VectorConfig(dimension=dim)})
    rng = np.random.default_rng(9)
    rids = [uuid.UUID(int=i + 11).hex for i in range(4)]
    texts = [{"a/title": "the quick brown fox", "a/summary": "a lazy dog"}, {"a/title": "graph search on hbm", "f/file1": "quick fox notes"},
             {"a/title": "nothing in common"}, {"t/text": "brown fox quick"}]
    (tmp_path / "index").mkdir()
    keys = {}
    for i, rid in enumerate(rids):
        res = P.Resource()
        res.resource.uuid, res.shard_id = rid, shard
        res.metadata.created.seconds, res.metadata.modified.seconds = 1000 + 100 * i, 5000 - 100 * i
        for fid, text in texts[i].items():
            res.texts[fid].text = text
            pid = f"{rid}/{fid}/0-{len(text)}"
            par = res.paragraphs[fid].paragraphs[pid]
            par.start, par.end = 0, len(text)
            par.sentences[pid].vector.extend(rng.standard_normal(dim).astype(np.float32).tolist())
            keys.setdefault((rid, fid), []).append(pid)
        (tmp_path / f"index/{rid}").write_bytes(res.SerializeToString())
        binding.index(P.IndexMessage(shard=shard, resource=rid, typemessage=0, storage_key=f"index/{rid}", kbid="kb").SerializeToString())
    binding.wait_for_sync()

    def ids(expr):
        req = P.SearchRequest(shard_ids=[shard], vector=[0.1] * dim, vectorset="en", result_per_page=50, min_score_semantic=-1e9, with_duplicates=True)
        req.field_filter.CopyFrom(expr)
        return sorted(d.doc_id.id for d in binding.search(req).vector.documents)

    def want(pairs):
        return sorted(p for pair in pairs for p in keys[pair])

    e = P.FilterExpression()
    e.date.field, e.date.since.seconds, e.date.until.seconds = 0, 1100, 1200   # created 1100 and 1200
    assert ids(e) == want([(rids[1], "a/title"), (rids[1], "f/file1"), (rids[2], "a/title")])
    e = P.FilterExpression()
    e.keyword.keyword = "quick fox"                                             # a phrase
    assert ids(e) == want([(rids[1], "f/file1")])
    e.keyword.keyword = "fox"
    assert ids(e) == want([(rids[0], "a/title"), (rids[1], "f/file1"), (rids[3], "t/text")])
    e = P.FilterExpression()
    e.resource_field_prefix.resource_id, e.resource_field_prefix.field_type, e.resource_field_prefix.field_id_prefix = str(uuid.UUID(rids[0])), "a", "ti"
    assert ids(e) == want([(rids[0], "a/title")])
    e = P.FilterExpression()
    e.bool_not.date.field, e.bool_not.date.until.seconds = 1, 4800             # modified > 4800: resources 0 and 1
    assert ids(e) == want([(rids[0], "a/title"), (rids[0], "a/summary"), (rids[1], "a/title"), (rids[1], "f/file1")])
    e = P.FilterExpression()
    e.keyword.keyword = "absent"
    assert ids(e) == []
    binding.close()
