"""Order by date (TopDocs::order_by_fast_field) on a machine without a GPU: the oracle (tests/order_oracle.py) against a literal
sorted() transcription and the golden fixture, the cross-shard merge rule, and the mirror's order flow (text.py, binding.py) over the
emulated C ABI (tests/order_emulator.py), restating the reference's order tests."""
import os
import uuid

import numpy as np
import pytest

import order_emulator
import order_oracle as OO
from nucliadb_b200 import _lib
from nucliadb_b200 import text as T
from nucliadb_b200.binding import merge_order_key

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "order_small.npz")


def _secs(rng, n, n_distinct=20, p_none=0.1):
    s = (1_500_000_000 + rng.integers(0, n_distinct, n) * 86_400).astype(np.int64)
    s[rng.random(n) < p_none] = OO.NONE
    return s


@pytest.mark.parametrize("order_type", [OO.DESC, OO.ASC])
def test_oracle_equals_the_literal_rule(order_type):
    rng = np.random.default_rng(1)
    for trial in range(20):
        n = int(rng.integers(1, 300))
        secs = _secs(rng, n, n_distinct=int(rng.integers(1, 10)))
        if trial % 4 == 0:
            secs[rng.integers(0, n, 3)] = [(1 << 63) - 1, -(1 << 63) + 1, 0]
        mask = rng.random(n) < 0.6
        for k in (1, 5, n + 3):
            d, s = OO.order_topk(mask, secs, k, order_type)
            want = OO.literal_order(np.nonzero(mask)[0], secs, order_type)[:k]
            assert d.tolist() == want and s.tolist() == [int(secs[x]) for x in want]


def test_golden_fixture_matches_the_oracle():
    g = np.load(GOLDEN, allow_pickle=False)
    qo, k = g["query_off"], int(g["k"])
    queries = [g["query_terms"][qo[i]:qo[i + 1]].tolist() for i in range(len(qo) - 1)]
    n_docs = len(g["created"])
    assert (g["created"] == OO.NONE).any() and (g["modified"] == OO.NONE).any()
    assert len(np.unique(g["created"])) < n_docs // 10   # heavy ties
    for q, conj, field, typ, docs, total in zip(g["exp_q"], g["exp_conj"], g["exp_field"], g["exp_type"], g["exp_docs"], g["exp_total"]):
        secs = (g["created"], g["modified"])[field]
        d, s, tot = OO.search(n_docs, g["term_off"], g["post_doc"], queries[q], bool(conj), g["alive"], secs, k, int(typ))
        assert d.tolist() == [x for x in docs.tolist() if x >= 0] and tot == total
        assert s.tolist() == [int(secs[x]) for x in d]


def test_merge_order_key_rule():
    """Date in the requested direction, undated last, then the shard's position in the request, then the rank inside the shard."""
    rows = [(100, 1, 0), (None, 0, 0), (100, 0, 1), (50, 1, 1), (200, 0, 0), (100, 0, 2)]
    desc = sorted(rows, key=lambda r: merge_order_key(r[0], _lib.NIDX_ORDER_DESC, r[1], r[2]))
    assert desc == [(200, 0, 0), (100, 0, 1), (100, 0, 2), (100, 1, 0), (50, 1, 1), (None, 0, 0)]
    asc = sorted(rows, key=lambda r: merge_order_key(r[0], _lib.NIDX_ORDER_ASC, r[1], r[2]))
    assert asc == [(50, 1, 1), (100, 0, 1), (100, 0, 2), (100, 1, 0), (200, 0, 0), (None, 0, 0)]


@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.setattr(_lib, "_lib", order_emulator.OrderEmulatedLib())


def test_int_order_pagination(emulated):
    """nidx_text/tests/test_search.rs::test_int_order_pagination: an empty body, one result per page, ordered by created DESC:
    one result and a next page."""
    docs = [T.TextDoc("r1", "/t/title", "the first document", created=1_700_000_000, modified=1_700_000_100),
            T.TextDoc("r2", "/t/title", "the second document", created=1_700_000_050, modified=1_700_000_060)]
    s = T.TextSearcher.open([docs])
    resp = s.search(T.DocumentSearchRequest(body="", result_per_page=1, min_score=-3.4e38, order=T.OrderBy(_lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_DESC)))
    assert len(resp.results) == 1 and resp.next_page and resp.total == 2
    assert resp.results[0].uuid == "r2" and resp.results[0].date == 1_700_000_050 and resp.results[0].score is None


def test_paragraph_order_by(emulated):
    """nidx_paragraph/tests/reader.rs::test_order_by: "this is the" ordered by created matches 3 paragraphs."""
    texts = ["this is the title", "a first paragraph", "the second one", "and the third", "another field body text"]
    docs = [T.TextDoc("r", "/t/mytext", t, created=1_700_000_000, modified=1_700_000_000) for t in texts]
    s = T.ParagraphSearcher.open([docs])
    resp = s.search(T.DocumentSearchRequest(body="this is the", result_per_page=20, order=T.OrderBy(_lib.NIDX_ORDER_CREATED, _lib.NIDX_ORDER_DESC)))
    assert resp.total == 3 and len(resp.results) == 3 and not resp.next_page
    assert [r.field for r in resp.results] == ["/t/mytext"] * 3 and all(r.date == 1_700_000_000 for r in resp.results)


@pytest.mark.parametrize("cls", [T.TextSearcher, T.ParagraphSearcher])
def test_mirror_order_over_segments_equals_the_literal_rule(emulated, cls):
    rng = np.random.default_rng(3)
    words = [f"w{i}" for i in range(20)]
    n = 150
    created, modified = _secs(rng, n, 12), _secs(rng, n, 5)
    docs = [T.TextDoc(f"u{i:03d}", "/a/f", " ".join(rng.choice(words, size=6)), (f"/l/{i % 4}",),
                      None if created[i] == OO.NONE else int(created[i]), None if modified[i] == OO.NONE else int(modified[i])) for i in range(n)]
    segs = [docs[:60], docs[60:100], docs[100:]]
    ords = [(0, i) for i in range(60)] + [(1, i) for i in range(40)] + [(2, i) for i in range(50)]
    s = cls.open(segs)
    for body in ("w1 w2", "w3", ""):
        toks = T.tokenize(body)
        hit = [set(T.tokenize(d.text)) for d in docs]
        matched = [i for i in range(n) if not toks or (all if cls.conjunction else any)(t in hit[i] for t in toks)]
        for field, secs in ((_lib.NIDX_ORDER_CREATED, created), (_lib.NIDX_ORDER_MODIFIED, modified)):
            for typ in (_lib.NIDX_ORDER_DESC, _lib.NIDX_ORDER_ASC):
                for k in (1, 7, 200):
                    resp = s.search(T.DocumentSearchRequest(body=body, result_per_page=k, order=T.OrderBy(field, typ), min_score=99.0))
                    want = sorted(matched, key=lambda i: (T.date_sort_key(None if secs[i] == OO.NONE else int(secs[i]), typ), ords[i]))[:k]
                    assert [r.uuid for r in resp.results] == [docs[i].uuid for i in want], (body, field, typ, k)
                    assert [r.date for r in resp.results] == [None if secs[i] == OO.NONE else int(secs[i]) for i in want]
                    assert resp.total == len(matched) and resp.next_page == (len(matched) > k)
        # ordered + faceted: the facets of the unordered request, the results of the ordered one
        o = T.OrderBy(_lib.NIDX_ORDER_MODIFIED, _lib.NIDX_ORDER_ASC)
        both = s.search(T.DocumentSearchRequest(body=body, result_per_page=5, faceted=["/l"], order=o))
        assert both.facets == s.search(T.DocumentSearchRequest(body=body, result_per_page=5, faceted=["/l"])).facets
        plain = s.search(T.DocumentSearchRequest(body=body, result_per_page=5, order=o))
        assert (both.results, both.total, both.next_page) == (plain.results, plain.total, plain.next_page)


def test_requests_without_order_are_unchanged(emulated):
    docs = [T.TextDoc(f"u{i}", "/a/f", f"common w{i % 3}", created=1_000 + i) for i in range(30)]
    s = T.TextSearcher.open([docs[:10], docs[10:]])
    resp = s.search(T.DocumentSearchRequest(body="common", result_per_page=5))
    assert all(r.score is not None and r.date is None for r in resp.results) and len(resp.results) == 5
    assert s.search(T.DocumentSearchRequest(body="", result_per_page=5)).results == []   # AllQuery without an order: as before


def _index(binding, tmp_path, shard, i, when, text, with_meta=True):
    from nucliadb_b200 import nidx_protos as P

    rid = uuid.UUID(int=i + 1).hex
    res = P.Resource()
    res.resource.uuid, res.resource.shard_id, res.shard_id = rid, shard, shard
    if with_meta:
        res.metadata.created.seconds = when
        res.metadata.modified.seconds = when
    res.labels.append(f"/dummy{i:03d}")
    res.texts[f"dummy-{i:03d}"].text = text
    (tmp_path / f"index/{rid}").write_bytes(res.SerializeToString())
    binding.index(P.IndexMessage(shard=shard, resource=rid, typemessage=0, storage_key=f"index/{rid}", kbid="kb").SerializeToString())


def test_search_sorting_on_the_binding(emulated, tmp_path):
    """nidx/tests/integration/search_sorting.rs: 20 resources one second apart, a page of 5, ASC / DESC x CREATED / MODIFIED; here
    spread over two shards, plus a resource without metadata (indexed, no date: last in both directions)."""
    from nidx_binding import NidxBinding
    from nucliadb_b200 import nidx_protos as P

    binding = NidxBinding({"INDEXER__OBJECT_STORE": "file", "INDEXER__FILE_PATH": str(tmp_path)})
    shards = [binding.new_shard("kb", {}) for _ in range(2)]
    (tmp_path / "index").mkdir()
    now = 1_760_000_000
    for i in range(20):
        _index(binding, tmp_path, shards[i % 2], i, now - (20 - i), f"Dummy text {i:03d}")
    _index(binding, tmp_path, shards[0], 20, 0, "Dummy text undated", with_meta=False)
    binding.wait_for_sync()
    fields = [f"/dummy-{i:03d}" for i in range(20)]
    for sort_by in (P.OrderBy.CREATED, P.OrderBy.MODIFIED):
        for typ in (P.OrderBy.ASC, P.OrderBy.DESC):
            req = P.SearchRequest(shard_ids=shards, document=True, paragraph=True, result_per_page=5)
            req.order.sort_by, req.order.type = sort_by, typ
            resp = binding.search(req)
            want = fields[:5] if typ == P.OrderBy.ASC else fields[::-1][:5]
            assert [r.field for r in resp.document.results] == want
            assert [r.date.seconds for r in resp.document.results] == [now - 20 + int(f[-3:]) for f in want]
            assert all(r.date.nanos == 0 and r.WhichOneof("sort_value") == "date" for r in resp.document.results)
            assert resp.document.total == 21 and resp.document.next_page
            req.result_per_page = 25
            every = binding.search(req).document.results
            assert len(every) == 21 and every[-1].field == "/dummy-020" and every[-1].WhichOneof("sort_value") is None
    plain = P.SearchRequest(shard_ids=shards, body="dummy", document=True, result_per_page=5)
    assert all(r.WhichOneof("sort_value") == "score" for r in binding.search(plain).document.results)
    binding.close()
