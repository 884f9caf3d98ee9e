"""Order by date on the device (bm25_order_kernel, bm25_order_facet_kernel, date_topk_all_kernel) against tests/order_oracle.py,
exactly: ids, dates, counts and totals for OR and AND, use_tf 0 / 1, CREATED / MODIFIED x ASC / DESC, alive bits, corpora of more
than one tile with skip-row terms, k in {1, 10, 100, 1024}, heavy date ties, undated documents, a segment with one distinct date,
the ends of the i64 range and both `mem` modes; out_total equals nidx_txt_search's; ordered + faceted gives the faceted search's
counts and the ordered search's top-k; the listing over several CTAs; and search_sorting.rs through NidxBinding over gRPC across
two shards."""
import uuid

import numpy as np
import pytest

import order_oracle as OO
from nucliadb_b200 import _lib
from test_gpu_facets import _alive, _corpus, _queries, _segment

pytestmark = pytest.mark.gpu


def _dates(n, seed, n_distinct, p_none=0.1):
    rng = np.random.default_rng(seed)
    s = (1_400_000_000 + rng.integers(0, n_distinct, n) * 3_600).astype(np.int64)
    s[rng.random(n) < p_none] = OO.NONE
    return s


def _check(seg, c, qs, qt, qo, k, conj, alive, secs, field, typ, use_tf=False):
    mode = _lib.NIDX_BM25_AND if conj else _lib.NIDX_BM25_OR
    docs, dates, counts, total = seg.search_ordered(qt, qo, k, field, typ, mode)
    _, _, _, plain_total = seg.search(qt, qo, k, mode=mode, use_tf=use_tf)
    assert np.array_equal(total, plain_total)
    for i, q in enumerate(qs):
        d, s, tot = OO.search(c["n_docs"], c["term_off"], c["post_doc"], q, conj, alive, secs, k, typ)
        assert int(counts[i]) == len(d) and int(total[i]) == tot, (i, q)
        assert np.array_equal(docs[i, :len(d)].astype(np.int64), d) and np.array_equal(dates[i, :len(d)], s), (i, q, k)
        assert (docs[i, len(d):] == _lib.NIL).all() and (dates[i, len(d):] == OO.NONE).all()
    return docs, dates, counts, total


@pytest.fixture(scope="module")
def big():
    c = _corpus(11, 300_000)   # 3 tiles of 131 072 documents; terms with df >= 256 have skip rows
    c["created"] = _dates(c["n_docs"], 1, 500)        # ~600 documents per date
    c["modified"] = _dates(c["n_docs"], 2, 40_000)
    c["modified"][:7] = [(1 << 63) - 1, -(1 << 63) + 1, -1, 0, 1, (1 << 62), -(1 << 62)]
    return c


@pytest.mark.parametrize("conj", [False, True])
@pytest.mark.parametrize("use_tf", [False, True])
def test_ordered_search_equals_the_oracle(big, conj, use_tf):
    c = big
    assert int(np.max(np.diff(c["term_off"].astype(np.int64)))) >= 256
    alive = _alive(c["n_docs"], 3)
    seg = _segment(c, alive)
    seg.set_dates(c["created"], c["modified"])
    qs, qt, qo = _queries(c, 31 + conj, 6, conj)
    for field, secs in ((_lib.NIDX_ORDER_CREATED, c["created"]), (_lib.NIDX_ORDER_MODIFIED, c["modified"])):
        for typ in (OO.DESC, OO.ASC):
            for k in (1, 10, 100, 1024):
                _check(seg, c, qs, qt, qo, k, conj, alive, secs, field, typ, use_tf)
    # ordered + faceted: the faceted search's counts, the ordered search's top-k
    mode = _lib.NIDX_BM25_AND if conj else _lib.NIDX_BM25_OR
    plain = seg.search_ordered(qt, qo, 100, _lib.NIDX_ORDER_MODIFIED, OO.ASC, mode)
    both = seg.search_ordered(qt, qo, 100, _lib.NIDX_ORDER_MODIFIED, OO.ASC, mode, facets=[b"l", b"k"])
    faceted = seg.search_faceted(qt, qo, 100, [b"l", b"k"], mode=mode, use_tf=use_tf)
    assert all(np.array_equal(a, b) for a, b in zip(plain, both[:4])) and np.array_equal(both[4], faceted[4])
    seg.close()


def test_single_date_no_dates_device_memory_and_listing(big):
    import torch

    c = big
    alive = _alive(c["n_docs"], 4)
    seg = _segment(c, alive)
    qs, qt, qo = _queries(c, 5, 6, False)
    with pytest.raises(_lib.NidxError) as e:
        seg.search_ordered(qt, qo, 10)
    assert e.value.code == -1
    with pytest.raises(_lib.NidxError):
        seg.list_ordered(10)
    one = np.full(c["n_docs"], 1_700_000_000, dtype=np.int64)   # one distinct date: doc ascending
    one[::7] = OO.NONE
    seg.set_dates(one, c["modified"])
    for typ in (OO.DESC, OO.ASC):
        _check(seg, c, qs, qt, qo, 100, False, alive, one, _lib.NIDX_ORDER_CREATED, typ)
    # device memory mode equals the host mode
    host = seg.search_ordered(qt, qo, 50, _lib.NIDX_ORDER_MODIFIED, OO.DESC)
    dev = seg.search_ordered(torch.from_numpy(qt.astype(np.int32)).cuda(), torch.from_numpy(qo.astype(np.int32)).cuda(), 50, _lib.NIDX_ORDER_MODIFIED, OO.DESC)
    torch.cuda.synchronize()
    assert np.array_equal(dev[0].cpu().numpy().view(np.uint32), host[0]) and np.array_equal(dev[1].cpu().numpy(), host[1])
    assert np.array_equal(dev[2].cpu().numpy(), host[2]) and np.array_equal(dev[3].cpu().numpy().astype(np.uint64), host[3])
    # the listing: several CTAs' worth of documents, every k, both mem modes
    for field, secs in ((_lib.NIDX_ORDER_CREATED, one), (_lib.NIDX_ORDER_MODIFIED, c["modified"])):
        for typ in (OO.DESC, OO.ASC):
            for k in (1, 10, 100, 1024):
                docs, dates, count, total = seg.list_ordered(k, field, typ)
                d, s, tot = OO.list_all(c["n_docs"], alive, secs, k, typ)
                assert count == len(d) and total == tot and np.array_equal(docs[:count].astype(np.int64), d) and np.array_equal(dates[:count], s), (field, typ, k)
            ddev = seg.list_ordered(1024, field, typ, device_out=True)
            torch.cuda.synchronize()
            h = seg.list_ordered(1024, field, typ)
            assert np.array_equal(ddev[0].cpu().numpy().view(np.uint32), h[0]) and np.array_equal(ddev[1].cpu().numpy(), h[1])
            assert int(ddev[2].item()) == h[2] and int(ddev[3].item()) == h[3]
    seg.close()


def test_listing_with_more_k_than_alive_documents():
    c = _corpus(5, 40_000, n_terms=500)
    alive_b = np.zeros(c["n_docs"], dtype=bool)
    alive_b[np.random.default_rng(9).choice(c["n_docs"], 300, replace=False)] = True
    alive = np.concatenate([np.packbits(alive_b, bitorder="little"), np.zeros(-((c["n_docs"] + 7) // 8) % 8, np.uint8)]).view(np.uint64)
    seg = _segment(c, alive)
    secs = _dates(c["n_docs"], 7, 20, p_none=0.3)
    seg.set_dates(secs, secs)
    for typ in (OO.DESC, OO.ASC):
        docs, dates, count, total = seg.list_ordered(1024, _lib.NIDX_ORDER_CREATED, typ)
        d, s, tot = OO.list_all(c["n_docs"], alive, secs, 1024, typ)
        assert total == 300 and count == 300 and np.array_equal(docs[:count].astype(np.int64), d) and np.array_equal(dates[:count], s)
        assert (docs[count:] == _lib.NIL).all()
    seg.close()


def test_search_sorting_through_the_binding_over_grpc(tmp_path):
    """nidx/tests/integration/search_sorting.rs: 20 resources one second apart, a page of 5, ASC / DESC x CREATED / MODIFIED,
    over two shards and gRPC; requests without an order still sort by score."""
    import grpc

    from nidx_binding import NidxBinding
    from nucliadb_b200 import nidx_protos as P

    binding = NidxBinding({"INDEXER__OBJECT_STORE": "file", "INDEXER__FILE_PATH": str(tmp_path)})
    shards = [binding.new_shard("kb", {}) for _ in range(2)]
    (tmp_path / "index").mkdir()
    now = 1_760_000_000
    for i in range(20):
        shard, rid = shards[i % 2], uuid.UUID(int=i + 1).hex
        res = P.Resource()
        res.resource.uuid, res.resource.shard_id, res.shard_id = rid, shard, shard
        res.metadata.created.seconds = now - (20 - i)
        res.metadata.modified.seconds = now - (20 - i)
        res.labels.append(f"/dummy{i:03d}")
        res.texts[f"dummy-{i:03d}"].text = f"Dummy text {i:03d}"
        (tmp_path / f"index/{rid}").write_bytes(res.SerializeToString())
        binding.index(P.IndexMessage(shard=shard, resource=rid, typemessage=0, storage_key=f"index/{rid}", kbid="kb").SerializeToString())
    binding.wait_for_sync()
    search = grpc.insecure_channel(f"127.0.0.1:{binding.searcher_port}").unary_unary(
        P.SEARCH_METHOD, request_serializer=lambda m: m.SerializeToString(), response_deserializer=P.SearchResponse.FromString)
    for sort_by in (P.OrderBy.CREATED, P.OrderBy.MODIFIED):
        for typ in (P.OrderBy.ASC, P.OrderBy.DESC):
            for body in ("", "dummy"):
                req = P.SearchRequest(shard_ids=shards, body=body, document=True, result_per_page=5)
                req.order.sort_by, req.order.type = sort_by, typ
                resp = search(req)
                fields = [r.field for r in resp.document.results]
                assert fields == (sorted(fields) if typ == P.OrderBy.ASC else sorted(fields, reverse=True))
                assert fields == [f"/dummy-{i:03d}" for i in (range(5) if typ == P.OrderBy.ASC else range(19, 14, -1))]
                assert all(r.WhichOneof("sort_value") == "date" and r.date.nanos == 0 for r in resp.document.results)
                assert resp.document.total == 20 and resp.document.next_page
    plain = search(P.SearchRequest(shard_ids=shards, body="dummy", document=True, result_per_page=5))
    assert all(r.WhichOneof("sort_value") == "score" for r in plain.document.results) and plain.document.total == 20
    binding.close()
