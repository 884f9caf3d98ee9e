"""Facet counts on the device (bm25_facet_kernel, facet_count_all_kernel) against tests/facet_oracle.py, exactly: OR and AND,
with and without tf, alive bits, min_score and every search-after mode, corpora of more than one tile with skip-row terms, more
buckets than shared memory holds, both `mem` modes; the faceted call's top-k / Count equal nidx_txt_search's bit for bit; and
SearchRequest.faceted through NidxBinding over gRPC across two shards."""
import uuid

import numpy as np
import pytest

import facet_oracle as FO
from nucliadb_b200 import _lib
from nucliadb_b200 import text as T

pytestmark = pytest.mark.gpu


def _corpus(seed, n_docs, n_terms=3000, toks=12, n_wide=0):
    rng = np.random.default_rng(seed)
    zipf = 1.0 / np.arange(1, n_terms + 1) ** 0.9
    terms = rng.choice(n_terms, size=n_docs * toks, p=zipf / zipf.sum()).astype(np.int64)
    docs = np.repeat(np.arange(n_docs, dtype=np.int64), toks)
    key, tf = np.unique(terms * n_docs + docs, return_counts=True)
    post_term, post_doc = key // n_docs, (key % n_docs).astype(np.uint32)
    term_off = np.zeros(n_terms + 1, dtype=np.uint64)
    term_off[1:] = np.cumsum(np.bincount(post_term, minlength=n_terms))
    fieldnorm = rng.integers(4, 40, n_docs).astype(np.uint8)
    # labels: /l/s{a}/x{b} (three levels), /k/{c}, some documents carrying /l itself or several labels under one child;
    # n_wide > 0 adds /m/{0..n_wide-1} (a request with more buckets than shared memory holds)
    keys = {b"l", b"k"} | {f"l\0s{a}".encode() for a in range(40)} | {f"l\0s{a}\0x{b}".encode() for a in range(40) for b in range(25)}
    keys |= {f"k\0{c}".encode() for c in range(30)} | {f"m\0{i:05d}".encode() for i in range(n_wide)}
    keys = sorted(keys)
    n_lab = rng.integers(0, 5, n_docs)
    ords = rng.zipf(1.3, size=int(n_lab.sum())) % len(keys)
    off = np.zeros(n_docs + 1, dtype=np.uint64)
    rows = np.split(ords, np.cumsum(n_lab)[:-1])
    rows = [np.unique(r) for r in rows]
    off[1:] = np.cumsum([len(r) for r in rows])
    flat = np.concatenate(rows).astype(np.uint32) if len(rows) else np.zeros(0, np.uint32)
    return dict(n_docs=n_docs, n_terms=n_terms, term_off=term_off, post_doc=post_doc, post_tf=tf.astype(np.uint32), fieldnorm=fieldnorm,
                keys=keys, doc_off=off, ords=flat)


def _segment(c, alive=None):
    from nucliadb_b200.segment import TextSegment

    seg = TextSegment.create(c["n_docs"], c["n_terms"], c["term_off"], c["post_doc"], c["post_tf"], c["fieldnorm"])
    seg.set_facets(c["keys"], c["doc_off"], c["ords"])
    if alive is not None:
        seg.set_alive(alive)
    return seg


def _alive(n, seed):
    bits = np.random.default_rng(seed).random(n) < 0.8
    b = np.packbits(bits, bitorder="little")
    return np.concatenate([b, np.zeros(-len(b) % 8, np.uint8)]).view(np.uint64)


def _queries(c, seed, nq, conj):
    rng = np.random.default_rng(seed)
    qs = []
    for i in range(nq):
        n = int(rng.integers(1, 4)) if conj else int(rng.integers(1, 60))
        qs.append(sorted(set(rng.integers(0, 40 if conj else c["n_terms"], n).tolist())))
    qo = np.asarray([0] + list(np.cumsum([len(q) for q in qs])), dtype=np.uint32)
    return qs, np.asarray([t for q in qs for t in q], dtype=np.uint32), qo


def _expected(c, qs, request, conj, alive):
    bucket, b_req, _ = FO.plan(c["keys"], request)
    return np.stack([FO.count(c["doc_off"], c["ords"], bucket, len(b_req), FO.matched(c["n_docs"], c["term_off"], c["post_doc"], q, conj, alive))
                     for q in qs])


@pytest.fixture(scope="module")
def big():
    return _corpus(11, 300_000, n_wide=6000)   # 3 tiles of 131 072 documents; terms with df >= 256 have skip rows


@pytest.mark.parametrize("conj", [False, True])
@pytest.mark.parametrize("use_tf", [False, True])
def test_device_counts_equal_the_oracle_and_the_search_is_unchanged(big, conj, use_tf):
    c = big
    assert int(np.max(np.diff(c["term_off"].astype(np.int64)))) >= 256
    alive = _alive(c["n_docs"], 3)
    seg = _segment(c, alive)
    qs, qt, qo = _queries(c, 21 + conj, 12, conj)
    mode = _lib.NIDX_BM25_AND if conj else _lib.NIDX_BM25_OR
    for request in ([b"l"], [b"l", b"k"], [b""], [b"l\0s1", b"l\0s3", b"k"], [b"m"]):   # [b"m"]: 6000 buckets, global counters
        want = _expected(c, qs, request, conj, alive)
        docs, scores, counts, total = seg.search(qt, qo, 101, mode=mode, use_tf=use_tf)
        fd, fs, fc, ft, facets = seg.search_faceted(qt, qo, 101, request, mode=mode, use_tf=use_tf)
        assert np.array_equal(facets, want), request
        assert np.array_equal(fd, docs) and np.array_equal(fs.view(np.uint32), scores.view(np.uint32)) and np.array_equal(fc, counts) and np.array_equal(ft, total)
        assert (want.sum(axis=1) > 0).any()
    # min_score and search-after change the results, never the matched set
    med = float(np.median(scores[0, : max(int(counts[0]), 1)]))
    for after in (None, (med, 1, 0), (med, 2, int(docs[0, 0])), (med, 3, 0)):
        d0, s0, c0, t0 = seg.search(qt, qo, 50, mode=mode, use_tf=use_tf, min_score=med / 2, after=after)
        d1, s1, c1, t1, f1 = seg.search_faceted(qt, qo, 50, [b"l", b"k"], mode=mode, use_tf=use_tf, min_score=med / 2, after=after)
        assert np.array_equal(d0, d1) and np.array_equal(s0.view(np.uint32), s1.view(np.uint32)) and np.array_equal(c0, c1) and np.array_equal(t0, t1)
        assert np.array_equal(f1, _expected(c, qs, [b"l", b"k"], conj, alive))
    seg.close()


def test_device_memory_mode_and_all_documents(big):
    import torch

    c = big
    alive = _alive(c["n_docs"], 4)
    seg = _segment(c, alive)
    qs, qt, qo = _queries(c, 5, 6, False)
    out = seg.search_faceted(torch.from_numpy(qt.astype(np.int32)).cuda(), torch.from_numpy(qo.astype(np.int32)).cuda(), 20, [b"l", b"k"])
    torch.cuda.synchronize()
    assert np.array_equal(out[4].cpu().numpy().astype(np.int64), _expected(c, qs, [b"l", b"k"], False, alive))
    host = seg.search_faceted(qt, qo, 20, [b"l", b"k"])
    assert np.array_equal(out[0].cpu().numpy().view(np.uint32), host[0]) and np.array_equal(out[3].cpu().numpy().astype(np.uint64), host[3])
    for request in ([b"l"], [b""], [b"l", b"k", b"m"], [b"m"]):
        bucket, b_req, b_ord = FO.plan(c["keys"], request)
        want = FO.count(c["doc_off"], c["ords"], bucket, len(b_req), FO.alive_mask(c["n_docs"], alive))
        assert np.array_equal(seg.facet_count_all(request).astype(np.int64), want)
        dev = seg.facet_count_all(request, device_out=True)
        torch.cuda.synchronize()
        assert np.array_equal(dev.cpu().numpy().astype(np.int64), want)
        r, o = seg.facet_buckets(request + request[:1])   # duplicates collapse
        assert np.array_equal(r, b_req) and np.array_equal(o, b_ord)
    with pytest.raises(_lib.NidxError) as e:
        seg.facet_buckets([b"l", b"l\0s1"])
    assert e.value.code == -1
    seg.close()


def test_faceted_search_through_the_binding_over_grpc(tmp_path):
    import grpc

    from nidx_binding import NidxBinding
    from nucliadb_b200 import nidx_protos as P

    binding = NidxBinding({"INDEXER__OBJECT_STORE": "file", "INDEXER__FILE_PATH": str(tmp_path)})
    shards = [binding.new_shard("kb", {}) for _ in range(2)]
    rng = np.random.default_rng(8)
    words = ["fox", "dog", "graph", "hbm", "search", "label"]
    indexed = []   # (shard, rid, field labels, paragraph labels, text)
    (tmp_path / "index").mkdir()
    for i in range(24):
        shard, rid = shards[i % 2], uuid.UUID(int=i + 1).hex
        res = P.Resource()
        res.resource.uuid, res.resource.shard_id, res.shard_id = rid, shard, shard
        rlabels = sorted({f"/l/set{int(rng.integers(0, 3))}/x{int(rng.integers(0, 4))}" for _ in range(int(rng.integers(0, 3)))} | ({"/k/a"} if i % 3 else set()))
        res.labels.extend(rlabels)
        text = " ".join(rng.choice(words, size=5))
        res.texts["a/title"].text = text
        plabel = f"/k/p{i % 4}"
        par = res.paragraphs["a/title"].paragraphs[f"{rid}/a/title/0-{len(text)}"]
        par.start, par.end, par.field = 0, len(text), "a/title"
        par.labels.append(plabel)
        (tmp_path / f"index/{rid}").write_bytes(res.SerializeToString())
        binding.index(P.IndexMessage(shard=shard, resource=rid, typemessage=0, storage_key=f"index/{rid}", kbid="kb").SerializeToString())
        indexed.append((rid, rlabels, plabel, text))
    binding.wait_for_sync()
    search = grpc.insecure_channel(f"127.0.0.1:{binding.searcher_port}").unary_unary(
        P.SEARCH_METHOD, request_serializer=lambda m: m.SerializeToString(), response_deserializer=P.SearchResponse.FromString)

    def python_counts(body, paragraph):
        out = {}
        for rid, rlabels, plabel, text in indexed:
            if body and body not in text.split():
                continue
            labels = list(rlabels) + ([plabel] if paragraph else [])
            for group in ("/l", "/k"):
                for c in {"/".join(l.split("/")[:3]) for l in labels if l.startswith(group + "/")}:
                    out.setdefault(group, {})[c] = out.setdefault(group, {}).get(c, 0) + 1
        return {g: sorted(v.items(), key=lambda t: (-t[1], T.facet_key(t[0]))) for g, v in out.items()}

    for body in ("fox", ""):
        base = P.SearchRequest(shard_ids=shards, body=body, result_per_page=5, paragraph=True, document=True)
        faceted = P.SearchRequest()
        faceted.CopyFrom(base)
        faceted.faceted.labels.extend(["/l", "/k"])
        plain, resp = search(base), search(faceted)
        for kind, par in (("document", False), ("paragraph", True)):
            got = {g: [(r.tag, r.total) for r in v.facetresults] for g, v in getattr(resp, kind).facets.items()}
            assert got == python_counts(body, par), (body, kind)
            assert len(getattr(plain, kind).facets) == 0
            a, b = getattr(plain, kind), getattr(resp, kind)
            assert list(a.results) == list(b.results) and a.total == b.total and a.next_page == b.next_page
        faceted.only_faceted = True
        only = search(faceted)
        for kind in ("document", "paragraph"):
            r = getattr(only, kind)
            assert len(r.results) == 0 and r.total == 0 and not r.next_page and dict(r.facets) == dict(getattr(resp, kind).facets)
    nested = P.SearchRequest(shard_ids=shards, body="fox", result_per_page=5, document=True)
    nested.faceted.labels.extend(["/l", "/l/set1"])
    with pytest.raises(grpc.RpcError) as e:
        search(nested)
    assert e.value.code() == grpc.StatusCode.INVALID_ARGUMENT
    binding.close()
