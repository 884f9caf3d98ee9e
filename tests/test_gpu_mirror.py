"""The reference's own integration tests, restated against the Python mirror of its interface
(nucliadb_b200.vector / .text) running on the GPU.  Each test names the Rust test it follows."""
import os
import uuid

import numpy as np
import pytest

import oracle as O
from oracle import disk_v2
from conftest import make_queries, make_vectors
from nucliadb_b200 import _lib
from nucliadb_b200 import text as T
from nucliadb_b200 import vector as V
from nucliadb_b200.segment import VectorSegment

pytestmark = pytest.mark.gpu

RID = "9cb39c75f8d9498d8f82d92b173011f5"
DIM = 64


def sentence(i):
    v = np.zeros(DIM, np.float32)
    v[i] = 1.0
    return v


@pytest.mark.parametrize("similarity", [V.Similarity.Dot, V.Similarity.Cosine])
def test_basic_search(similarity):  # nidx_vector/tests/test_basic_search.rs:39-143
    cfg = V.VectorConfig(dimension=DIM, similarity=similarity)
    elems = [V.Elem(f"{RID}/a/title/0-{i}", [sentence(i)]) for i in range(DIM)]
    seg = V.VectorIndexer.index_elems(elems, cfg)
    searcher = V.VectorSearcher.open(cfg, [(seg, 1)])
    res = searcher.search(V.VectorSearchRequest(vector=sentence(5), result_per_page=10, min_score=-1.0))
    assert len(res.documents) == 10
    assert res.documents[0].doc_id == f"{RID}/a/title/0-5"
    assert res.documents[0].score > 0.9999 and res.documents[1].score < 0.0001
    q = np.zeros(DIM, np.float32)
    q[42], q[43], q[44], q[45] = 0.7, 0.59, 0.35, 0.2
    res = searcher.search(V.VectorSearchRequest(vector=q, result_per_page=10, min_score=-1.0))
    assert [d.doc_id for d in res.documents[:4]] == [f"{RID}/a/title/0-{i}" for i in (42, 43, 44, 45)]
    assert res.documents[0].score > 0.6 and res.documents[1].score > 0.5 and res.documents[2].score > 0.3 and res.documents[3].score > 0.15
    assert res.documents[5].score == 0.0


def test_dimension_mismatch_is_an_error():  # searcher.rs:255-262, searcher.rs test at 590-606
    cfg = V.VectorConfig(dimension=3, similarity=V.Similarity.Dot)
    seg = V.VectorIndexer.index_elems([V.Elem(f"{RID}/f/field/0-100", [[1.0, 2.0, 3.0]])], cfg)
    searcher = V.VectorSearcher.open(cfg, [(seg, 1)])
    with pytest.raises(V.NidxError):
        searcher.search(V.VectorSearchRequest(vector=[4.0, 6.0], result_per_page=20))


def test_vectors_deduplication():  # searcher.rs:610-686
    cfg = V.VectorConfig(dimension=3, similarity=V.Similarity.Dot)
    elems = [V.Elem(f"{RID}/f/field/0-100", [[1.0, 2.0, 3.0]]), V.Elem(f"{RID}/f/field/100-200", [[1.0, 2.0, 3.0]])]
    seg = V.VectorIndexer.index_elems(elems, cfg)
    searcher = V.VectorSearcher.open(cfg, [(seg, 1)])
    r = searcher.search(V.VectorSearchRequest(vector=[4.0, 6.0, 7.0], result_per_page=20, with_duplicates=True))
    assert len(r.documents) == 2
    r = searcher.search(V.VectorSearchRequest(vector=[4.0, 6.0, 7.0], result_per_page=20, with_duplicates=False))
    assert len(r.documents) == 1


def test_deletions_and_sequences():  # tests/test_basic_search.rs:145-214, lib.rs:188-199
    cfg = V.VectorConfig(dimension=DIM, similarity=V.Similarity.Dot)
    other = "00000000000000000000000000000002"
    seg1 = V.VectorIndexer.index_elems([V.Elem(f"{RID}/a/title/0-{i}", [sentence(i)]) for i in range(10)], cfg)
    seg2 = V.VectorIndexer.index_elems([V.Elem(f"{other}/a/title/0-{i}", [sentence(i + 10)]) for i in range(10)], cfg)
    searcher = V.VectorSearcher.open(cfg, [(seg1, 1), (seg2, 3)], deletions=[(RID, 2), (other, 2)])
    r = searcher.search(V.VectorSearchRequest(vector=sentence(3), result_per_page=10, min_score=-1.0))
    assert all(d.doc_id.startswith(other) for d in r.documents) and len(r.documents) == 10   # seq 2 deletion hides only seg1 (seq 1)


def test_filtered_search():  # tests/test_basic_search.rs:216-392
    cfg = V.VectorConfig(dimension=DIM, similarity=V.Similarity.Dot)
    rids = [f"{i:032x}" for i in range(1, 5)]
    labels = [["/l/a", "/l/b"], ["/l/a"], ["/l/b"], []]
    elems = [V.Elem(f"{rids[i]}/a/title/0-1", [sentence(i)], labels=labels[i]) for i in range(4)]
    seg = V.VectorIndexer.index_elems(elems, cfg)
    searcher = V.VectorSearcher.open(cfg, [(seg, 1)])

    def ids(formula=None, prefilter=None, op=V.FilterOperator.And):
        req = V.VectorSearchRequest(vector=np.ones(DIM, np.float32), result_per_page=10, min_score=-1.0, filtering_formula=formula, filter_operator=op)
        return sorted(d.doc_id[:32] for d in searcher.search(req, prefilter).documents)

    assert ids() == rids
    assert ids(V.Literal("/l/a")) == rids[:2]
    assert ids(V.Operation("and", (V.Literal("/l/a"), V.Literal("/l/b")))) == rids[:1]
    assert ids(V.Operation("or", (V.Literal("/l/a"), V.Literal("/l/b")))) == rids[:3]
    assert ids(V.Not(V.Literal("/l/a"))) == rids[2:]
    pre = V.PrefilterResult.some([V.FieldId(uuid.UUID(rids[3]), "/a/title"), V.FieldId(uuid.UUID(rids[0]), "/a/title")])
    assert ids(None, pre) == [rids[0], rids[3]]
    assert ids(V.Literal("/l/a"), pre) == [rids[0]]
    assert ids(V.Literal("/l/a"), pre, V.FilterOperator.Or) == [rids[0], rids[1], rids[3]]
    assert ids(None, V.PrefilterResult.none()) == []


def test_min_score():  # tests/test_min_score.rs:61-164
    cfg = V.VectorConfig(dimension=4, similarity=V.Similarity.Dot)
    vecs = [[1, 0, 0, 0], [0.9, 0.1, 0, 0], [0.5, 0.5, 0, 0], [0, 1, 0, 0], [-1, 0, 0, 0]]
    seg = V.VectorIndexer.index_elems([V.Elem(f"{RID}/a/t/0-{i}", [np.asarray(v, np.float32)]) for i, v in enumerate(vecs)], cfg)
    searcher = V.VectorSearcher.open(cfg, [(seg, 1)])
    n = lambda ms: len(searcher.search(V.VectorSearchRequest(vector=[1.0, 0, 0, 0], result_per_page=10, min_score=ms)).documents)
    assert n(-1.0) == 5 and n(0.0) == 4 and n(0.6) == 2 and n(0.95) == 1 and n(1.5) == 0


def test_segment_files_round_trip(tmp_path):  # hnsw/disk/v2.rs:339-473 + data_store/v2/vector_store.rs
    v = make_vectors(3000, 48, seed=21)
    seg = VectorSegment.create(v, 48, similarity=_lib.NIDX_SIM_DOT, m=8, m0=16, ef_construction=40)
    seg.build_hnsw(seed=2, max_batch=64)
    g = seg.get_graph()
    seg.save(str(tmp_path))
    # the files are the reference's: check them with the pure-Python restatement of the format
    graph = open(tmp_path / "hnsw.graph", "rb").read()
    assert disk_v2.entrypoint(graph) == (g["entry_node"], g["entry_layer"])
    upper_off = np.concatenate([[0], np.cumsum(g["level"])[:-1]])
    for node in (0, 1, 17, 2999, int(g["entry_node"])):
        assert disk_v2.get_out_edges(graph, node, 0) == [int(x) for x in g["adj0"][node] if x != 0xFFFFFFFF]
        for l in range(1, int(g["level"][node]) + 1):
            assert disk_v2.get_out_edges(graph, node, l) == [int(x) for x in g["adjU"][int(upper_off[node]) + l - 1] if x != 0xFFFFFFFF]
    raw = open(tmp_path / "vectors.bin", "rb").read()
    assert raw == disk_v2.write_vectors_bin(v, range(len(v)))
    assert os.path.getsize(tmp_path / "hnsw.edges") == 4 * (int((g["adj0"] != 0xFFFFFFFF).sum()) + int((g["adjU"][: g["upper_rows"]] != 0xFFFFFFFF).sum()))
    # and open() gives back a segment that searches identically
    seg2 = VectorSegment.open(str(tmp_path), 48, similarity=_lib.NIDX_SIM_DOT, m=8, m0=16, ef_construction=40)
    q = make_queries(v, 32)
    a = seg.search(q, 10, ef=40, method=_lib.NIDX_METHOD_HNSW)
    b = seg2.search(q, 10, ef=40, method=_lib.NIDX_METHOD_HNSW)
    assert (a[0] == b[0]).all() and np.array_equal(a[1], b[1])
    g2 = seg2.get_graph()
    assert (g2["adj0"] == g["adj0"]).all() and np.array_equal(g2["w0"], g["w0"])


def test_open_reference_written_segment(tmp_path):
    """A segment written in the reference's format by the oracle (not by us) loads and searches."""
    v = make_vectors(500, 32, seed=22)
    og = O.hnsw_build(v, sim=O.SIM_DOT, M=30, M0=60, efC=100)       # reference constants
    layers = []
    for l in range(og.entry_layer + 1):
        layers.append({n: [(int(t), float(w)) for t, w in zip(og.edges(n, l), (og.w0[n] if l == 0 else og.wU[int(og.upper_off[n]) + l - 1]))]
                       for n in range(len(v)) if og.level[n] >= l})
    graph, edges = disk_v2.serialize_graph(layers, len(v), og.entry_node, og.entry_layer)
    open(tmp_path / "hnsw.graph", "wb").write(graph)
    open(tmp_path / "hnsw.edges", "wb").write(edges)
    open(tmp_path / "vectors.bin", "wb").write(disk_v2.write_vectors_bin(v, range(len(v))))
    seg = VectorSegment.open(str(tmp_path), 32, similarity=_lib.NIDX_SIM_DOT)     # default config = reference constants
    q = make_queries(v, 16)
    ids, sc, cnt = seg.search(q, 5, ef=30, min_score=0.0, method=_lib.NIDX_METHOD_HNSW)
    oi, os_, oc, _ = O.hnsw_search(v, og, q, 5, 30, sim=O.SIM_DOT, min_score=0.0)
    assert (ids == oi).all() and np.array_equal(sc, os_) and (cnt == oc).all()


def test_text_search_and_min_score():  # nidx_text/tests/test_search.rs:311-332, nidx_paragraph/tests/reader.rs:316-340
    docs = [T.TextDoc("r1", "a/title", "The little prince lives on a small planet"),
            T.TextDoc("r1", "a/summary", "A prince and a fox become friends on the planet"),
            T.TextDoc("r2", "a/title", "Shoot for the moon and the stars"),
            T.TextDoc("r3", "a/title", "nothing to see here")]
    s = T.TextSearcher.open([docs[:2], docs[2:]])
    r = s.search(T.DocumentSearchRequest(body="prince planet", result_per_page=20, min_score=0.0))
    assert r.total == 2 and [x.field for x in r.results] and {x.uuid for x in r.results} == {"r1"}
    assert s.search(T.DocumentSearchRequest(body="prince planet", result_per_page=20, min_score=100.0)).results == []
    assert s.search(T.DocumentSearchRequest(body="prince moon", result_per_page=20)).total == 0        # conjunction by default
    p = T.ParagraphSearcher.open([docs[:2], docs[2:]])
    r = p.search(T.DocumentSearchRequest(body="prince moon", result_per_page=20))
    assert r.total == 3                                                                                     # OR of terms
    assert r.results[0].score.bm25 >= r.results[-1].score.bm25
    assert all((x.score.docaddr >> 32) in (0, 1) for x in r.results)
    r1 = p.search(T.DocumentSearchRequest(body="prince moon", result_per_page=1))
    assert r1.next_page and len(r1.results) == 1


def test_maxsim():  # nidx_vector/tests/test_maxsim.rs:22-150
    e = np.eye(5, dtype=np.float32)
    query = np.concatenate([e[0], e[3]])
    d0, d1, d2 = [e[1], e[2], e[4]], [e[0], e[1], e[2]], [e[0], e[2], e[3]]
    cfg = V.VectorConfig(dimension=5, similarity=V.Similarity.Cosine, vector_cardinality=V.VectorCardinality.Multi)
    elems = [V.Elem(f"{RID}/f/d0/0-123", d0), V.Elem(f"{RID}/f/d1/0-123", d1), V.Elem(f"{RID}/f/d2/0-123", d2)]
    seg = V.VectorIndexer.index_elems(elems, cfg)
    searcher = V.VectorSearcher.open(cfg, [(seg, 1)])
    r = searcher.search(V.VectorSearchRequest(vector=query, result_per_page=1, min_score=-10.0))
    assert len(r.documents) == 1 and r.documents[0].doc_id == f"{RID}/f/d2/0-123" and r.documents[0].score == 2.0
    r = searcher.search(V.VectorSearchRequest(vector=query, result_per_page=10, min_score=1.5))   # min_score on the maxsim score only
    assert len(r.documents) == 1 and r.documents[0].doc_id == f"{RID}/f/d2/0-123" and r.documents[0].score == 2.0
    r = searcher.search(V.VectorSearchRequest(vector=query, result_per_page=2, min_score=-10.0))
    assert [d.doc_id for d in r.documents] == [f"{RID}/f/d2/0-123", f"{RID}/f/d1/0-123"]
    assert [d.score for d in r.documents] == [2.0, 1.0]


def test_paragraph_search_after():  # nidx_paragraph/src/reader.rs:350-392 is_after; nidx/tests/integration/search_after.rs
    docs = [T.TextDoc(f"r{i}", "a/title", "prince " + " ".join(["filler"] * i)) for i in range(12)]
    p = T.ParagraphSearcher.open([docs[:6], docs[6:]])
    full = p.search(T.DocumentSearchRequest(body="prince", result_per_page=20))
    assert len(full.results) == 12 and full.total == 12
    page1 = p.search(T.DocumentSearchRequest(body="prince", result_per_page=5))
    assert page1.next_page and [r.uuid for r in page1.results] == [r.uuid for r in full.results[:5]]
    last = page1.results[-1]
    page2 = p.search(T.DocumentSearchRequest(body="prince", result_per_page=5, search_after=T.SearchAfter(last.score.bm25, "keep_after", last.score.docaddr)))
    assert page2.total == 12                                   # Count still sees everything
    got, want = [r.uuid for r in page2.results], [r.uuid for r in full.results[5:10]]
    assert got == want
    none = p.search(T.DocumentSearchRequest(body="prince", result_per_page=5, search_after=T.SearchAfter(full.results[-1].score.bm25, "drop")))
    assert none.results == []
    keep = p.search(T.DocumentSearchRequest(body="prince", result_per_page=20, search_after=T.SearchAfter(full.results[3].score.bm25, "keep")))
    assert [r.uuid for r in keep.results] == [r.uuid for r in full.results if r.score.bm25 <= full.results[3].score.bm25]


def test_merge_segments_with_deletions():  # nidx_vector/src/segment/tests.rs merge flows + lib.rs:166-200
    cfg = V.VectorConfig(dimension=DIM, similarity=V.Similarity.Dot)
    other = "00000000000000000000000000000002"
    seg1 = V.VectorIndexer.index_elems([V.Elem(f"{RID}/a/title/0-{i}", [sentence(i)], labels=["/l/one"]) for i in range(20)], cfg)
    seg2 = V.VectorIndexer.index_elems([V.Elem(f"{other}/a/title/0-{i}", [sentence(i + 20)], labels=["/l/two"]) for i in range(30)], cfg)
    merged = V.VectorIndexer.merge(cfg, [(seg1, 1), (seg2, 3)], deletions=[(RID, 2), (other, 2)])
    assert merged.records == 30 and all(k.startswith(other) for k in merged.keys)       # seq-2 deletion only hits seg1 (seq 1)
    searcher = V.VectorSearcher.open(cfg, [(merged, 4)])
    r = searcher.search(V.VectorSearchRequest(vector=sentence(25), result_per_page=3, min_score=-1.0))
    assert r.documents[0].doc_id == f"{other}/a/title/0-5" and r.documents[0].score > 0.9999
    r = searcher.search(V.VectorSearchRequest(vector=sentence(25), result_per_page=3, min_score=-1.0, filtering_formula=V.Literal("/l/one")))
    assert r.documents == []
    both = V.VectorIndexer.merge(cfg, [(V.VectorIndexer.index_elems([V.Elem(f"{RID}/a/title/0-{i}", [sentence(i)]) for i in range(5)], cfg), 1), (merged, 4)])
    assert both.records == 35 and both.keys[0].startswith(other)                         # largest segment first (segment.rs:103-105)
    # merge_indexes reuses the first operand's graph when it has no deletions (segment.rs:143-167)
    g2, gm, gb = seg2.segment.get_graph(), merged.segment.get_graph(), both.segment.get_graph()
    assert np.array_equal(g2["adj0"], gm["adj0"]) and np.array_equal(g2["level"], gm["level"])      # nothing to insert: the graph is seg2's
    assert np.array_equal(gb["level"][:30], gm["level"]) and (gb["adj0"][30:, 0] != 0xFFFFFFFF).all()  # the 5 new nodes are linked in
    r = V.VectorSearcher.open(cfg, [(both, 5)]).search(V.VectorSearchRequest(vector=sentence(3), result_per_page=1, min_score=-1.0), method=_lib.NIDX_METHOD_HNSW)
    assert r.documents[0].doc_id == f"{RID}/a/title/0-3"
