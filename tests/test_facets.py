"""Facet counts (tantivy's FacetCollector) on a machine without a GPU: the oracle (tests/facet_oracle.py) against a literal
transcription of the counting rule over label strings, the golden fixture, merge_facets (shard_merge.rs:380-414 and its tests),
and the mirror's facet flow (text.py, binding.py) over the emulated C ABI (tests/facet_emulator.py)."""
import os

import numpy as np
import pytest

import facet_emulator
import facet_oracle as FO
from nucliadb_b200 import _lib
from nucliadb_b200 import text as T
from nucliadb_b200.binding import merge_facets

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "facets_small.npz")


def literal_counts(labels_per_doc, matched, request):
    """The counting rule as written: for each requested facet F and each direct child C of F, the number of matched documents
    carrying C or a descendant of C, once per document; a label equal to F counts nothing; '/' counts the top-level facets."""
    out = {}
    for f in dict.fromkeys(r for r in request if r.startswith("/")):
        fs = [] if f == "/" else f[1:].split("/")
        for d, labels in enumerate(labels_per_doc):
            if not matched[d]:
                continue
            kids = set()
            for label in labels:
                ls = label[1:].split("/")
                if len(ls) > len(fs) and ls[: len(fs)] == fs:
                    kids.add("/" + "/".join(ls[: len(fs) + 1]))
            for c in kids:
                out[(f, c)] = out.get((f, c), 0) + 1
    return out


def make_corpus(seed, n_docs=300, n_terms=40):
    """Postings + labels with several labels under one child, labels equal to requested facets, and unlabelled documents."""
    rng = np.random.default_rng(seed)
    vocab = ["/l", "/l/a", "/l/a/x", "/l/a/y", "/l/b", "/l/b/z", "/l/c", "/e/p", "/e/q/r", "/e", "/k/1", "/k/2/3", "/la/x", "/ll"]
    labels = [sorted(set(rng.choice(vocab, size=rng.integers(0, 5)).tolist())) for _ in range(n_docs)]
    pairs = sorted({(int(rng.integers(0, n_terms)), d) for d in range(n_docs) for _ in range(6)})
    term_off = np.zeros(n_terms + 1, dtype=np.uint64)
    term_off[1:] = np.cumsum(np.bincount([p[0] for p in pairs], minlength=n_terms))
    post_doc = np.asarray([p[1] for p in pairs], dtype=np.uint32)
    return labels, term_off, post_doc


def dictionary(labels_per_doc):
    keys = sorted({T.facet_key(l) for ls in labels_per_doc for l in ls})
    ord_of = {k: i for i, k in enumerate(keys)}
    rows = [sorted(ord_of[T.facet_key(l)] for l in set(ls)) for ls in labels_per_doc]
    off = np.zeros(len(rows) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(r) for r in rows])
    return keys, off, np.asarray([o for r in rows for o in r], dtype=np.uint32)


def oracle_counts(keys, off, ords, mask, request):
    valid = [r for r in dict.fromkeys(request) if T.facet_key(r) is not None]
    enc = [T.facet_key(r) for r in valid]
    bucket, b_req, b_ord = FO.plan(keys, enc)
    c = FO.count(off, ords, bucket, len(b_req), mask)
    out = {}
    for b, (r, o) in enumerate(zip(b_req, b_ord)):
        depth = len(FO._segments(enc[r]))
        child = T.facet_path(b"\0".join(FO._segments(keys[o])[: depth + 1]))
        if c[b]:
            out[(valid[r], child)] = int(c[b])
    return out


REQUESTS = [["/l"], ["/l", "/e", "/k"], ["/"], ["/l/a", "/l/b", "/e"], ["", "/l", "/l", "nolabel"], ["/x"], ["/l/a/x"]]


@pytest.mark.parametrize("conj", [False, True])
@pytest.mark.parametrize("with_alive", [False, True])
def test_oracle_counts_equal_the_literal_rule(conj, with_alive):
    for seed in range(3):
        labels, term_off, post_doc = make_corpus(seed)
        keys, off, ords = dictionary(labels)
        rng = np.random.default_rng(100 + seed)
        alive = None
        if with_alive:
            alive = np.packbits(rng.random(len(labels)) < 0.7, bitorder="little")
            alive = np.concatenate([alive, np.zeros(-len(alive) % 8, np.uint8)]).view(np.uint64)
        for terms in ([1, 2, 3], [5], [0, 7, 9, 11, 13], [], [999]):
            mask = FO.matched(len(labels), term_off, post_doc, terms, conj, alive)
            for request in REQUESTS:
                assert oracle_counts(keys, off, ords, mask, request) == literal_counts(labels, mask, request), (seed, terms, request)


def test_nested_request_is_rejected_by_the_oracle():
    with pytest.raises(ValueError):
        FO.plan([b"l", b"l\0a"], [b"l", b"l\0a"])
    with pytest.raises(ValueError):
        FO.plan([b"l"], [b"", b"l"])
    FO.plan([b"l", b"la"], [b"l", b"la"])   # siblings that share a byte prefix are not nested


def load_golden():
    """tests/golden/facets_small.npz -> (labels per document, term_off, post_doc, alive, queries, requests, expected
    {(query, conj, request): {(group, tag): count}})."""
    g = np.load(GOLDEN, allow_pickle=False)
    lo, flat = g["label_off"], [str(x) for x in g["labels"]]
    labels = [flat[lo[i]:lo[i + 1]] for i in range(len(lo) - 1)]
    qo, ro = g["query_off"], g["request_off"]
    queries = [g["query_terms"][qo[i]:qo[i + 1]].tolist() for i in range(len(qo) - 1)]
    requests = [[str(x) for x in g["requests"][ro[i]:ro[i + 1]]] for i in range(len(ro) - 1)]
    exp = {(q, c, r): {} for q in range(len(queries)) for c in (0, 1) for r in range(len(requests))}
    for q, c, r, grp, tag, n in zip(g["exp_q"], g["exp_conj"], g["exp_req"], g["exp_group"], g["exp_tag"], g["exp_count"]):
        exp[(int(q), int(c), int(r))][(str(grp), str(tag))] = int(n)
    return labels, g["term_off"], g["post_doc"], g["alive"], queries, requests, exp


def test_golden_fixture_matches_the_oracle():
    labels, term_off, post_doc, alive, queries, requests, exp = load_golden()
    keys, off, ords = dictionary(labels)
    for qi, terms in enumerate(queries):
        for conj in (0, 1):
            mask = FO.matched(len(labels), term_off, post_doc, terms, bool(conj), alive)
            for ri, request in enumerate(requests):
                assert oracle_counts(keys, off, ords, mask, request) == exp[(qi, conj, ri)]
                assert literal_counts(labels, mask, request) == exp[(qi, conj, ri)]


def test_merge_facets_restates_shard_merge_tests():
    """shard_merge.rs:566-610 / 905-950: counts of equal (group, tag) pairs add up across shards; nothing is cut."""
    def shard(facets):
        out = {}
        for tag, total in facets:
            out.setdefault("/" + tag.split("/")[1], []).append((tag, total))
        return out

    merged = merge_facets([shard([("/l/label-A", 10), ("/l/label-B", 5)]),
                           shard([("/l/label-A", 3), ("/l/label-C", 7), ("/e/table", 12)]),
                           shard([("/e/chair", 3), ("/e/table", 20)])])
    assert merged["/l"] == [("/l/label-A", 13), ("/l/label-C", 7), ("/l/label-B", 5)]
    assert merged["/e"] == [("/e/table", 32), ("/e/chair", 3)]
    many = merge_facets([{"/l": [(f"/l/{i:03d}", 1) for i in range(50)]}, {"/l": [(f"/l/{i:03d}", 1) for i in range(50, 100)]}])
    assert len(many["/l"]) == 100


@pytest.fixture
def emulated(monkeypatch):
    monkeypatch.setattr(_lib, "_lib", facet_emulator.FacetEmulatedLib())


def test_paragraph_faceted_search_groups(emulated):
    """nidx_paragraph/tests/reader.rs:344-370 on the mirror: groups /c, /e, /l are present and "" (not a facet) is absent."""
    field1 = ["/e/mylabel"]
    field2 = ["/f/body", "/l/mylabel2"]
    docs = [T.TextDoc("r", "/t/mytext", txt, tuple(field1 + par)) for txt, par in
            [("this is the title", ["/c/ool"]), ("a first paragraph", ["/e/myentity"]), ("the second one", ["/tantivy", "/test", "/label1"]),
             ("and the third", ["/three", "/label2"])]]
    docs += [T.TextDoc("r", "/t/other", "another field body text", tuple(field2))]
    s = T.ParagraphSearcher.open([docs])
    resp = s.search(T.DocumentSearchRequest(body="", result_per_page=20, faceted=["", "/l", "/e", "/c"]))
    assert sorted(resp.facets) == ["/c", "/e", "/l"]
    assert resp.facets["/e"] == [T.FacetResult("/e/mylabel", 4), T.FacetResult("/e/myentity", 1)]
    assert resp.facets["/l"] == [T.FacetResult("/l/mylabel2", 1)] and resp.results == []


@pytest.mark.parametrize("cls", [T.TextSearcher, T.ParagraphSearcher])
def test_mirror_facets_over_segments_equal_the_literal_rule(emulated, cls):
    rng = np.random.default_rng(5)
    words = [f"w{i}" for i in range(30)]
    labels, _, _ = make_corpus(9, n_docs=120)
    docs = [T.TextDoc(f"u{i}", "/a/f", " ".join(rng.choice(words, size=8)), tuple(labels[i])) for i in range(120)]
    segs = [docs[:50], docs[50:90], docs[90:]]
    s = cls.open(segs)
    for body in ("w1 w2", "w3", "w4 w5 w6", ""):
        toks = T.tokenize(body)
        if not toks:
            matched = np.ones(len(docs), dtype=bool)
        else:
            hit = [set(T.tokenize(d.text)) for d in docs]
            matched = np.asarray([(all if cls.conjunction else any)(t in h for t in toks) for h in hit])
        for request in REQUESTS:
            resp = s.search(T.DocumentSearchRequest(body=body, result_per_page=5, faceted=request))
            lit = literal_counts(labels[:120], matched, request)
            want = {}
            for (f, c), n in lit.items():
                want.setdefault(f, []).append((-n, T.facet_key(c), c))
            assert {f: [(r.tag, r.total) for r in v] for f, v in resp.facets.items()} == {f: [(c, -n) for n, _, c in sorted(v)[:50]] for f, v in want.items()}
            plain = s.search(T.DocumentSearchRequest(body=body, result_per_page=5))
            assert (resp.results, resp.total, resp.next_page) == (plain.results, plain.total, plain.next_page)
            only = s.search(T.DocumentSearchRequest(body=body, result_per_page=5, faceted=request, only_faceted=True))
            assert only.facets == resp.facets and only.results == [] and only.total == 0 and not only.next_page


def test_mirror_rejects_a_nested_request_and_cuts_at_fifty(emulated):
    docs = [T.TextDoc(f"u{i}", "/a/f", "common word", (f"/l/{i:03d}",) + (("/l/hot",) if i % 2 else ())) for i in range(120)]
    s = T.TextSearcher.open([docs[:60], docs[60:]])
    with pytest.raises(ValueError):
        s.search(T.DocumentSearchRequest(body="common", faceted=["/l", "/l/hot"]))
    resp = s.search(T.DocumentSearchRequest(body="common", faceted=["/l"]))
    got = resp.facets["/l"]
    assert len(got) == 50 and got[0] == T.FacetResult("/l/hot", 60)
    assert [r.tag for r in got[1:]] == [f"/l/{i:03d}" for i in range(49)]   # equal counts: facet order
