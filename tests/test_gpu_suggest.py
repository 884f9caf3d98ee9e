"""Suggest's paragraph pass on the device (ParagraphSearcher.suggest_masks / suggest: nidx_txt_suggest_mask, the keyword pass on views and
nidx_txt_suggest_fuzzy) against the host model (tests/suggest_model.py), bit for bit: hit ids, scores, the pass that answered and the
matches, on random corpora of several segments with deletions and repeated paragraphs, at the top_k, literal length, code point,
phrase, expansion and mask edges."""
import numpy as np
import pytest

import suggest_model as SM
from nucliadb_b200 import suggest as S
from nucliadb_b200.text import ParagraphSearcher, TextDoc

pytestmark = pytest.mark.gpu

ALPHA = "abcdeéßz"


def corpus(seed, n_segs=3, n_docs=300, n_words=400, prefix=""):
    rng = np.random.default_rng(seed)
    words = sorted({prefix + "".join(rng.choice(list(ALPHA), rng.integers(2 if not prefix else 3, 8))) for _ in range(n_words)})
    segs = []
    for s in range(n_segs):
        docs = []
        for d in range(n_docs):
            text = " ".join(rng.choice(words, rng.integers(1, 12)))
            labels = tuple(f"/l/c{c}" for c in range(3) if rng.random() < 0.4) + ("/s/p/en",)
            groups = ("g1",) if rng.random() < 0.3 else ()
            docs.append(TextDoc(f"{s:08x}{d:024x}", "/a/title" if d % 2 else "/a/summary", text, labels, groups=groups, repeated=bool(rng.random() < 0.1)))
        segs.append(docs)
    alive = [rng.random(n_docs) < 0.9 for _ in range(n_segs)]
    return words, segs, alive


def open_searcher(segs, alive):
    ps = ParagraphSearcher.open(segs)
    for s, a in zip(ps.segments, alive):
        s.set_alive(a)
    return ps


def host_bits(words, n):
    return np.unpackbits(np.asarray(words.cpu().numpy() if hasattr(words, "cpu") else words).view(np.uint8), bitorder="little")[:n].astype(bool)


def check(ps, model, alive, body, k, masks):
    got = ps.suggest(body, k, masks)
    mm = [a & host_bits(m, len(a)) for a, m in zip(alive, masks)]
    hits, fuzzy, matches = model.suggest(body, k, mm)
    assert got.fuzzy == fuzzy or not hits, body
    assert [(h.segment, h.doc) for h in got.hits] == [(o, d) for _, o, d in hits], body
    assert np.array_equal(np.asarray([h.score for h in got.hits], np.float32).view(np.uint32),
                          np.asarray([s for s, _, _ in hits], np.float32).view(np.uint32)), body
    for h in got.hits[: S.RESULTS_PER_PAGE]:
        assert h.matches == (matches.get((h.segment, h.doc), []) if fuzzy else []), body
    return got


def mutate(rng, w):
    i = int(rng.integers(0, len(w)))
    return w[:i] + "y" + w[i + 1:]


@pytest.fixture(scope="module")
def random_shard():
    words, segs, alive = corpus(7)
    ps = open_searcher(segs, alive)
    yield words, segs, alive, ps, SM.SuggestModel(segs)
    for s in ps.segments:
        s._gpu.close()


def test_keyword_and_fallback_passes_at_the_edges(random_shard):
    words, segs, alive, ps, model = random_shard
    rng = np.random.default_rng(1)
    masks = ps.suggest_masks()
    rep = [np.asarray([d.repeated for d in s]) for s in segs]
    assert all(np.array_equal(host_bits(m, len(r)), ~r) for m, r in zip(masks, rep))   # no filter: every paragraph not repeated
    long_words = [w for w in words if len(w.encode()) >= 4]
    bodies = [words[3], words[10] + " " + words[20], mutate(rng, long_words[0]), mutate(rng, long_words[5]) + " " + mutate(rng, long_words[9]),
              "ab", "abc", "abcd", "zéß", "éé", "ßzéa", f'"{words[1]} {words[2]}" {mutate(rng, long_words[2])}',
              f'-{words[4]} {mutate(rng, long_words[3])}', f'"{segs[0][5].text.split()[0]} {segs[0][5].text.split()[-1]}"', "qqqq", ""]
    fuzzy_seen = keyword_seen = False
    for body in bodies:
        for k in (1, 10, 11, 20, 1024):
            got = check(ps, model, alive, body, k, masks)
            fuzzy_seen |= got.fuzzy and bool(got.hits)
            keyword_seen |= not got.fuzzy and bool(got.hits)
    assert fuzzy_seen and keyword_seen


def test_masks_none_all_some_filters_and_security(random_shard):
    from nucliadb_b200 import nidx_protos as P

    words, segs, alive, ps, model = random_shard
    rng = np.random.default_rng(2)
    body = mutate(rng, [w for w in words if len(w.encode()) >= 5][0])

    cases = [(None, None, False, lambda d: True), (_facet(P, "/l/c0"), None, False, lambda d: "/l/c0" in d.labels),
             (_facet(P, "/l/nothing"), None, False, lambda d: False), (_facet(P, "/s/p/en"), None, False, lambda d: True),
             (None, ["g1"], False, lambda d: not d.groups or "g1" in d.groups), (None, [], False, lambda d: not d.groups),
             (_facet(P, "/l/c1"), ["g2"], True, lambda d: "/l/c1" in d.labels and not d.groups)]
    for pfilter, security, op_or, keep in cases:
        masks = ps.suggest_masks(security, pfilter, None, op_or)
        for s, m, a in zip(segs, masks, alive):
            want = np.asarray([keep(d) and not d.repeated for d in s]) & a
            assert np.array_equal(host_bits(m, len(s)) & a, want)
        for k in (1, 20):
            check(ps, model, alive, body, k, masks)
            check(ps, model, alive, words[7], k, masks)


def _facet(P, f):
    e = P.FilterExpression()
    e.facet.facet = f
    return e


def test_more_than_ten_thousand_expansions():
    words, segs, alive = corpus(11, n_segs=2, n_docs=6000, n_words=14000, prefix="pre")
    ps = open_searcher(segs, alive)
    try:
        model = SM.SuggestModel(segs)
        assert len(model.expansion("prey", True)) > 10000
        masks = ps.suggest_masks()
        for k in (10, 1024):
            got = check(ps, model, alive, "prey", k, masks)
            assert got.fuzzy and len(got.hits) == k
        bits, counts = ps._suggest_dict.expand([("prey", 1, True)])
        assert int(counts[0]) == len(model.expansion("prey", True))
    finally:
        for s in ps.segments:
            s._gpu.close()


def test_fuzzy_pass_rejects_out_of_range_input(random_shard):
    from nucliadb_b200 import _lib

    _, _, _, ps, _ = random_shard
    seg = ps.segments[0]._gpu
    with pytest.raises(_lib.NidxError) as e:
        seg.suggest_fuzzy([(_lib.NIDX_SG_FUZZY, 0)], None, 0, len(ps.vocab), [], 10)   # no expansion row 0
    assert e.value.code == -1
    with pytest.raises(_lib.NidxError):
        seg.suggest_fuzzy([(_lib.NIDX_SG_TERM, 0)], None, 0, len(ps.vocab), [], 1025)
    with pytest.raises(_lib.NidxError):
        seg.suggest_fuzzy([(_lib.NIDX_SG_TERM, 0)] * 65, None, 0, len(ps.vocab), [], 10)
    with pytest.raises(ValueError):
        ps.suggest("abc", 1025, ps.suggest_masks())


def test_exact_terms_and_phrases_that_match_in_the_fuzzy_pass(random_shard):
    """The fuzzy pass's TERM and PHRASE clauses, which a body cannot make match there (the keyword pass would have answered), run
    directly: scores with their BM25 terms, bit for bit against the model."""
    words, segs, alive, ps, model = random_shard
    rng = np.random.default_rng(3)
    masks = ps.suggest_masks()
    mm = [a & host_bits(m, len(a)) for a, m in zip(alive, masks)]
    text = [d.text.split() for d in segs[1] if len(d.text.split()) >= 3]
    long_words = [w for w in words if len(w.encode()) >= 4]
    cases = [[(S.TERM, text[0][0]), (S.PHRASE, text[1][:2]), (S.FUZZY, mutate(rng, long_words[0])), (S.FUZZY_PREFIX, long_words[1][:3] + "y")],
             [(S.PHRASE, text[2][1:3]), (S.TERM, "qq"), (S.PHRASE, [text[3][0], "qq"]), (S.TERM, text[4][1])],
             [(S.FUZZY, text[5][0]), (S.TERM, text[5][0]), (S.PHRASE, text[5][:3])]]
    for clauses in cases:
        for k in (1, 20, 1024):
            views = [s._gpu.view(m) for s, m in zip(ps.segments, masks)]
            try:
                got = ps._suggest_fuzzy(clauses, k, views)
            finally:
                for v in views:
                    v.close()
            hits, matches = model.fuzzy_pass(clauses, k, mm)
            assert [(h.segment, h.doc) for h in got] == [(o, d) for _, o, d in hits], clauses
            assert np.array_equal(np.asarray([h.score for h in got], np.float32).view(np.uint32),
                                  np.asarray([s for s, _, _ in hits], np.float32).view(np.uint32)), clauses
            for h in got[: S.RESULTS_PER_PAGE]:
                assert h.matches == matches[(h.segment, h.doc)], clauses
    # the exact and phrase clauses did add to the scores: a 0.5 * (count of fuzzy clauses) score is not every hit's
    hits, _ = model.fuzzy_pass(cases[1], 1024, mm)
    assert hits and all(s not in (0.0, 0.5, 1.0) for s, _, _ in hits)


def _json_index(segs, device=0):
    """A JSON document {"a": i % 3} for every paragraph (its own resource) but each fourth, with the paragraph's access groups."""
    import json

    from nucliadb_b200 import json_index as J

    docs = [(d.uuid, J.flatten({"t/p": json.dumps({"a": i % 3})}), tuple(d.groups)) for s in segs for i, d in enumerate(s) if i % 4]
    return J.JsonIndex(docs, device=device)


def test_masks_with_text_and_json_prefilters_under_and_or_with_security(random_shard):
    """suggest_masks with a device prefilter (field_filter on the text index, json_filter on the JSON index, combined as the binding
    combines them) under AND and OR, with a paragraph_filter and security, against a host restatement; then the passes on the model."""
    from nucliadb_b200 import nidx_protos as P
    from nucliadb_b200.text import TextSearcher
    from nucliadb_b200.vector import PrefilterResult
    from test_json_model import path

    words, segs, alive, ps, model = random_shard
    ts = TextSearcher.open([[TextDoc(d.uuid, d.field, d.text, d.labels, groups=d.groups) for d in s] for s in segs])
    ji = _json_index(segs)
    try:
        text_f = _facet(P, "/l/c2")
        json_f = path("t/p", "a", int=1)
        rng = np.random.default_rng(4)
        body = mutate(rng, [w for w in words if len(w.encode()) >= 5][1])
        for op_or in (False, True):
            for security in (None, ["g1"], []):
                for pfilter, use_text, use_json in ((None, True, False), (_facet(P, "/l/c0"), True, False), (_facet(P, "/l/c0"), True, True),
                                                    (None, False, True), (_facet(P, "/l/c1"), False, True)):
                    def sec(d):
                        return security is None or not d.groups or any(g in security for g in d.groups)

                    pre = ts.prefilter(text_f if use_text else None, security=security) if use_text or security is not None else None
                    if use_json:
                        _, found, res_bits = ji.prefilter(json_f, security)
                        pre = (pre or PrefilterResult.all()).combine(ji, res_bits, found, op_or)
                    if pre is not None and pre.kind == "none":
                        continue

                    def text_ok(i, d):
                        return ("/l/c2" in d.labels and sec(d)) if use_text else (sec(d) if security is not None else True)

                    def json_ok(i, d):
                        return i % 4 != 0 and i % 3 == 1 and sec(d)

                    def comb(i, d):
                        if pre is None or pre.kind == "all":
                            return None
                        if not use_json:
                            return text_ok(i, d)
                        t = text_ok(i, d) if (use_text or security is not None) else None
                        if t is None:
                            return json_ok(i, d)
                        return (t or json_ok(i, d)) if op_or else (t and json_ok(i, d))

                    masks = ps.suggest_masks(security, pfilter, pre, op_or)
                    for s, m, a in zip(segs, masks, alive):
                        want = []
                        for i, d in enumerate(s):
                            p = None if pfilter is None else pfilter.facet.facet in d.labels
                            c = comb(i, d)
                            ops = [x for x in (p, c) if x is not None]
                            v = (any(ops) if op_or else all(ops)) if ops else True
                            want.append(v and sec(d) and not d.repeated)
                        assert np.array_equal(host_bits(m, len(s)) & a, np.asarray(want) & a), (op_or, security, pfilter, use_text, use_json)
                    check(ps, model, alive, body, 20, masks)
                    check(ps, model, alive, words[9], 20, masks)
    finally:
        ji.close()
        for s in ts.segments:
            s._gpu.close()
