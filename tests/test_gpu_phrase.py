"""Exact phrases on the device (nidx_txt_set_positions + nidx_txt_search_phrases) against tests/phrase_model.py bit for bit:
ids, scores, counts and Count, in OR and AND, beside Basic and TF terms, with deletions, union statistics, search-after, facets and
date order; the ABI's limits; and the calls without phrases equal to nidx_txt_search / _faceted / _ordered."""
import numpy as np
import pytest

import bm25_model as M
import phrase_model as PM

pytestmark = pytest.mark.gpu


def make_corpus(seed, n_docs, vocab=300, long_every=0):
    """Token-id documents with positions (a dropped long token every so often leaves a gap) -> (doc_tokens, positions dict)."""
    rng = np.random.default_rng(seed)
    docs = []
    for d in range(n_docs):
        n = int(rng.integers(3, 30))
        if long_every and d % long_every == 0:
            n = 90
        ids = (rng.zipf(1.3, n) - 1) % vocab
        if long_every and d % long_every == 0:
            ids = np.resize(np.arange(7, 7 + 64), n)   # a long run of distinct terms: phrases of up to 64 words match
        long = bool(long_every) and d % long_every == 0
        pos, toks = 0, []
        for t in ids:
            if not long and rng.random() < 0.03:
                pos += 1   # a token RemoveLongFilter dropped
            toks.append((pos, int(t)))
            pos += 1
        docs.append(toks)
    return docs


def index(docs, n_terms):
    """-> term_off, post_doc, post_tf, fieldnorm_id, positions dict, positions array (posting order)."""
    pos = PM.token_positions(docs)
    pairs = sorted(pos)
    term_off = np.zeros(n_terms + 1, np.uint64)
    term_off[1:] = np.cumsum(np.bincount([t for t, _ in pairs], minlength=n_terms))
    post_doc = np.asarray([d for _, d in pairs], np.uint32)
    post_tf = np.asarray([len(pos[p]) for p in pairs], np.uint32)
    from nucliadb_b200.text import fieldnorm_to_id
    fn = np.asarray([fieldnorm_to_id(len(t)) for t in docs], np.uint8)
    return term_off, post_doc, post_tf, fn, pos, PM.positions_in_posting_order(term_off, post_doc, pos)


def sample_phrases(docs, rng, n, lo=2, hi=5):
    out = []
    while len(out) < n:
        d = docs[int(rng.integers(len(docs)))]
        m = int(rng.integers(lo, hi + 1))
        if len(d) < m:
            continue
        s = int(rng.integers(len(d) - m + 1))
        out.append([t for _, t in d[s:s + m]])
    return out


N_TERMS = 300
N_DOCS = 4096 * 3 + 77   # four fine tiles, the last one partial


@pytest.fixture(scope="module")
def seg():
    from nucliadb_b200.segment import TextSegment
    docs = make_corpus(1, N_DOCS, N_TERMS, long_every=997)
    term_off, post_doc, post_tf, fn, pos, flat = index(docs, N_TERMS)
    s = TextSegment.create(N_DOCS, N_TERMS, term_off, post_doc, post_tf, fn)
    s.set_positions(flat)
    model = PM.PhraseModel(N_DOCS, N_TERMS, term_off, post_doc, post_tf, fn, pos=pos)
    return s, model, docs


def queries(docs, seed, nq):
    rng = np.random.default_rng(seed)
    qs = []
    for i in range(nq):
        terms = [int(t) for t in rng.integers(0, N_TERMS + 3, int(rng.integers(0, 4)))]   # ids >= N_TERMS: unknown
        phrases = sample_phrases(docs, rng, int(rng.integers(1, 3)))
        if i % 7 == 0:
            phrases.append([int(t) for t in rng.integers(0, 20, 2)])   # frequent words, mostly no match
        if i % 11 == 0:
            phrases.append([0, 0])                                     # a repeated term
        if i % 13 == 0:
            phrases.append([5, N_TERMS + 1])                           # a word the dictionary lacks
        qs.append((terms, phrases))
    return qs


def run(s, qs, k, **kw):
    qt = np.asarray([t for q in qs for t in q[0]], np.uint32)
    qo = np.zeros(len(qs) + 1, np.uint32)
    qo[1:] = np.cumsum([len(q[0]) for q in qs])
    ph = [(i, p) for i, q in enumerate(qs) for p in q[1]]
    return s.search_phrases(qt, qo, ph, k, **kw)


def check(got, want):
    for g, w, name in zip(got, want, ("docs", "scores", "counts", "total")):
        assert np.array_equal(np.asarray(g), np.asarray(w)), name


@pytest.mark.parametrize("mode,use_tf", [(M.OR, False), (M.OR, True), (M.AND, True), (M.AND, False)])
def test_phrases_bit_identical(seg, mode, use_tf):
    s, model, docs = seg
    qs = queries(docs, 2, 1100)   # one batch of more than 1024 queries
    k = 16
    check(run(s, qs, k, mode=mode, use_tf=use_tf), model.search(qs, k, mode=mode, use_tf=use_tf))
    check(run(s, qs[:1], k, mode=mode, use_tf=use_tf), model.search(qs[:1], k, mode=mode, use_tf=use_tf))


def test_phrase_lengths_2_to_64(seg):
    s, model, docs = seg
    run_ = [t for _, t in docs[0]]   # document 0 holds the 64 distinct terms 7 .. 70 in a row
    qs = [([], [run_[i:i + m]]) for m in (2, 3, 8, 17, 33, 64) for i in (0, 1)]
    got = run(s, qs, 8, use_tf=False)
    check(got, model.search(qs, 8, use_tf=False))
    assert (np.asarray(got[3]) >= 1).all()


def test_skip_rows_on_both_sides(seg):
    """Drivers below and above BM_SKIP_DF postings, and phrases whose virtual lists get a skip row."""
    s, model, docs = seg
    df = np.diff(model.term_off)
    rare, common = [int(t) for t in np.nonzero((df > 0) & (df < 256))[0][:4]], [int(t) for t in np.nonzero(df >= 256)[0][:6]]
    assert rare and len(common) >= 2
    qs = [([], [[common[i], common[j]]]) for i in range(len(common)) for j in range(len(common))]
    qs += [([], [[r, c]]) for r in rare for c in common[:2]] + [([], [[c, r]]) for r in rare for c in common[:2]]
    for mode in (M.OR, M.AND):
        check(run(s, qs, 32, mode=mode), model.search(qs, 32, mode=mode))


def test_deletions(seg):
    s, model, docs = seg
    rng = np.random.default_rng(5)
    alive = rng.random(N_DOCS) < 0.7
    bits = np.packbits(np.r_[alive, np.zeros((-N_DOCS) % 64, bool)].astype(np.uint8), bitorder="little").view(np.uint64)
    m2 = PM.PhraseModel(N_DOCS, N_TERMS, model.term_off, model.post_doc, model.post_tf, model.fieldnorm_id, pos=model.pos, alive_bits=bits)
    s.set_alive(bits)
    try:
        qs = queries(docs, 6, 200)
        for mode in (M.OR, M.AND):
            check(run(s, qs, 10, mode=mode, use_tf=False), m2.search(qs, 10, mode=mode, use_tf=False))
    finally:
        s.set_alive(None)


def test_search_after(seg):
    s, model, docs = seg
    qs = queries(docs, 7, 64)
    for q in range(0, 64, 9):
        d, sc = model.ranked(qs[q], M.OR, False)[:2]
        if len(d) < 3:
            continue
        for mode in (1, 2, 3):
            after = (float(sc[1]), mode, int(d[1]))
            check(run(s, [qs[q]], 10, use_tf=False, after=after), model.search([qs[q]], 10, use_tf=False, after=after))


def test_union_statistics_over_segments():
    from nucliadb_b200.segment import TextSegment
    parts = [make_corpus(10 + i, n, N_TERMS) for i, n in enumerate((3000, 5000, 700))]
    idx = [index(p, N_TERMS) for p in parts]
    total_docs = sum(len(p) for p in parts)
    total_tokens = sum(len(d) for p in parts for d in p)
    df = sum(np.diff(i[0]).astype(np.uint64) for i in idx)
    qs = queries(parts[1], 11, 100)
    for p, (term_off, post_doc, post_tf, fn, pos, flat) in zip(parts, idx):
        s = TextSegment.create(len(p), N_TERMS, term_off, post_doc, post_tf, fn)
        s.set_stats(total_docs, total_tokens, df)
        s.set_positions(flat)
        model = PM.PhraseModel(len(p), N_TERMS, term_off, post_doc, post_tf, fn, pos=pos, total_docs=total_docs, total_tokens=total_tokens,
                               doc_freq=df)
        check(run(s, qs, 12, use_tf=False), model.search(qs, 12, use_tf=False))
        s.close()


def test_facets_and_date_order(seg):
    s, model, docs = seg
    keys = sorted({f"l\0{d % 5}".encode() for d in range(5)} | {b"l"})
    doc_off = np.arange(N_DOCS + 1, dtype=np.uint64)
    ords = np.asarray([keys.index(f"l\0{d % 5}".encode()) for d in range(N_DOCS)], np.uint32)
    s.set_facets(keys, doc_off, ords)
    created = (np.arange(N_DOCS, dtype=np.int64) * 7919) % 1000
    s.set_dates(created, created)
    qs = queries(docs, 8, 50)
    got = run(s, qs, 10, use_tf=False, facets=[b"l"])
    want = model.search(qs, 10, use_tf=False)
    check(got[:4], want)
    b_req, b_ord = s.facet_buckets([b"l"])
    for q, query in enumerate(qs):
        matched = model.ranked(query, M.OR, False)[0]
        cnt = np.bincount(np.asarray(matched, np.int64) % 5, minlength=5)
        assert [int(x) for x in got[4][q]] == [int(cnt[int(keys[o].split(b"\0")[1])]) for o in b_ord]
    for mode in (M.OR, M.AND):
        d, dates, counts, total = run(s, qs, 10, mode=mode, order=(0, 0))
        for q, query in enumerate(qs):
            matched = model.ranked(query, mode, True)[0]
            top = sorted(matched, key=lambda x: (-created[x], x))[:10]
            assert int(total[q]) == len(matched) and int(counts[q]) == len(top)
            assert [int(x) for x in d[q][: len(top)]] == [int(x) for x in top]


def test_without_phrases_equal_the_plain_calls(seg):
    s, model, docs = seg
    rng = np.random.default_rng(9)
    qs = [([int(t) for t in rng.integers(0, N_TERMS, int(rng.integers(1, 6)))], []) for _ in range(300)]
    qt = np.asarray([t for q in qs for t in q[0]], np.uint32)
    qo = np.zeros(len(qs) + 1, np.uint32)
    qo[1:] = np.cumsum([len(q[0]) for q in qs])
    keys = sorted({f"l\0{d % 5}".encode() for d in range(5)} | {b"l"})
    s.set_facets(keys, np.arange(N_DOCS + 1, dtype=np.uint64), np.asarray([keys.index(f"l\0{d % 5}".encode()) for d in range(N_DOCS)], np.uint32))
    created = (np.arange(N_DOCS, dtype=np.int64) * 31) % 977
    s.set_dates(created, created)
    for mode in (M.OR, M.AND):
        for use_tf in (False, True):
            check(s.search_phrases(qt, qo, [], 10, mode=mode, use_tf=use_tf), s.search(qt, qo, 10, mode=mode, use_tf=use_tf))
            a, b = s.search_phrases(qt, qo, [], 10, mode=mode, use_tf=use_tf, facets=[b"l"]), s.search_faceted(qt, qo, 10, [b"l"], mode=mode, use_tf=use_tf)
            for x, y in zip(a, b):
                assert np.array_equal(x, y)
        a, b = s.search_phrases(qt, qo, [], 10, mode=mode, order=(1, 1)), s.search_ordered(qt, qo, 10, 1, 1, mode)
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


def test_limits_are_einval(seg):
    from nucliadb_b200._lib import NidxError
    from nucliadb_b200.segment import TextSegment
    s, model, docs = seg
    qt, qo = np.zeros(0, np.uint32), np.asarray([0, 0], np.uint32)
    for ph in ([(0, [3])], [(0, list(range(65)))], [(1, [3, 4])], [(0, [1, 2])] * 129):
        with pytest.raises(NidxError) as e:
            s.search_phrases(qt, qo, ph, 10)
        assert e.value.code == -1
    qt2, qo2 = np.arange(127, dtype=np.uint32), np.asarray([0, 127], np.uint32)
    s.search_phrases(qt2, qo2, [(0, [1, 2])], 10)   # 128 clauses: accepted
    with pytest.raises(NidxError):
        s.search_phrases(qt2, qo2, [(0, [1, 2])] * 2, 10)
    t = TextSegment.create(2, 2, np.asarray([0, 1, 2], np.uint64), np.asarray([0, 1], np.uint32), np.asarray([1, 1], np.uint32), np.asarray([1, 1], np.uint8))
    with pytest.raises(NidxError):   # no positions yet
        t.search_phrases(qt, qo, [(0, [0, 1])], 1)
    with pytest.raises(NidxError):   # a count that does not add up
        t.set_positions(np.asarray([0], np.uint32))
    t.set_positions(np.asarray([0, 1], np.uint32))
    t.close()


TRICKY = ["That's a too *tricky* resource", "It's very important to do-stuff", "It's not that important to do-stuff",
          "W'h'a't a -w-e-i-r-d p\"ara\"gra\"ph"]   # nidx_paragraph/tests/reader.rs:71-90, one paragraph each


@pytest.mark.parametrize("body,total", [('"It\'s very important to do-stuff"', 1), ("important", 2), ('"important to do"', 2),
                                        ('"very important" tricky', 2), ("ara", 1), ("paragraph", 0)])
def test_reference_known_answers(body, total):
    """nidx_paragraph/tests/reader.rs:452-490 test_query_parsing_weird_stuff (the fuzzy-only cases are not restated)."""
    from nucliadb_b200.text import DocumentSearchRequest, ParagraphSearcher, TextDoc
    ps = ParagraphSearcher.open([[TextDoc(f"r{i}", "f", t) for i, t in enumerate(TRICKY)]])
    assert ps.search(DocumentSearchRequest(body=body)).total == total

