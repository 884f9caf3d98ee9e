"""Suggest's fuzzy pass (suggest.cuh through nidx_txt_suggest_fuzzy, TextSegment.suggest_fuzzy and ParagraphSearcher.suggest) against
the host model (tests/suggest_model.py), bit for bit, on the corpora of tests/test_suggest_edge_models.py, which also shows that each
edge is reached: expanded, exact and phrase lists over several 1 024-posting chunks with expansions that straddle 64-term words and
leave words without chunks, clause layouts up to 64 clauses, the match list at 0 / 1 / 10 / 16 hits and past its 4 096-entry first
capacity, segments of 1 to 4 097 documents with and without alive bits, and a segment past the scored pass's and the scatter's grids
with its ties over many top-k CTAs; then the expansion at 64 literals of 4 096 code points."""
import numpy as np
import pytest

import suggest_model as SM
import test_suggest_edge_models as E
from nucliadb_b200 import _lib
from nucliadb_b200 import suggest as S
from nucliadb_b200.text import ParagraphSearcher
from test_gpu_suggest import check, host_bits, open_searcher

pytestmark = pytest.mark.gpu


def sm_count():
    import torch

    return torch.cuda.get_device_properties(0).multi_processor_count


def close(ps):
    for s in ps.segments:
        s._gpu.close()
    if ps._suggest_dict is not None:
        ps._suggest_dict.close()


def fuzzy(ps, clauses, k, masks):
    views = [s._gpu.view(m) for s, m in zip(ps.segments, masks)]
    try:
        return ps._suggest_fuzzy(clauses, k, views)
    finally:
        for v in views:
            v.close()


def same_hits(got, hits, what):
    assert [(h.segment, h.doc) for h in got] == [(o, d) for _, o, d in hits], what
    assert np.array_equal(np.asarray([h.score for h in got], np.float32).view(np.uint32),
                          np.asarray([s for s, _, _ in hits], np.float32).view(np.uint32)), what


def check_fuzzy(ps, model, clauses, k, masks, mm):
    got = fuzzy(ps, clauses, k, masks)
    hits, matches = model.fuzzy_pass(clauses, k, mm)
    same_hits(got, hits, clauses)
    for h in got[: S.RESULTS_PER_PAGE]:
        assert h.matches == matches[(h.segment, h.doc)], clauses
    return got


def device_spec(ps, clauses):
    """_suggest_fuzzy's translation of clauses for nidx_txt_suggest_fuzzy -> (spec, expansion bitsets, rows, phrases)."""
    if ps._suggest_dict is None:   # the vocabulary goes to the device on the first fuzzy pass
        fuzzy(ps, [(S.FUZZY, "zzqqz")], 1, ps.suggest_masks())
    auto = [(v, S.FUZZY_DISTANCE, kind == S.FUZZY_PREFIX) for kind, v in clauses if kind in (S.FUZZY, S.FUZZY_PREFIX)]
    bits = ps._suggest_dict.expand(auto)[0] if auto else None
    spec, phrases, row = [], [], 0
    for kind, v in clauses:
        if kind in (S.FUZZY, S.FUZZY_PREFIX):
            spec.append((_lib.NIDX_SG_FUZZY, row))
            row += 1
        elif kind == S.TERM:
            spec.append((_lib.NIDX_SG_TERM, ps.vocab.get(v, _lib.NIL)))
        else:
            spec.append((_lib.NIDX_SG_PHRASE, len(phrases)))
            phrases.append([ps.vocab.get(t, 0xFFFFFFF0) for t in v])
    if phrases:
        ps._ensure_positions()
    return spec, bits, len(auto), phrases


def segment_hits(model, clauses, k, mm, o):
    """The model's best k of segment o alone (a direct call on one segment)."""
    hits, _ = model.fuzzy_pass(clauses, 1 << 30, [m if i == o else np.zeros_like(m) for i, m in enumerate(mm)])
    return hits[:k]


def want_triples(model, clauses, exps, o, ids, n):
    """(hit, clause, term id) of every expanded term of every fuzzy clause found in each of the first n hits, sorted."""
    out = []
    for h in range(n):
        words = {t for _, t in model.toks[o][int(ids[h])]}
        for c, e in enumerate(exps):
            if e is not None:
                out += [(h, c, model.vocab[t]) for t in e & words]
    return sorted(out)


@pytest.fixture(scope="module")
def chunk_shard():
    segs, alive, order = E.chunk_corpus()
    ps = open_searcher(segs, alive)
    model = SM.SuggestModel(segs)
    assert [model.vocab[w] for w in order] == [ps.vocab[w] for w in order] == list(range(len(order)))
    yield segs, alive, ps, model
    close(ps)


def test_chunked_expansions_through_suggest_and_the_fuzzy_pass(chunk_shard):
    """The expanded terms of a fuzzy and a fuzzy-prefix literal at dfs of 1 .. 5 000 per segment, in words 63/64 and 127/128 and
    with words of no chunk between: through suggest (the literals miss the keyword pass) and _suggest_fuzzy."""
    segs, alive, ps, model = chunk_shard
    masks = ps.suggest_masks()
    mm = [a & host_bits(m, len(a)) for a, m in zip(alive, masks)]
    for body in (f"{E.FZ} {E.FP}", f"{E.FP} {E.FZ}", E.FP, f"{E.FZ} zzqqz {E.FP}"):
        for k in (1, 10, 1024):
            got = check(ps, model, alive, body, k, masks)
            assert got.fuzzy and got.hits, body
    for clauses in ([(S.FUZZY, E.FZ)], [(S.FUZZY_PREFIX, E.FP)], [(S.FUZZY, E.FZ), (S.FUZZY_PREFIX, E.FP)],
                    [(S.FUZZY_PREFIX, E.FP), (S.FUZZY, E.FZ), (S.FUZZY_PREFIX, E.FP2)]):
        for k in (1, 20, 1024):
            check_fuzzy(ps, model, clauses, k, masks, mm)
    # segment by segment, so that each segment's own layout decides the hits
    clauses = [(S.FUZZY, E.FZ), (S.FUZZY_PREFIX, E.FP)]
    for o in (1, 2):
        only = [m if i == o else m * 0 for i, m in enumerate(masks)]
        for k in (1, 1024):
            check_fuzzy(ps, model, clauses, k, only, [a & host_bits(m, len(a)) for a, m in zip(alive, only)])
    # windows of documents that only a term's later chunks reach: document d holds every word of df > d, so the best k of the whole
    # segment come from first chunks; past 1 023, 2 047 and 4 095 only chunks 1, 2 and the partial chunk 4 of a list hold them
    for lo in (1023, 1024, 2048, 4096):
        win = [pack(np.arange(len(a)) >= lo) for a in alive]
        wm = [a & host_bits(m, len(a)) for a, m in zip(alive, win)]
        for cl in ([(S.FUZZY, E.FZ)], [(S.FUZZY_PREFIX, E.FP)], clauses):
            for k in (1, 1024):
                check_fuzzy(ps, model, cl, k, win, wm)


def pack(bits_bool):
    """bool per document -> uint64 words (padding bits zero)."""
    w = np.zeros(max((len(bits_bool) + 63) // 64, 1) * 8, dtype=np.uint8)
    p = np.packbits(np.asarray(bits_bool, dtype=bool), bitorder="little")
    w[: len(p)] = p
    return w.view(np.uint64)


def test_clause_layouts_with_multi_chunk_terms_and_phrases(chunk_shard):
    """TERM at df 1 024 / 1 025 / 3 000, PHRASE at a capacity of 2 500 with 700 / 1 024 / 1 025 / 0 matches and one at frequency 300
    in a document, TERM(NIL), TERMs absent from a segment, in several orders; 64 clauses; passes in which no clause owns a task."""
    segs, alive, ps, model = chunk_shard
    masks = ps.suggest_masks()
    mm = [a & host_bits(m, len(a)) for a, m in zip(alive, masks)]
    layouts = E.clause_layouts()
    assert len(layouts[8]) == _lib.NIDX_SG_MAX_CLAUSES
    for clauses in layouts:
        for k in (1, 20, 1024):
            check_fuzzy(ps, model, clauses, k, masks, mm)
    assert fuzzy(ps, layouts[-1], 10, masks) == []


def test_match_lists_at_every_hit_count_and_past_the_first_capacity(chunk_shard):
    """TextSegment.suggest_fuzzy directly: match_hits 0, 1, 10, 16 and match_cap 0, 5 and 4 096; the triples are the model's expansions
    found in each hit.  16 hits with 640 expanded terms each (> 4 096 triples) re-run with room for the whole list."""
    segs, alive, ps, model = chunk_shard
    masks = ps.suggest_masks()
    mm = [a & host_bits(m, len(a)) for a, m in zip(alive, masks)]
    cases = [[(S.FUZZY, E.FZ), (S.FUZZY_PREFIX, E.FP)], [(S.FUZZY_PREFIX, E.FP), (S.FUZZY_PREFIX, E.FP2)],
             E.clause_layouts()[8]]
    big_seen = False
    for clauses in cases:
        spec, bits, rows, phrases = device_spec(ps, clauses)
        exps = [model.expansion(v, kind == S.FUZZY_PREFIX) if kind in (S.FUZZY, S.FUZZY_PREFIX) else None for kind, v in clauses]
        for o, (s, m) in enumerate(zip(ps.segments, masks)):
            v = s._gpu.view(m)
            try:
                for k in (16, 40):
                    want = segment_hits(model, clauses, k, mm, o)
                    for mh in (0, 1, 10, 16):
                        for cap in (0, 5, 4096):
                            ids, scores, count, trip = v.suggest_fuzzy(spec, bits, rows, len(ps.vocab), phrases, k, mh, cap)
                            assert [(o, int(d)) for d in ids] == [(oo, d) for _, oo, d in want], (clauses, o, k)
                            assert np.array_equal(scores.view(np.uint32), np.asarray([x for x, _, _ in want], np.float32).view(np.uint32))
                            exp = want_triples(model, clauses, exps, o, ids, min(mh, count))
                            assert trip == exp, (o, k, mh, cap)
                            big_seen |= len(trip) > 4096
            finally:
                v.close()
    assert big_seen


@pytest.fixture(scope="module")
def space_shard():
    segs, alive = E.space_corpus()
    ps = open_searcher(segs, alive)
    bare = ParagraphSearcher.open(segs)   # no alive bits: views of raw masks, and direct calls with A.alive == NULL
    yield segs, alive, ps, bare, SM.SuggestModel(segs)
    close(ps)
    close(bare)


def padded(bits_bool, pad_value=True):
    """bool per document -> uint64 words with every padding bit past n_docs = pad_value."""
    n = len(bits_bool)
    w = np.zeros(max((n + 63) // 64, 1) * 64, dtype=bool)
    w[:n] = bits_bool
    w[n:] = pad_value
    return np.packbits(w, bitorder="little").view(np.uint64)


def test_document_space_from_one_to_4097_documents(space_shard):
    segs, alive, ps, bare, model = space_shard
    clauses = [(S.FUZZY_PREFIX, E.SP), (S.TERM, "wordb"), (S.TERM, "wordc")]
    sizes = [len(s) for s in segs]
    assert sizes == list(E.SPACE_SIZES)
    rng = np.random.default_rng(8)
    pf = [rng.random(n) < 0.5 for n in sizes]
    sec = [np.arange(n) % 4 != 1 for n in sizes]
    # the suggest mask from operands whose padding bits are set: its own padding bits are zero
    pmasks = []
    for s, p, q in zip(ps.segments, pf, sec):
        out, matching = s._gpu.suggest_mask(padded(q), padded(p), None)
        n = s.n_docs
        assert np.array_equal(host_bits(out, (n + 63) // 64 * 64)[n:], np.zeros((n + 63) // 64 * 64 - n, bool))
        assert np.array_equal(host_bits(out, n), p & q) and matching == int((p & q).sum())
        pmasks.append(out)
    few = [padded(np.arange(n) % 50 == 7) for n in sizes]   # fewer hits than k = 1 024
    for masks in (ps.suggest_masks(), pmasks, few, [padded(np.ones(n, bool)) for n in sizes]):
        mm = [a & host_bits(m, len(a)) for a, m in zip(alive, masks)]
        for k in (1, 10, 1024):
            got = check(ps, model, alive, E.SP, k, masks)
            assert got.fuzzy
            check_fuzzy(ps, model, clauses, k, masks, mm)
        ones = [np.ones(n, bool) for n in sizes]
        mm = [host_bits(m, n) for m, n in zip(masks, sizes)]
        for k in (1, 1024):
            check(bare, model, ones, E.SP, k, masks)   # views of masks with their padding bits set, no alive bits below
            check_fuzzy(bare, model, clauses, k, masks, mm)
    # the segments themselves, without alive bits (the score kernel reads no alive word)
    spec, bits, rows, phrases = device_spec(bare, clauses)
    for o, s in enumerate(bare.segments):
        for k in (1, 10, 1024):
            ids, scores, count, trip = s._gpu.suggest_fuzzy(spec, bits, rows, len(bare.vocab), phrases, k, min(k, 10))
            want = segment_hits(model, clauses, k, [np.ones(n, bool) for n in sizes], o)
            assert [(o, int(d)) for d in ids] == [(oo, d) for _, oo, d in want]
            assert np.array_equal(scores.view(np.uint32), np.asarray([x for x, _, _ in want], np.float32).view(np.uint32))


def test_segment_past_the_grids_with_ties_over_many_topk_ctas():
    """300 000 documents (the scored pass wraps past sm_count * 8 CTAs of 8 warps of 32 documents), 10 000 expanded terms with
    postings (one chunk each: the scatter wraps past sm_count * 64 warps), every document tied at 0.5; scores restated with numpy."""
    segs, alive, words = E.big_corpus()
    sm = sm_count()
    assert E.BIG_DOCS > sm * 8 * 8 * 32
    ps = open_searcher(segs, alive)
    try:
        model = SM.SuggestModel(segs)
        m1 = model.models[1]
        chunks = sum(-(-int(m1.term_off[model.vocab[w] + 1] - m1.term_off[model.vocab[w]]) // E.CHUNK) for w in words)
        assert chunks > sm * 64   # warp tasks of the scatter in segment 1
        masks = ps.suggest_masks()
        mm = [a & host_bits(m, len(a)) for a, m in zip(alive, masks)]
        word_of = {d: words[d % E.BIG_TERMS] for d in range(E.BIG_DOCS)}
        for k in (1, 10, 1024):
            got = ps.suggest(E.BIG, k, masks)
            want = E.big_fuzzy_pass(model, mm, False, k)
            assert got.fuzzy
            same_hits(got.hits, want, k)
            for h in got.hits[: S.RESULTS_PER_PAGE]:
                assert h.matches == (sorted(words) if h.segment == 0 else [word_of[h.doc]])
            got = fuzzy(ps, [(S.FUZZY_PREFIX, E.BIG), (S.TERM, "boost")], k, masks)
            same_hits(got, E.big_fuzzy_pass(model, mm, True, k), k)
    finally:
        close(ps)


def test_expansion_at_64_literals_and_4096_code_points(chunk_shard):
    segs, alive, ps, model = chunk_shard
    from nucliadb_b200.segment import SuggestDict

    vocab_terms = sorted(ps.vocab, key=ps.vocab.get)
    lits = E.expansion_literals()
    assert len(lits) == 64 and sum(len(t) for t, _, _ in lits) == 4096
    d = SuggestDict(vocab_terms)
    try:
        bits, counts = d.expand(lits)
        rows = bits.cpu().numpy().view(np.uint64)
        for r, (t, dist, prefix) in enumerate(lits):
            want = E.expected_expansion(vocab_terms, t, dist, prefix)
            if dist == 1 and len(t) <= 16:
                assert want == model.expansion(t, prefix), t
            got = {vocab_terms[i] for i in np.nonzero(host_bits(rows[r], len(vocab_terms)))[0]}
            assert got == want and int(counts[r]) == len(want), (r, t, dist, prefix)
    finally:
        d.close()
    masks = ps.suggest_masks()
    got = ps.suggest("a" * 2048 + " " + "b" * 2048, 10, masks)   # 4 096 code points: allowed, within distance 1 of no word
    assert got.fuzzy and got.hits == []
    with pytest.raises(ValueError):
        ps.suggest("a" * 2048 + " " + "b" * 2049, 10, masks)
