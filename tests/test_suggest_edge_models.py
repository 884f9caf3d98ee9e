"""The corpora of tests/test_gpu_suggest_edges.py, built here and checked without a GPU: each edge of the fuzzy pass that file is
meant to reach is asserted on the corpus itself (per-segment document frequencies around the 1 024-posting chunk, the 64-term words
of the expansions with and without postings, phrase capacity against matched length, the size of the match list, 64 clauses, the
ties), and the host model (tests/suggest_model.py) is run on the same inputs.

Every corpus sets its document frequencies exactly: in a segment, document d holds word w iff d < df(w), plus one filler word, and a
vocabulary segment (segment 0) names every word in its first document, in the order that fixes the term ids."""
from __future__ import annotations

import numpy as np
import pytest

import suggest_model as SM
from nucliadb_b200 import suggest as S
from nucliadb_b200.text import TextDoc

ALPHA = "abcdefghijklmnopqrstuvwxyz"
CHUNK = 1024                     # SG_CHUNK: postings per warp task of the scatter
H100_SMS = 132                   # the scored pass wraps past sms * 8 CTAs * 8 warps * 32 documents; the scatter past sms * 64 warps
FZ, FP, FP2 = "mnopq", "wxyzv", "qrstu"   # a fuzzy literal and two fuzzy-prefix literals; none is in a vocabulary
DFS = (1, 1023, 1024, 1025, 2048, 2049, 5000)
N_EDGE_DOCS = 6000               # documents of segments 1 and 2 of the chunk corpus


def letters(i: int, n: int) -> str:
    return "".join(ALPHA[(i // 26 ** j) % 26] for j in range(n))


def filler(i: int) -> str:
    return "fil" + letters(i, 4)   # within distance 1 of no literal, as a word or as a prefix


def e1(i: int) -> str:
    """The i-th distance-1 substitution of FZ (125 of them)."""
    p, c = divmod(i, 25)
    alts = [a for a in ALPHA if a != FZ[p]]
    return FZ[:p] + alts[c] + FZ[p + 1:]


def e2(i: int) -> str:
    return FP + letters(i, 3)


def e3(i: int) -> str:
    return FP2 + letters(i, 3)


def _docs(seg: int, tokens: list) -> list:
    return [TextDoc(f"{seg:08x}{d:024x}", "/a/title" if d % 2 else "/a/summary", " ".join(t)) for d, t in enumerate(tokens)]


def _layout_docs(order: list, df: dict, n_docs: int, seg: int, extra=None) -> list:
    """Document d of a segment: the words w of `order` with d < df[w] in id order, then extra(d)'s tokens, then one filler."""
    toks = []
    for d in range(n_docs):
        t = [w for w in order if d < df.get(w, 0)]
        if extra is not None:
            t += extra(d)
        t.append(filler(1000 + d % 97))
        toks.append(t)
    return _docs(seg, toks)


# ---- the chunk corpus: fuzzy, fuzzy-prefix, exact-term and phrase lists across the 1 024-posting chunks ------------------------
N_E2, N_E3 = 320, 320            # fuzzy-prefix expansions of FP and FP2 (each > 300: the match list of 16 hits passes 4 096)
PHRASE_CAP = 2500
PHRASES = {"p1": 700, "p2": CHUNK, "p3": CHUNK + 1, "p4": 0}   # matched length in segment 1 (capacity PHRASE_CAP)
PHRASE_FREQ = 300                # occurrences of the phrase "rra rrb" in document 0 of segment 2 (above the fieldnorm byte)


def chunk_layout():
    """-> (vocabulary order, {word: (df in segment 1, df in segment 2)}) of the chunk corpus.

    Words of 64 term ids (the expansion bitsets' words) of segment 1 / segment 2, for FZ's and FP's expanded terms:
      0: id 63 = FZ (1025 / 0)
      1: id 64 = FZ (1024 / 1), id 126 = FZ (1 / 5000), id 127 = FP (2049 / 0)
      2: id 128 = FP (2048 / 1023), id 129 = FZ (1023 / 0)
      3: FZ and FP terms found in segment 2 only (1024, 2049, 1, 1025): no chunk of either clause in segment 1
      4: FP (5000 / 0), FZ (2048 / 0), FP (1 / 0), FZ (5000 / 2048)
      5: fillers only: no chunk of either clause in either segment
      6: FZ (2049 / 1025), FP (1024 / 2048), FP (1025 / 0), FP (1023 / 5000)
    then the exact terms and the phrase words, then the rest of FZ's, FP's and FP2's expansions (segment 0 only: more words without
    chunks in segments 1 and 2)."""
    slots: dict = {63: (e1(0), 1025, 0), 64: (e1(1), 1024, 1), 126: (e1(2), 1, 5000), 127: (e2(0), 2049, 0), 128: (e2(1), 2048, 1023),
                   129: (e1(3), 1023, 0), 192: (e1(4), 0, 1024), 200: (e2(2), 0, 2049), 240: (e1(5), 0, 1), 255: (e2(3), 0, 1025),
                   256: (e2(4), 5000, 0), 270: (e1(6), 2048, 0), 300: (e2(5), 1, 0), 319: (e1(7), 5000, 2048),
                   384: (e1(8), 2049, 1025), 400: (e2(6), 1024, 2048), 420: (e2(8), 1025, 0), 447: (e2(7), 1023, 5000)}
    order, df = [], {}
    for i in range(448):
        if i in slots:
            w, a, b = slots[i]
        else:
            w, a, b = filler(i), 0, 0
        order.append(w)
        df[w] = (a, b)
    for w, a, b in (("tmaaa", 1024, 0), ("tmaab", 1025, 3000), ("tmaac", 3000, 1024)):
        order.append(w)
        df[w] = (a, b)
    for p in PHRASES:
        for w in (p + "a", p + "b"):
            order.append(w)
            df[w] = (PHRASE_CAP, PHRASE_CAP)
    order += ["rra", "rrb"]
    df["rra"] = df["rrb"] = (0, 1)
    order += [e1(i) for i in range(9, 40)] + [e2(i) for i in range(9, N_E2)] + [e3(i) for i in range(N_E3)]
    return order, df


def chunk_corpus():
    """-> (segments of TextDoc, alive per segment, vocabulary order).  Segment 0: 20 documents, the first holding every word in id
    order and the first 16 every expansion of FP and FP2; segments 1 and 2: N_EDGE_DOCS documents each on chunk_layout's dfs, the
    phrase pairs adjacent ("pNa pNb") in the first PHRASES[pN] documents of segment 1 (every document of segment 2 below the capacity)
    and reversed below the capacity after that, and "rra rrb" PHRASE_FREQ times in document 0 of segment 2."""
    order, df = chunk_layout()
    fp_all = [e2(i) for i in range(N_E2)] + [e3(i) for i in range(N_E3)]
    seg0 = [list(order)] + [list(fp_all) for _ in range(15)] + [[filler(2000 + d)] for d in range(4)]
    plain = [w for w in order if w[:2] not in ("p1", "p2", "p3", "p4", "rr")]

    def phrase_tokens(seg):
        def extra(d):
            t = []
            for p, m in PHRASES.items():
                if d < (m if seg == 1 else PHRASE_CAP):
                    t += [p + "a", p + "b", "sep"]
                elif d < PHRASE_CAP:
                    t += [p + "b", p + "a", "sep"]
            if seg == 2 and d == 0:
                t += ["rra", "rrb"] * PHRASE_FREQ
            return t
        return extra

    segs = [_docs(0, seg0)]
    for s in (1, 2):
        segs.append(_layout_docs(plain, {w: df.get(w, (0, 0))[s - 1] for w in plain}, N_EDGE_DOCS, s, phrase_tokens(s)))
    rng = np.random.default_rng(41)
    alive = [np.ones(len(segs[0]), dtype=bool)] + [rng.random(N_EDGE_DOCS) < 0.95 for _ in (1, 2)]
    return segs, alive, order


def clause_layouts():
    """Fuzzy-pass clause lists (suggest.fuzzy_clauses' format) over the chunk corpus: fuzzy clauses between TERM(NIL), TERMs absent
    from a segment and multi-chunk TERM / PHRASE clauses in several orders, a pass of exactly 64 clauses (8 fuzzy, the last 8), and
    passes in which no clause owns a task in segments 1 and 2."""
    fz, fp, fp2 = (S.FUZZY, FZ), (S.FUZZY_PREFIX, FP), (S.FUZZY_PREFIX, FP2)
    nil, t1024, t1025, t3000 = (S.TERM, "zzqqz"), (S.TERM, "tmaaa"), (S.TERM, "tmaab"), (S.TERM, "tmaac")
    ph = {p: (S.PHRASE, [p + "a", p + "b"]) for p in PHRASES}
    ph_freq = (S.PHRASE, ["rra", "rrb"])
    ph_nil = (S.PHRASE, ["p1a", "zzqqz"])
    layouts = [
        [fz, fp],
        [t1024, t1025, t3000],
        [ph["p1"], ph["p2"], ph["p3"], ph["p4"]],
        [ph_freq, fz],
        [nil, fz, t1024, fp, ph["p3"], nil],
        [ph["p2"], nil, fp, t3000, fz, t1024],
        [fz, ph["p4"], t1025, nil, fp, ph["p1"], t1024],
        [t1024, t1024, fz, fz, ph["p3"], fp, t3000],
    ]
    others = [nil, t1024, t1025, t3000, ph["p1"], ph["p2"], ph["p3"], ph["p4"], ph_freq, ph_nil]
    fuzzy8 = [fz, fp, fp2, (S.FUZZY, "mnopr"), (S.FUZZY, e1(0)), (S.FUZZY_PREFIX, e2(1)), (S.FUZZY, "tmaab"), (S.FUZZY_PREFIX, "wxyzw")]
    layouts.append([others[i % len(others)] for i in range(56)] + fuzzy8)
    layouts.append([(S.FUZZY, "zzzzz"), nil, ph_nil, (S.TERM, "rra")])   # no task in segment 1 (and an empty expansion)
    layouts.append([nil, ph_nil, nil])
    return layouts


# ---- document space: segments of 1 .. 4 097 documents, and one above the scored pass's grid ------------------------------------
SPACE_SIZES = (1, 31, 32, 33, 63, 64, 65, 4097)
SP = "sgfxk"    # the space corpora's fuzzy-prefix literal


def space_corpus():
    """Segments of SPACE_SIZES documents: document d holds an expansion of SP (each of 40 used by many documents), every third a
    second word "wordb" and every fifth "wordc"; alive drops every seventh document."""
    segs = []
    for s, n in enumerate(SPACE_SIZES):
        toks = [[SP + letters(d % 40, 2)] + (["wordb"] if d % 3 == 0 else []) + (["wordc"] if d % 5 == 0 else []) + [filler(d % 13)]
                for d in range(n)]
        segs.append(_docs(s, toks))
    alive = [np.arange(n) % 7 != 3 for n in SPACE_SIZES]
    return segs, alive


BIG_DOCS = 300_000
BIG_TERMS = 10_000
BIG = "tiepq"


def big_corpus():
    """One segment of BIG_DOCS documents, each holding one of BIG_TERMS expansions of BIG (30 postings each: one chunk, so more
    chunks than the scatter's warps) and every 101st "boost"; a vocabulary segment of one document names the words first."""
    words = [BIG + letters(i, 3) for i in range(BIG_TERMS)]
    seg0 = [words + ["boost"]]
    toks = [[words[d % BIG_TERMS]] + (["boost"] if d % 101 == 0 else []) for d in range(BIG_DOCS)]
    alive = [np.ones(1, dtype=bool), np.arange(BIG_DOCS) % 9 != 4]
    return [_docs(0, seg0), _docs(1, toks)], alive, words


def big_fuzzy_pass(model, masks, with_boost: bool, k: int):
    """The big corpus's fuzzy pass [(FUZZY_PREFIX, BIG)] (+ [(TERM, "boost")]) restated with numpy, by the model's rule (its
    per-document loop is slow at this size): every document matches BIG's clause (1.0, every word is one of its expansions); "boost"
    adds w * f32(1 / (1 + norm)) in clause order; the score is 0.5 times the sum.  -> the best k [(score, segment, doc)]."""
    import bm25_model as M

    f = np.float32
    w = f(M.term_weight(model.df[model.vocab["boost"]], model.total_docs))
    t = model.vocab["boost"]
    keys = []
    for o, (m, mask) in enumerate(zip(model.models, masks)):
        s = np.full(m.n_docs, f(1.0), dtype=np.float32)
        if with_boost:
            has = np.zeros(m.n_docs, dtype=bool)
            has[m.post_doc[m.term_off[t]:m.term_off[t + 1]]] = True
            v = (w * (f(1.0) / (f(1.0) + model.norm[m.fieldnorm_id]).astype(np.float32))).astype(np.float32)
            s = np.where(has, (s + v).astype(np.float32), s)
        s = (f(0.5) * s).astype(np.float32)
        d = np.nonzero(np.asarray(mask, dtype=bool))[0]
        keys.append((s[d], np.full(len(d), o), d))
    s, o, d = (np.concatenate(x) for x in zip(*keys))
    best = np.lexsort((d, o, -s))[:k]
    return [(float(s[i]), int(o[i]), int(d[i])) for i in best]


# ---- the expansion at its limits ------------------------------------------------------------------------------------------------
def expansion_literals():
    """64 literals (term, distance, prefix) of exactly 4 096 code points in all: 56 short ones around the chunk corpus's words at
    distances 0 - 2 with and without prefix, then 8 long ones that take the rest."""
    short = [FZ, FP, FP2, e1(0), e2(1), "tmaab", "p1a", "fila", "mnop", "wxyz", "qrst", "zzzz"]
    out = []
    for i in range(56):
        out.append((short[i % len(short)], i % 3, (i // 3) % 2 == 1))
    used = sum(len(t) for t, _, _ in out)
    rest = 4096 - used
    for i in range(8):
        n = rest // 8 + (1 if i < rest % 8 else 0)
        out.append(((FP + "b" * n)[:n], 1, i % 2 == 0))
    return out


def expected_expansion(vocab_terms, term, d, prefix):
    """graph_model.fuzzy_match over the vocabulary, skipping the entries whose length alone rules them out (the DP of a long term
    is slow): |len(entry) - len(term)| > d cannot match, nor (prefix) an entry shorter than the term less d."""
    import graph_model as GM

    m = len(term)
    out = set()
    for e in vocab_terms:
        if len(e) + d < m or (not prefix and len(e) > m + d):
            continue
        if GM.fuzzy_match(term, e, d, prefix):
            out.add(e)
    return out


# ---- the checks --------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def chunk():
    segs, alive, order = chunk_corpus()
    return segs, alive, order, SM.SuggestModel(segs)


def _seg_df(model, seg, word):
    m = model.models[seg]
    t = model.vocab[word]
    return int(m.term_off[t + 1] - m.term_off[t])


def test_chunk_corpus_reaches_the_chunk_edges(chunk):
    segs, alive, order, model = chunk
    assert [model.vocab[w] for w in order] == list(range(len(order)))   # the vocabulary segment fixed the ids
    _, df = chunk_layout()
    for w, (a, b) in df.items():
        assert (_seg_df(model, 1, w), _seg_df(model, 2, w)) == (a, b), w
    for lit, prefix in ((FZ, False), (FP, True)):
        exp = model.expansion(lit, prefix)
        assert lit not in model.vocab
        assert set(DFS) <= {_seg_df(model, 1, w) for w in exp}, lit   # every df of the list, in segment 1 alone
        ids = sorted(model.vocab[w] for w in exp)
        words = sorted({i // 64 for i in ids})
        chunks = [[sum(-(-_seg_df(model, s, w) // CHUNK) for w in exp if model.vocab[w] // 64 == j) for j in range(words[-1] + 1)] for s in (1, 2)]
        # a word with expanded terms but no chunk in segment 1 lies between words with chunks
        empty = [j for j in words if chunks[0][j] == 0]
        assert any(any(chunks[0][i] for i in range(j)) and any(chunks[0][i] for i in range(j + 1, len(chunks[0]))) for j in empty), chunks[0]
        assert sum(chunks[0]) > len([w for w in exp if _seg_df(model, 1, w)])   # some term takes several chunks
    fz_ids = {model.vocab[w] for w in model.expansion(FZ, False)}
    fp_ids = {model.vocab[w] for w in model.expansion(FP, True)}
    assert {63, 64} <= fz_ids and {127, 128} <= fp_ids   # the expansions straddle the 64-term word boundaries
    # documents 4 096 and up of segment 1 are reached only by the partial fifth chunk of a 5 000-posting list
    late = [np.zeros(len(alive[0]), bool), alive[1] & (np.arange(len(alive[1])) >= 4 * CHUNK), np.zeros(len(alive[2]), bool)]
    for lit, kind in ((FZ, S.FUZZY), (FP, S.FUZZY_PREFIX)):
        exp = model.expansion(lit, kind == S.FUZZY_PREFIX)
        assert max(_seg_df(model, 1, w) for w in exp) == 5000
        hits, _ = model.fuzzy_pass([(kind, lit)], 1024, late)
        assert len(hits) == int(late[1][: 5000].sum()) > 800


def test_chunk_corpus_terms_and_phrases(chunk):
    segs, alive, order, model = chunk
    assert [_seg_df(model, 1, w) for w in ("tmaaa", "tmaab", "tmaac")] == [1024, 1025, 3000]
    assert [_seg_df(model, 2, w) for w in ("tmaaa", "tmaab", "tmaac")] == [0, 3000, 1024]
    for p, m in PHRASES.items():
        ph = [model.vocab[p + "a"], model.vocab[p + "b"]]
        for s, want in ((1, m), (2, PHRASE_CAP)):
            d, f = model.models[s].phrase_postings(ph)
            cap = min(_seg_df(model, s, p + "a"), _seg_df(model, s, p + "b"))
            assert cap == PHRASE_CAP and len(d) == want, (p, s)
            assert cap > CHUNK
    d, f = model.models[2].phrase_postings([model.vocab["rra"], model.vocab["rrb"]])
    assert list(d) == [0] and int(f[0]) == PHRASE_FREQ > 255


def test_chunk_corpus_clause_layouts_on_the_model(chunk):
    segs, alive, order, model = chunk
    layouts = clause_layouts()
    assert len(layouts[8]) == 64 and sum(k in (S.FUZZY, S.FUZZY_PREFIX) for k, _ in layouts[8]) == 8
    assert [k in (S.FUZZY, S.FUZZY_PREFIX) for k, _ in layouts[8]][56:] == [True] * 8
    # the last two layouts own no task in segment 1: TERM(NIL), an absent TERM, a phrase of an unknown word, an empty expansion
    assert not model.expansion("zzzzz", False) and _seg_df(model, 1, "rra") == 0 and "zzqqz" not in model.vocab
    hits_seen = 0
    for clauses in layouts:
        hits, matches = model.fuzzy_pass(clauses, 1024, alive)
        hits_seen += bool(hits)
        assert all(s > 0 for s, _, _ in hits)
    assert hits_seen >= 9
    hits, _ = model.fuzzy_pass(layouts[-1], 10, alive)
    assert hits == []


def test_chunk_corpus_match_list_passes_4096(chunk):
    segs, alive, order, model = chunk
    e2s, e3s = model.expansion(FP, True), model.expansion(FP2, True)
    assert len(e2s) >= 300 and len(e3s) >= 300
    toks = model.toks[0]
    triples = sum(len({t for _, t in toks[d]} & e2s) + len({t for _, t in toks[d]} & e3s) for d in range(16))
    assert triples > 4096
    hits, _ = model.fuzzy_pass([(S.FUZZY_PREFIX, FP), (S.FUZZY_PREFIX, FP2)], 16, [alive[0], alive[1] & False, alive[2] & False])
    assert [d for _, _, d in hits] == list(range(16)) and {s for s, _, _ in hits} == {1.0}


def test_space_corpus_sizes_and_ties():
    segs, alive = space_corpus()
    assert [len(s) for s in segs] == list(SPACE_SIZES)
    model = SM.SuggestModel(segs)
    hits, _ = model.fuzzy_pass([(S.FUZZY_PREFIX, SP)], 1 << 20, alive)
    # every alive document ties at 0.5; the 4 097-document segment takes two top-k CTAs, and its last document is alive
    assert {s for s, _, _ in hits} == {0.5} and len(hits) == sum(int(a.sum()) for a in alive) > 1024
    assert len(segs[-1]) > 4096 and alive[-1][4096]
    hits, _ = model.fuzzy_pass([(S.FUZZY_PREFIX, SP), (S.TERM, "wordb"), (S.TERM, "wordc")], 1 << 20, alive)
    assert len({s for s, _, _ in hits}) >= 4   # 0.5 alone, with wordb, with wordc, with both


def test_big_corpus_passes_the_grids():
    segs, alive, words = big_corpus()
    assert BIG_DOCS > H100_SMS * 8 * 8 * 32                       # the scored pass's grid-stride loop wraps
    assert BIG_TERMS > H100_SMS * 64                               # one chunk per expanded term: the scatter's loop wraps
    assert int(alive[1].sum()) > 4096                             # ties at 0.5 over many top-k CTAs
    model = SM.SuggestModel([segs[0], segs[1][:3000]])             # the numpy restatement against the model's loop, on a slice
    a = [alive[0], alive[1][:3000]]
    for boost in (False, True):
        clauses = [(S.FUZZY_PREFIX, BIG)] + ([(S.TERM, "boost")] if boost else [])
        want, _ = model.fuzzy_pass(clauses, 1024, a)
        got = big_fuzzy_pass(model, a, boost, 1024)
        assert [(o, d) for _, o, d in got] == [(o, d) for _, o, d in want]
        assert np.array_equal(np.float32([s for s, _, _ in got]).view(np.uint32), np.float32([s for s, _, _ in want]).view(np.uint32))


def test_expansion_literals_fill_the_automaton():
    lits = expansion_literals()
    assert len(lits) == 64 and sum(len(t) for t, _, _ in lits) == 4096
    assert {d for _, d, _ in lits} == {0, 1, 2} and {p for _, _, p in lits} == {False, True}
