"""Exact phrases on the host side: nidx_paragraph's query grammar against the reference's own test expectations
(tests/golden/paragraph_grammar.json), the phrase semantics against an independent scan of token sequences, and the kernel's
fixed-point model with phrase clauses (tests/phrase_model.py) against float64 within bm25_model's error bound."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import bm25_model as M
import phrase_model as PM
from nucliadb_b200.text import paragraph_query_tokens, parse_paragraph_query, tokenize, tokenize_with_positions

HERE = os.path.dirname(os.path.abspath(__file__))
CASES = json.load(open(os.path.join(HERE, "golden", "paragraph_grammar.json"), encoding="utf-8"))["cases"]


@pytest.mark.parametrize("case", CASES, ids=[c["source"].split("/")[-1] for c in CASES])
def test_grammar_matches_the_reference(case):
    assert [list(t) for t in paragraph_query_tokens(case["query"])] == case["tokens"]
    words, phrases = parse_paragraph_query(case["query"])
    assert {"words": words, "phrases": phrases} == case["clauses"]


@pytest.mark.parametrize("body", ["rag database", '"rag" database', 'a "unclosed quote', 'x "" y "z"', "-minus word", "Hello, WORLD!",
                                  'one "two three"', "x" * 45 + ' "' + "y" * 41 + '" z'])
def test_literals_stay_as_today(body):
    """A body without a closed quote around two or more words yields tokenize()'s term list, long words dropped as before."""
    words, phrases = parse_paragraph_query(body)
    assert phrases == [] and words == tokenize(body)


def test_positions_keep_the_gap_of_a_dropped_word():
    text = "alpha " + "b" * 40 + " gamma delta"
    assert tokenize_with_positions(text) == [(0, "alpha"), (2, "gamma"), (3, "delta")]
    assert [t for _, t in tokenize_with_positions(text)] == tokenize(text)


def scan_freq(tokens, phrase):
    """Independent restatement: count the start positions s with tokens[s + i] == phrase[i] for every i (tokens: position -> term)."""
    return sum(all(tokens.get(s + i) == t for i, t in enumerate(phrase)) for s in range(max(tokens, default=-1) + 1))


@pytest.mark.parametrize("seq,phrase,want", [("a a a", "a a", 2), ("a b a b a b", "a b a", 2), ("a b _ c", "b c", 0), ("a b c", "c b", 0),
                                              ("x a b a b", "a b", 2), ("a a a a", "a a a", 2)])
def test_phrase_frequency(seq, phrase, want):
    toks = {i: w for i, w in enumerate(seq.split()) if w != "_"}   # "_": a dropped word (a gap)
    pos = {}
    for p, w in toks.items():
        pos.setdefault(w, []).append(p)
    lists = [pos.get(w, []) for w in phrase.split()]
    assert PM.phrase_freq(lists) == scan_freq(toks, phrase.split()) == want


def small_corpus(seed, n_docs=400, vocab=12):
    rng = np.random.default_rng(seed)
    docs = []
    for _ in range(n_docs):
        n = int(rng.integers(2, 16))
        pos, toks = 0, []
        for t in rng.integers(0, vocab, n):
            pos += 1 if rng.random() < 0.1 else 0
            toks.append((pos, int(t)))
            pos += 1
        docs.append(toks)
    return docs


def build(docs, vocab, **kw):
    from nucliadb_b200.text import fieldnorm_to_id
    pos = PM.token_positions(docs)
    pairs = sorted(pos)
    term_off = np.zeros(vocab + 1, np.uint64)
    term_off[1:] = np.cumsum(np.bincount([t for t, _ in pairs], minlength=vocab))
    post_doc = np.asarray([d for _, d in pairs], np.uint32)
    post_tf = np.asarray([len(pos[p]) for p in pairs], np.uint32)
    fn = np.asarray([fieldnorm_to_id(len(t)) for t in docs], np.uint8)
    return PM.PhraseModel(len(docs), vocab, term_off, post_doc, post_tf, fn, pos=pos, **kw)


def test_phrase_matches_equal_the_token_scan():
    docs = small_corpus(1)
    m = build(docs, 12)
    for phrase in ([0, 1], [3, 3], [2, 5, 2], [1, 1, 1], [4, 7, 9, 4]):
        d, f = m.phrase_postings(phrase)
        want = {i: scan_freq(dict(t), phrase) for i, t in enumerate((((p, w) for p, w in doc) for doc in docs))}
        assert dict(zip(d.tolist(), f.tolist())) == {i: x for i, x in want.items() if x}


def test_phrase_weight_sums_idf_in_order_with_repeats_and_union_statistics():
    docs = small_corpus(2)
    df = np.full(12, 300, np.int64)
    df[3] = 7
    m = build(docs, 12, total_docs=5000, total_tokens=40000, doc_freq=df)
    idf = [np.float32(M.O.bm25_idf(int(df[t]), 5000)) for t in (3, 1, 3)]
    s = np.float32(np.float32(idf[0] + idf[1]) + idf[2])
    assert m.phrase_weight([3, 1, 3]) == np.float32(s * np.float32(1 + M.K1))
    assert m.phrase_weight([3, 12]) == 0.0   # a word the dictionary lacks


@pytest.mark.parametrize("mode,use_tf", [(M.OR, False), (M.OR, True), (M.AND, True)])
def test_model_within_its_bound_of_float64(mode, use_tf):
    """Fixed-point scores with phrase clauses against the float64 sum of the clauses' real-valued scores (bm25_model.error_bound)."""
    docs = small_corpus(3)
    m = build(docs, 12)
    rng = np.random.default_rng(4)
    for _ in range(40):
        terms = [int(t) for t in rng.integers(0, 14, int(rng.integers(0, 3)))]
        phrases = [[int(t) for t in rng.integers(0, 12, int(rng.integers(2, 4)))] for _ in range(int(rng.integers(1, 3)))]
        d, score, sums, csum, npost, s = m.ranked((terms, phrases), mode, use_tf)
        exact = np.zeros(len(d))
        w = m.weights(terms) + [m.phrase_weight(p) for p in phrases]
        for i, doc in enumerate(d):
            nc = m.norm[m.fieldnorm_id[doc]].astype(np.float64)
            for t, wt in zip(terms, w):
                if t < 12 and (t, int(doc)) in m.pos:
                    tf = 1 if not use_tf else len(m.pos[(t, int(doc))])
                    exact[i] += float(wt) * tf / (tf + nc)
            for p, wt in zip(phrases, w[len(terms):]):
                f = PM.phrase_freq([m.pos.get((t, int(doc)), []) for t in p])
                if f:
                    exact[i] += float(wt) * f / (f + nc)
        assert np.allclose(csum, exact, rtol=1e-12, atol=0)
        assert (np.abs(score - exact) <= M.error_bound(score, csum, npost, s)).all()


def test_phrases_struct_has_the_header_layout(tmp_path):
    import os
    import subprocess

    from nucliadb_b200 import _lib as L
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "l.c"
    src.write_text(f'#include <stdio.h>\n#include <stddef.h>\n#include "{root}/include/nidx_b200.h"\nint main(void) {{ printf("%zu %zu %zu %zu %zu", '
                   "sizeof(nidx_txt_phrases), offsetof(nidx_txt_phrases, terms), offsetof(nidx_txt_phrases, off), offsetof(nidx_txt_phrases, query), "
                   "offsetof(nidx_txt_phrases, n)); return 0; }\n")
    subprocess.run(["gcc", "-o", str(tmp_path / "l"), str(src)], check=True)
    got = [int(x) for x in subprocess.run([str(tmp_path / "l")], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(L.TxtPhrases)] + [getattr(L.TxtPhrases, f).offset for f, _ in L.TxtPhrases._fields_]
