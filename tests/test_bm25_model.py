"""The host model of the BM25 kernel's arithmetic (tests/bm25_model.py) against float64 and against the oracle, on the CPU.
The GPU tests (test_gpu_text.py) pin the kernel to the model bit for bit; these pin the model within its stated error bound of the
real-valued BM25 score, so together they bound the kernel's error."""
import numpy as np
import pytest

import bm25_model as M
import oracle as O
from test_oracle_crosscheck import naive_bm25


def small_corpus(seed, n_docs=2500, n_terms=60, max_len=70, big_tf=False):
    rng = np.random.default_rng(seed)
    docs = [list(((rng.zipf(1.3, int(rng.integers(1, max_len))) - 1) % n_terms).astype(int)) for _ in range(n_docs)]
    if big_tf:   # a few documents repeat one term thousands of times (tf far above the length-normalised constant)
        for i in rng.choice(n_docs, 20, replace=False):
            docs[i] = docs[i] + [int(rng.integers(0, n_terms))] * int(rng.integers(500, 5000))
    doc_off = np.concatenate([[0], np.cumsum([len(d) for d in docs])])
    return docs, O.Postings(doc_off, np.concatenate(docs).astype(np.uint32), n_terms)


def check_against_float64(docs, P, model, queries, mode, use_tf, k):
    weights = [model.weight(t) for t in range(P.n_terms)]
    for query in queries:
        d, sc, _, csum, npost, s = model.ranked(query, mode, use_tf)
        want = naive_bm25(docs, P.n_terms, query, mode, use_tf, weights=weights, norm=model.norm)
        S = dict((i, x) for x, i in want)
        assert sorted(d.tolist()) == sorted(S)                              # the matched set is exact
        if not len(d):
            continue
        exact = np.array([S[int(i)] for i in d])
        bound = M.error_bound(sc, csum, npost, s)
        assert (np.abs(sc.astype(np.float64) - exact) <= bound).all()
        # the model's top-k is a float64 top-k up to the bound: no excluded document beats a returned one by more than both bounds
        if len(d) > k:
            floor = np.min(exact[:k] + bound[:k])
            assert (exact[k:] <= floor + bound[k:]).all()


@pytest.mark.parametrize("inflate", [False, True], ids=["own_stats", "shift_below_24"])
def test_model_within_its_bound_of_float64(inflate):
    docs, P = small_corpus(51, big_tf=True)
    kw = {}
    if inflate:   # weights inflated through the statistics: fewer fraction bits, so the 2^-s term of the bound dominates
        kw = dict(total_docs=1 << 50, total_tokens=(P.total_tokens // P.n_docs) << 50, doc_freq=P.doc_freq)
    model = M.Bm25Model.of(P, **kw)
    rng = np.random.default_rng(52)
    queries = [list(rng.choice(P.n_terms, 5, replace=False)) for _ in range(6)]
    queries += [[3, 3, 7], [1, P.n_terms + 5, 2], list(range(P.n_terms)) * 2]   # duplicates, an unknown id, 120 terms
    if inflate:
        assert model.shift(queries[-1]) <= 19
    check_against_float64(docs, P, model, queries, M.OR, True, 10)
    check_against_float64(docs, P, model, queries, M.OR, False, 10)
    check_against_float64(docs, P, model, [q[:2] for q in queries[:6]] + [[4, 4]], M.AND, True, 10)


@pytest.mark.parametrize("mode,use_tf", [(M.OR, False), (M.OR, True), (M.AND, True)])
def test_model_agrees_with_the_oracle(mode, use_tf):
    """Within the model's bound plus the oracle's own f32 error (three roundings per term, a recursive f32 sum of n terms); ids
    wherever the model's neighbours are further apart than that."""
    rng = np.random.default_rng(53)
    n_docs, n_terms = 20000, 3000
    lens = np.maximum(1, rng.lognormal(np.log(40), 0.6, n_docs).astype(np.int64))
    doc_off = np.concatenate([[0], np.cumsum(lens)])
    P = O.Postings(doc_off, ((rng.zipf(1.2, int(doc_off[-1])) - 1) % n_terms).astype(np.uint32), n_terms)
    model = M.Bm25Model.of(P)
    nterms = 3 if mode == M.AND else 12
    queries = [list(rng.choice(400, nterms, replace=False) + (0 if mode == M.AND else 20)) for _ in range(20)]
    k = 100
    od, osc, oc, otot = O.bm25_search(P, queries, k, mode=mode, use_tf=use_tf, nthreads=4)
    md, msc, mc, mtot = model.search(queries, k, mode, use_tf)
    assert (mc == oc).all() and (mtot == otot).all()
    for q, query in enumerate(queries):
        d, sc, _, csum, npost, s = model.ranked(query, mode, use_tf)
        tol = M.error_bound(sc, csum, npost, s) + 3.01 * M.U * csum + npost * 1.01 * M.U * csum
        pos = {int(x): j for j, x in enumerate(d)}
        c = int(oc[q])
        j = np.array([pos[int(x)] for x in od[q, :c]], dtype=np.int64)
        assert (np.abs(osc[q, :c].astype(np.float64) - sc[j]) <= tol[j] + M.error_bound(osc[q, :c], csum[j], npost[j], s)).all()
        for i in range(c):   # the same document wherever the model's neighbours are separated by more than both tolerances
            apart = (i == 0 or sc[i - 1] - sc[i] > tol[i - 1] + tol[i]) and (i + 1 >= len(d) or sc[i] - sc[i + 1] > tol[i] + tol[i + 1])
            if apart:
                assert od[q, i] == d[i]


def test_shift_rule_keeps_the_worst_document_inside_uint32():
    """128 query terms in one document, every one with the largest tf the postings hold and the shortest fieldnorm; weights inflated
    through the statistics (total_docs ~ 2^62) so that the shift drops well below 24.  The exact sum stays below 2^32, and one more
    fraction bit would break the rule's 4e9 limit."""
    n_terms = 130
    term_off = np.arange(n_terms + 1, dtype=np.uint64)                  # term t: one posting, on document 0
    post_doc = np.zeros(n_terms, dtype=np.uint32)
    post_tf = np.full(n_terms, M.TF_MAX, dtype=np.uint32)
    fieldnorm = np.zeros(2, dtype=np.uint8)
    model = M.Bm25Model(2, n_terms, term_off, post_doc, post_tf, fieldnorm, total_docs=(1 << 62) + 12345, total_tokens=1 << 62,
                        doc_freq=np.ones(n_terms, dtype=np.uint64))
    for query in (list(range(128)), [5] * 128, list(range(64)) * 2):
        s = model.shift(query)
        assert s <= 19
        w = model.weights(query)
        assert np.float32(np.float32(len(query)) * max(w)) * np.float32(2.0 ** (s + 1)) >= M.LIMIT   # the largest s that keeps the rule
        d, sc, sums, _, npost, s2 = model.ranked(query, M.OR, True)
        assert s2 == s and d.tolist() == [0] and int(npost[0]) == 128
        assert 2 ** 31 < int(sums[0]) < 2 ** 32
        assert int(sums[0]) == sum(int(np.rint(np.float32(np.float32(x * np.float32(2.0 ** s)) * model_frac(model)))) for x in w)


def model_frac(model):
    tff = np.float32(M.TF_MAX)
    return np.float32(tff / np.float32(tff + model.norm[0]))


def test_tf_above_24_bits_scores_as_the_clamp():
    """bm25_pack_kernel keeps tf in 24 bits: tf = 2^24 + 5 scores exactly as 0xFFFFFF (the reference's tf is u32; DESIGN.md §2)."""
    term_off = np.array([0, 2, 3], dtype=np.uint64)
    post_doc = np.array([0, 1, 2], dtype=np.uint32)
    fieldnorm = np.array([40, 40, 40], dtype=np.uint8)
    stats = dict(total_docs=3, total_tokens=300, doc_freq=np.array([2, 1], dtype=np.uint64))
    big = M.Bm25Model(3, 2, term_off, post_doc, np.array([(1 << 24) + 5, 1, M.TF_MAX], dtype=np.uint32), fieldnorm, **stats)
    d, sc = big.ranked([0, 1], M.OR, True)[:2]
    score = dict(zip(d.tolist(), sc.tolist()))
    clamp = M.Bm25Model(3, 2, term_off, post_doc, np.array([M.TF_MAX, 1, M.TF_MAX], dtype=np.uint32), fieldnorm, **stats)
    d2, sc2 = clamp.ranked([0, 1], M.OR, True)[:2]
    assert dict(zip(d2.tolist(), sc2.tolist())) == score


def test_f32_of_int_rounds_to_nearest_even():
    rng = np.random.default_rng(54)
    for n in [0, 1, (1 << 24) + 1, (1 << 24) + 3, (1 << 62) + 12345, (1 << 64) - 1] + [int(x) for x in rng.integers(0, 1 << 63, 200, dtype=np.int64)]:
        f = M.f32_of_int(n)
        lo, hi = np.nextafter(f, np.float32(0)), np.nextafter(f, np.float32(np.inf))
        err = abs(int(f) - n)
        assert err <= abs(int(lo) - n) and err <= abs(int(hi) - n)
        if err and (err == abs(int(lo) - n) or err == abs(int(hi) - n)):   # a tie goes to the even significand
            assert (int(f) >> (int(f).bit_length() - 24)) % 2 == 0
