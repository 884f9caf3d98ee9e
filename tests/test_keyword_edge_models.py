"""The references of tests/test_gpu_keyword_edges.py, checked on the corpora that file builds, without a GPU: the phrase model's
postings against a brute-force scan of the token streams (drivers with more than 32 start positions included), the facet oracle's
counts against a per-document loop, and the order oracle's top-k against the literal sorted() rule on the tie- and extreme-heavy
date columns."""
import numpy as np
import pytest

import facet_oracle as FO
import order_oracle as OO
import phrase_model as PM
import test_gpu_keyword_edges as E


def brute_phrase(toks, phrase):
    """(freq, start indices among the occurrences of phrase[0]) of one phrase in one token stream [(position, term)]."""
    at = dict(toks)
    firsts = [p for p, t in toks if t == phrase[0]]
    hits = [i for i, s in enumerate(firsts) if all(at.get(s + j) == t for j, t in enumerate(phrase))]
    return len(hits), hits


def test_phrase_postings_equal_a_scan_of_the_token_streams():
    docs, term_off, post_doc, post_tf, fn, pos, flat, r_docs, r2_docs = E.phrase_corpus()
    model = PM.PhraseModel(E.N_PH, E.N_PH_TERMS, term_off, post_doc, post_tf, fn, pos=pos)
    planted = sorted(set(r_docs) | set(r2_docs))
    # R and R2 occur in the planted documents only: their phrases' postings are the scan of those documents
    assert set(post_doc[term_off[E.R]:term_off[E.R + 2]].tolist()) <= set(planted)
    assert all(70 <= sum(t == E.R for _, t in docs[d]) <= 100 for d in r_docs)
    windows = set()
    for phrase in E.PHRASES + [p for q in E.phrase_queries() for p in q[1]]:
        if not {E.R, E.R2} & set(phrase) or E.UNKNOWN in phrase:
            continue
        d, f = model.phrase_postings(phrase)
        want = {}
        for doc in planted:
            n, hits = brute_phrase(docs[doc], phrase)
            if n:
                want[doc] = n
            if phrase[0] == E.R:
                windows |= {h // 32 for h in hits}
        assert dict(zip(d.tolist(), f.tolist())) == want, phrase
    assert windows >= {0, 1, 2}   # matches start in the first three 32-start windows of R
    # background phrases over the first, the 32nd / 33rd and the last fine tiles
    tiles = [range(0, 4096), range(31 * 4096, 33 * 4096), range(63 * 4096, E.N_PH)]
    for phrase in ([E.A, E.B], [E.B, E.A, E.C], [E.C, E.B]):
        d, f = model.phrase_postings(phrase)
        got = dict(zip(d.tolist(), f.tolist()))
        for tile in tiles:
            want = {doc: n for doc in tile for n in [brute_phrase(docs[doc], phrase)[0]] if n}
            assert {doc: n for doc, n in got.items() if doc in tile} == want, phrase
            assert want or phrase != [E.A, E.B]


def literal_count(doc_off, ords, bucket, n_buckets, mask):
    """One document at a time: +1 for every distinct bucket among its ords."""
    out = np.zeros(n_buckets, np.int64)
    for d in np.nonzero(mask)[0]:
        for b in {int(bucket[o]) for o in ords[int(doc_off[d]):int(doc_off[d + 1])]} - {FO.NIL}:
            out[b] += 1
    return out


def test_facet_oracle_counts_equal_a_per_document_loop():
    cases = []
    for name in E.CORPORA:
        c = E.edge_case(name)
        P = c["P"]
        for alive in c["alive"][:: max(len(c["alive"]) - 1, 1)]:   # none and the one that kills the tile-boundary documents
            cases.append((c["doc_off"], c["ords"], FO.matched(P.n_docs, P.term_off, P.post_doc, [0, 2], False, alive)))
    for n in (1, 7, 9, 4095, 4097):
        doc_off, ords = E.facets_for(n, 12 + n)
        cases.append((doc_off, ords, FO.alive_mask(n, E.random_alive(n, n, 0.6))))
    for doc_off, ords, mask in cases:
        for r in E.REQUESTS:
            bucket, b_req, _ = FO.plan(E.KEYS, r)
            assert np.array_equal(FO.count(doc_off, ords, bucket, len(b_req), mask), literal_count(doc_off, ords, bucket, len(b_req), mask)), r
    assert [len(FO.plan(E.KEYS, r)[1]) for r in E.REQUESTS] == [1, 4096, 4097, 11]
    # the grid-stride test's catalogue (132 SMs), its widest request
    doc_off, ords = E.facets_for(N_132, 9)
    bucket, b_req, _ = FO.plan(E.KEYS, [b"m", b"z"])
    mask = FO.alive_mask(N_132, E.random_alive(N_132, 11, 0.8))
    assert np.array_equal(FO.count(doc_off, ords, bucket, len(b_req), mask), literal_count(doc_off, ords, bucket, len(b_req), mask))


@pytest.mark.parametrize("name", E.CORPORA)
def test_order_oracle_equals_the_literal_rule_on_the_edge_dates(name):
    c = E.edge_case(name)
    n = c["P"].n_docs
    for secs in (c["created"], c["modified"]):
        if n:
            assert (secs[c["edges"][::2]] == OO.NONE).all()
        for alive in c["alive"]:
            mask = FO.alive_mask(n, alive)
            for typ in (OO.DESC, OO.ASC):
                d, s = OO.order_topk(mask, secs, 1024, typ)
                want = OO.literal_order(np.nonzero(mask)[0], secs, typ)[:1024]
                assert d.tolist() == want and np.array_equal(s, secs[want])


N_132 = 2 * (2 * 132 * 512 * 8) + 13   # the grid-stride test's segment on a 132-SM H100


def test_order_oracle_equals_the_literal_rule_on_the_catalogue_dates():
    columns = E.round_dates(N_132, 2 * 132 * 512 * 8)
    mask = FO.alive_mask(N_132, E.random_alive(N_132, 11, 0.8))
    assert 0 < mask.sum() < N_132 and columns[1][N_132 - 6] == E.EXTREMES[0] and columns[1][N_132 - 1] == OO.NONE
    for secs in columns:
        for typ in (OO.DESC, OO.ASC):
            d, s = OO.order_topk(mask, secs, 1024, typ)
            assert d.tolist() == OO.literal_order(np.nonzero(mask)[0], secs, typ)[:1024]
    for n in (1, 7, 9, 4095, 4097):
        for columns in E.tail_columns(n):
            for alive in (None, E.random_alive(n, n, 0.6)):
                mask = FO.alive_mask(n, alive)
                for secs in columns:
                    for typ in (OO.DESC, OO.ASC):
                        want = OO.literal_order(np.nonzero(mask)[0], secs, typ)[:1024]
                        assert OO.order_topk(mask, secs, 1024, typ)[0].tolist() == want
