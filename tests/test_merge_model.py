"""The cross-shard merge orders on the host: the models of tests/merge_model.py against the reference's own shard_merge.rs tests and
hand-worked kmerge_by cases, and NidxBinding's merge of shard responses against the models."""
import itertools
import math
import random
import uuid

import pytest

import merge_model as M

SHARD_A = uuid.UUID("aaaaaaaa-aaaa-aaaa-aaaa-aaaaaaaaaaaa").bytes
SHARD_B = uuid.UUID("bbbbbbbb-bbbb-bbbb-bbbb-bbbbbbbbbbbb").bytes


def _uuids(merged):
    return [item[3] for item in merged]


# ---- kmerge_by: hand-worked cases (itertools 0.14 heapify / sift_down / swap_remove) --------------------------------------------
@pytest.mark.parametrize("n_parts,want", [
    (2, [(1, 0), (0, 0), (1, 1), (0, 1), (1, 2), (0, 2)]),
    (3, [(2, 0), (0, 0), (2, 1), (0, 1), (1, 0), (1, 1)]),
    (5, [(2, 0), (0, 0), (2, 1), (0, 1), (4, 0), (1, 0), (3, 0), (4, 1), (1, 1), (3, 1)]),
])
def test_kmerge_ties_are_not_lower_part_first(n_parts, want):
    """Every part scores (1.0, 1.0, 0.5): `>=` holds both ways for equal heads, so the heap's shape orders the ties."""
    got = M.merge_vector_responses([[1.0, 1.0, 0.5]] * n_parts, 3 * n_parts)
    assert got[:len(want)] == want
    assert sorted(got) == sorted((p, j) for p in range(n_parts) for j in range(3))
    assert all(j == 2 for _, j in got[2 * n_parts:])                        # every 1.0 before every 0.5


def test_kmerge_empty_and_one_item_parts():
    assert M.merge_vector_responses([], 10) == []
    assert M.merge_vector_responses([[], [], []], 10) == []
    assert M.merge_vector_responses([[], [0.5], []], 10) == [(1, 0)]
    assert M.merge_vector_responses([[0.25], [], [0.75]], 10) == [(2, 0), (0, 0)]
    assert M.merge_vector_responses([[0.5], [0.5]], 10) == [(1, 0), (0, 0)]
    assert M.merge_vector_responses([[0.9, 0.1], [0.5]], 1) == [(0, 0)]
    assert M.merge_vector_responses([[0.9, 0.1], [0.5]], 0) == []
    # empty parts never enter the heap: the non-empty ones are heapified as if they stood alone
    assert M.merge_vector_responses([[1.0, 1.0], [1.0, 1.0]], 4) == [(1, 0), (0, 0), (1, 1), (0, 1)]
    assert M.merge_vector_responses([[], [1.0, 1.0], [], [1.0, 1.0]], 4) == [(3, 0), (1, 0), (3, 1), (1, 1)]


def test_kmerge_signed_zero_ties_and_distinct_scores():
    assert M.merge_vector_responses([[0.0], [-0.0]], 2) == [(1, 0), (0, 0)]                     # -0.0 >= 0.0 and 0.0 >= -0.0
    assert M.merge_vector_responses([[math.inf, 1.0], [math.inf]], 3) == [(1, 0), (0, 0), (0, 1)]
    rng = random.Random(3)
    for _ in range(200):                                                                        # distinct scores: a plain sort
        n = rng.randint(1, 9)
        scores = rng.sample(range(10_000), n * 6)
        parts = [sorted(scores[i * 6:(i + 1) * 6][:rng.randint(0, 6)], reverse=True) for i in range(n)]
        want = sorted(((-s, p, j) for p, part in enumerate(parts) for j, s in enumerate(part)))
        assert M.merge_vector_responses(parts, 1000) == [(p, j) for _, p, j in want]


def test_kmerge_is_a_merge_of_sorted_parts():
    """With a strict total order, kmerge_by of sorted inputs is the sorted union whatever the heap does."""
    rng = random.Random(11)
    for _ in range(200):
        n = rng.randint(1, 12)
        items = rng.sample(range(100_000), 40)
        parts = [sorted(items[rng.randint(0, 39):][:rng.randint(0, 5)]) for _ in range(n)]
        got = [x for _, _, x in M.kmerge_by(parts, lambda a, b: a < b)]
        assert got == sorted(itertools.chain.from_iterable(parts))


# ---- the reference's shard_merge.rs tests, restated -------------------------------------------------------------------------------
def _doc(rid, score, docaddr, shard=b""):
    return (score, shard, docaddr, rid)


@pytest.mark.parametrize("merge", [M.merge_document_responses, M.merge_paragraph_responses])
def test_merge_results_by_score(merge):
    """test_merge_document_results_by_score (and its paragraph twin)."""
    merged = merge([[_doc("foo", 3.0, 2), _doc("bar", 2.0, 1)], [_doc("baz", 4.0, 2), _doc("quux", 2.0, 2)]], 20)
    assert _uuids(merged) == ["baz", "foo", "bar", "quux"]


@pytest.mark.parametrize("merge", [M.merge_document_responses, M.merge_paragraph_responses])
def test_merge_results_shard_tiebreak(merge):
    """test_merge_document_results_shard_tiebreak: equal score and docaddr -> shard_id bytes descending; equal shard -> docaddr."""
    assert _uuids(merge([[_doc("foo", 2.0, 1, SHARD_B)], [_doc("bar", 2.0, 1, SHARD_A)]], 20)) == ["foo", "bar"]
    assert _uuids(merge([[_doc("foo", 2.0, 1, SHARD_A)], [_doc("bar", 2.0, 1, SHARD_B)]], 20)) == ["bar", "foo"]
    assert _uuids(merge([[_doc("foo", 2.0, 2, SHARD_A)], [_doc("bar", 2.0, 1, SHARD_A)]], 20)) == ["bar", "foo"]


@pytest.mark.parametrize("merge", [M.merge_document_responses, M.merge_paragraph_responses])
def test_merge_results_with_limit(merge):
    """test_merge_documents_with_limit (and the paragraph twin): 2 shards x 20 default-scored results."""
    shard = [_doc("", 0.0, 0)] * 20
    assert len(merge([shard, shard], 50)) == 40
    assert len(merge([shard, shard], 20)) == 20


def test_sort_key_equals_the_comparator():
    rng = random.Random(5)
    pool = [0.0, -0.0, 1.0, 2.5, -1.0, math.inf, -math.inf]
    shards = [b"", b"a", b"a\x00", b"b", SHARD_A, SHARD_B]
    items = [(rng.choice(pool), rng.choice(shards), rng.randint(0, 3)) for _ in range(300)]
    by_key = sorted(items, key=M.sort_documents_key)
    for a, b in zip(by_key, by_key[1:]):
        assert not M.sort_documents_less(b, a)
    assert M.sort_documents_less((0.0, b"", 0), (-0.0, b"", 0))                                  # total_cmp: +0 above -0
    assert M.sort_documents_less((1.0, b"a\x00", 0), (1.0, b"a", 0))                               # longer byte string is greater


# ---- NidxBinding's merge against the models ------------------------------------------------------------------------------------------
def _binding_merge(parts, k):
    from nucliadb_b200 import nidx_protos as P
    from nucliadb_b200.binding import NidxBinding

    req = P.SearchRequest(result_per_page=k)
    return NidxBinding._merge(None, req, parts)


def test_binding_merges_documents_by_shard_bytes_descending():
    """Shard ids listed in the request in ascending byte order: on a tie the LATER shard (greater bytes) ranks first."""
    from nucliadb_b200 import text as T

    sids = [str(uuid.UUID(int=0x1111 * (i + 1))) for i in range(3)]           # ascending bytes, ascending list order
    rng = random.Random(7)
    parts, model_parts = [], []
    for sid in sids:
        rows = sorted(((float(rng.choice([1.0, 2.0, 3.0])), rng.randint(0, 5)) for _ in range(6)), key=lambda t: (-t[0], t[1]))
        rows = [r for i, r in enumerate(rows) if r not in rows[:i]]
        res = [T.DocumentResult(uuid=f"{sid}-{a}", field="/a/title", score=T.ResultScore(bm25=s, docaddr=a), labels=[]) for s, a in rows]
        parts.append((sid, {"document": T.DocumentSearchResponse(results=res, total=len(res)),
                            "paragraph": T.DocumentSearchResponse(results=list(res), total=len(res))}))
        model_parts.append([(s, sid.encode(), a, f"{sid}-{a}") for s, a in rows])
    for k in (1, 4, 7, 100):
        resp = _binding_merge(parts, k)
        want = [(u, s) for s, _, _, u in M.merge_document_responses(model_parts, k)]
        for target in (resp.document, resp.paragraph):
            assert [(r.uuid, r.score.bm25) for r in target.results] == want
            assert [r.shard_id for r in target.results] == [u.rsplit("-", 1)[0].encode() for u, _ in want]


def test_binding_merges_vectors_by_kmerge():
    from nucliadb_b200 import vector as V

    for n_parts in (2, 3, 5):
        parts = []
        for p in range(n_parts):
            docs = [V.DocumentScored(doc_id=f"p{p}-{j}", score=s, labels=[], metadata=None) for j, s in enumerate((1.0, 1.0, 0.5))]
            parts.append((str(uuid.UUID(int=p + 1)), {"vector": docs}))
        for k in (1, 2, 3, n_parts + 1, 3 * n_parts, 100):
            resp = _binding_merge(parts, k)
            want = [f"p{p}-{j}" for p, j in M.merge_vector_responses([[1.0, 1.0, 0.5]] * n_parts, k)]
            assert [d.doc_id.id for d in resp.vector.documents] == want
