"""Host models of the cross-part merges of a search, independent of nucliadb_b200.

- ``kmerge_by``: itertools 0.14's ``KMergeBy`` (src/kmerge_impl.rs), which the reference's shard merge runs.  The crate's source
  is not part of the reference tree, so this restatement was written from memory of the crate: ``heapify`` over the non-empty
  inputs in input order, the branchless ``sift_down`` (the right child is taken when ``less_than(right, left)``), and ``next``
  yielding the head of ``heap[0]``, then advancing that input or ``swap_remove(0)``-ing it when exhausted, then ``sift_down(0)``.
  The one property the vector merge's tie order rests on -- equal heads are not resolved lower input first -- follows from the
  ``>=`` predicate (it holds both ways for equal scores) and any ``sift_down`` that swaps when ``less_than(child, parent)``.
- ``merge_vector_responses``: shard_merge.rs:332-348, ``kmerge_by(|a, b| a.score >= b.score).take(limit)`` on f32 scores.
- ``sort_documents_less`` / ``sort_documents_key`` (and the paragraph twins): the comparator of shard_merge.rs:211-231 / 289-309,
  ``bm25.total_cmp`` then ``shard_id`` bytes then docaddr reversed, ``.is_gt()``: bm25 descending, shard_id bytes DEScending,
  docaddr ascending.

Parts are taken in the order given: it stands for the order of the reference's ``responses`` vector, which follows node grouping
(grpc.rs:253-285), so the reference fixes no order across nodes; what is pinned here is kmerge_by's output for a given order.
"""
from __future__ import annotations

import functools
import struct


def kmerge_by(parts, less_than):
    """Merge the iterables `parts` -> yields (part index, position in the part, item) in kmerge_by's order."""
    heap = []                                    # [part, position, head, iterator]
    for p, it in enumerate(parts):               # HeadTail::new: inputs without a first item never enter the heap
        it = iter(it)
        for head in it:
            heap.append([p, 0, head, it])
            break

    def lt(a, b):
        return less_than(a[2], b[2])

    def sift_down(pos):
        child = 2 * pos + 1
        while child + 1 < len(heap):
            child += 1 if lt(heap[child + 1], heap[child]) else 0
            if not lt(heap[child], heap[pos]):
                return
            heap[pos], heap[child] = heap[child], heap[pos]
            pos, child = child, 2 * child + 1
        if child + 1 == len(heap) and lt(heap[child], heap[pos]):
            heap[pos], heap[child] = heap[child], heap[pos]

    for i in reversed(range(len(heap) // 2)):    # heapify
        sift_down(i)
    while heap:
        top = heap[0]
        out = (top[0], top[1], top[2])
        nxt = next(top[3], _END)
        if nxt is _END:                          # HeadTail::next -> None: swap_remove(0)
            last = heap.pop()
            if heap:
                heap[0] = last
        else:
            top[1], top[2] = top[1] + 1, nxt
        sift_down(0)
        yield out


_END = object()


def f32(x) -> float:
    return struct.unpack("<f", struct.pack("<f", float(x)))[0]


def merge_vector_responses(parts, k):
    """parts = per-part score lists (each sorted descending, as the shards return them) -> [(part, position)] of the first k items
    of kmerge_by(|a, b| a.score >= b.score).  IEEE comparisons on f32 values: -0.0 == +0.0, a NaN is never >=."""
    out = []
    if k <= 0:
        return out
    for p, j, _ in kmerge_by([[f32(s) for s in part] for part in parts], lambda a, b: a >= b):
        out.append((p, j))
        if len(out) == k:
            break
    return out


def total_order_key(x) -> int:
    """f32::total_cmp as an integer key: -NaN < -inf < ... < -0.0 < +0.0 < ... < +inf < +NaN."""
    (bits,) = struct.unpack("<i", struct.pack("<f", float(x)))
    return bits ^ 0x7FFFFFFF if bits < 0 else bits


def _cmp(a, b) -> int:
    return (a > b) - (a < b)


def sort_documents_cmp(a, b) -> int:
    """a, b = (bm25, shard_id bytes, docaddr): the reference's Ordering of a against b (Greater = a ranks first)."""
    c = _cmp(total_order_key(a[0]), total_order_key(b[0]))
    if c == 0:
        c = _cmp(bytes(a[1]), bytes(b[1]))
    if c == 0:
        c = -_cmp(a[2], b[2])
    return c


def sort_documents_less(a, b) -> bool:
    """sort_documents_fn(Score): the kmerge_by predicate, `.is_gt()` of the comparison."""
    return sort_documents_cmp(a, b) > 0


def sort_documents_key(item):
    """Sort key of (bm25, shard_id bytes, docaddr) in merged order (ascending key = earlier)."""
    return functools.cmp_to_key(lambda a, b: -sort_documents_cmp(a, b))(item)


# sort_paragraphs_fn(Score) is the same comparator over ParagraphResult's fields (shard_merge.rs:289-309)
sort_paragraphs_cmp, sort_paragraphs_less, sort_paragraphs_key = sort_documents_cmp, sort_documents_less, sort_documents_key


def merge_document_responses(parts, limit):
    """merge_document_responses / merge_paragraph_responses' results (shard_merge.rs:177-207, 233-264): parts = per-shard lists of
    (bm25, shard_id bytes, docaddr, payload...) -> the first `limit` items of kmerge_by(sort_documents_fn)."""
    out = []
    for _, _, item in kmerge_by(parts, sort_documents_less):
        if len(out) == limit:
            break
        out.append(item)
    return out


merge_paragraph_responses = merge_document_responses
