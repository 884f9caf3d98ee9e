"""Host-side orders of the cross-shard merge (nidx/src/searcher/shard_merge.rs), for NidxBinding's merge of shard responses.

``kmerge_by`` restates itertools 0.14's KMergeBy (kmerge_impl.rs), which merge_vector_responses runs with
``|a, b| a.score >= b.score``: heapify over the non-empty inputs in input order, the branchless sift_down, and next() yielding
the head of heap[0], then advancing that input or swap_remove(0)-ing it when exhausted, then sift_down(0).  That predicate holds
both ways for equal scores, so equal scores are not resolved first input first: the heap's shape decides (two inputs scoring
(1, 1, 0.5) come out (input, position) = (1,0) (0,0) (1,1) (0,1) ...).  The inputs' order stands for the reference's `responses`
vector; kmerge_parts_kernel (csrc/shard.cuh) runs the same algorithm on the device.
"""
from __future__ import annotations

import struct

_END = object()


def kmerge_by(parts, less_than):
    """Merge the iterables `parts` (each already in merged order) -> yields (input index, item) in kmerge_by's order."""
    heap = []                                    # [input, head, iterator]
    for i, it in enumerate(parts):
        it = iter(it)
        head = next(it, _END)
        if head is not _END:
            heap.append([i, head, it])

    def sift_down(pos):
        child = 2 * pos + 1
        while child + 1 < len(heap):
            child += 1 if less_than(heap[child + 1][1], heap[child][1]) else 0
            if not less_than(heap[child][1], heap[pos][1]):
                return
            heap[pos], heap[child] = heap[child], heap[pos]
            pos, child = child, 2 * child + 1
        if child + 1 == len(heap) and less_than(heap[child][1], heap[pos][1]):
            heap[pos], heap[child] = heap[child], heap[pos]

    for i in reversed(range(len(heap) // 2)):
        sift_down(i)
    while heap:
        top = heap[0]
        out = (top[0], top[1])
        nxt = next(top[2], _END)
        if nxt is _END:
            last = heap.pop()
            if heap:
                heap[0] = last
        else:
            top[1] = nxt
        sift_down(0)
        yield out


class _Descending:
    """Bytes that sort in reverse."""

    __slots__ = ("b",)

    def __init__(self, b: bytes):
        self.b = bytes(b)

    def __eq__(self, other):
        return self.b == other.b

    def __lt__(self, other):
        return self.b > other.b


def bm25_order_key(bm25: float, shard_id: bytes, docaddr: int):
    """Sort key (ascending = ranked first) of sort_documents_fn / sort_paragraphs_fn by score (shard_merge.rs:211-231, 289-309):
    bm25 by f32 total_cmp descending, then shard_id bytes DEScending, then docaddr ascending."""
    (bits,) = struct.unpack("<i", struct.pack("<f", bm25))
    total = bits ^ 0x7FFFFFFF if bits < 0 else bits
    return (-total, _Descending(shard_id), docaddr)
