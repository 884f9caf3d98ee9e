"""TEST INFRASTRUCTURE: tantivy's FacetCollector restated on the oracle's own matched set, to check the facet counts of
libnidx_b200.so (bm25_facet_kernel, facet_count_all_kernel) exactly.

FacetCollector [recalled] (tantivy 0.26 collector/facet_collector.rs, outside the reference's tree): add_facet(F) for every
requested facet, asserting that no requested facet is an ancestor of another; per segment it resolves F to the term-ord range of
its descendants and collapses every ord to the child of F it lies under; a document adds one to each DISTINCT collapsed child
(FacetSegmentCollector::collect keeps the last collapsed ord and skips repeats); a facet equal to F counts nothing.  Counts of the
segments add up.  Facets are tantivy's encoded keys: segments joined by 0x00 bytes, the root "/" = b"".

Everything here is numpy over the arguments of the C ABI (include/nidx_b200.h); nothing is shared with the library's host code."""
import numpy as np

NIL = 0xFFFFFFFF


def matched(n_docs, term_off, post_doc, terms, conj, alive_bits=None):
    """The set Count counts (bool[n_docs]): query match (OR: any term, AND: every term) AND alive.  Terms outside the
    vocabulary have no postings."""
    n_terms = len(term_off) - 1
    sets = []
    for t in terms:
        m = np.zeros(n_docs, dtype=bool)
        if int(t) < n_terms:
            m[post_doc[int(term_off[t]):int(term_off[t + 1])]] = True
        sets.append(m)
    if not sets:
        return np.zeros(n_docs, dtype=bool)
    out = np.logical_and.reduce(sets) if conj else np.logical_or.reduce(sets)
    return out & alive_mask(n_docs, alive_bits)


def alive_mask(n_docs, alive_bits=None):
    if alive_bits is None:
        return np.ones(n_docs, dtype=bool)
    bits = np.unpackbits(np.asarray(alive_bits, dtype=np.uint64).view(np.uint8), bitorder="little")
    return bits[:n_docs].astype(bool)


def _segments(key: bytes):
    return [] if key == b"" else key.split(b"\0")


def is_ancestor(a: bytes, b: bytes) -> bool:
    sa, sb = _segments(a), _segments(b)
    return len(sa) < len(sb) and sb[: len(sa)] == sa


def plan(keys, request):
    """keys: the dictionary (facet order); request: encoded facets.  -> (bucket[n_keys] ord -> bucket or NIL, bucket_req,
    bucket_ord) with the requests in facet order (duplicates collapse) and the children in facet order.  Raises ValueError
    for a request holding an ancestor of another of its facets."""
    uniq = sorted(set(request))
    for a in uniq:
        for b in uniq:
            if is_ancestor(a, b):
                raise ValueError("a requested facet is an ancestor of another requested facet")
    bucket = np.full(len(keys), NIL, dtype=np.uint32)
    b_req, b_ord = [], []
    for f in uniq:
        fs = _segments(f)
        children = {}
        for o, key in enumerate(keys):
            ks = _segments(key)
            if len(ks) > len(fs) and ks[: len(fs)] == fs:
                child = tuple(ks[: len(fs) + 1])
                if child not in children:
                    children[child] = len(b_req)
                    b_req.append(request.index(f))
                    b_ord.append(o)
                bucket[o] = children[child]
    return bucket, np.asarray(b_req, dtype=np.uint32), np.asarray(b_ord, dtype=np.uint32)


def count(doc_off, ords, bucket, n_buckets, mask):
    """Bucket counts over the documents of `mask`: one per (document, distinct bucket)."""
    doc_off = np.asarray(doc_off, dtype=np.int64)
    n_docs = len(doc_off) - 1
    if n_buckets == 0 or len(ords) == 0:
        return np.zeros(n_buckets, dtype=np.int64)
    doc = np.repeat(np.arange(n_docs, dtype=np.int64), np.diff(doc_off))
    b = bucket[np.asarray(ords, dtype=np.int64)].astype(np.int64)
    keep = (b != NIL) & mask[doc]
    pairs = np.unique(doc[keep] * n_buckets + b[keep])
    return np.bincount(pairs % n_buckets, minlength=n_buckets).astype(np.int64)
