"""TEST INFRASTRUCTURE: TopDocs::order_by_fast_field + Count restated in numpy on the facet oracle's matched set, to check the
date-ordered results of libnidx_b200.so (bm25_order_kernel, bm25_order_facet_kernel, date_topk_all_kernel) exactly.

What is pinned by the reference (nidx_text/src/reader.rs:208-287, nidx_text/src/schema.rs:48-57): the matched set and Count are the
BM25 search's, dates are seconds (DateTime::from_timestamp_secs(ts.seconds), returned as {seconds, nanos: 0}), DESC puts later dates
first and ASC earlier ones, min_score and search-after do not apply, next_page = total > result_per_page.
What is fixed here [recalled: tantivy's order_by_fast_field leaves them to its collector]: equal dates are ordered by doc ascending,
and documents without a date come after every dated document in both directions.

Everything here is numpy over the arguments of the C ABI (include/nidx_b200.h); nothing is shared with the library's host code."""
import numpy as np

from facet_oracle import alive_mask, matched  # noqa: F401  (re-exported: the matched set is the facet oracle's)

NONE = -(1 << 63)   # NIDX_DATE_NONE
DESC, ASC = 0, 1


def order_topk(mask, secs, k, order_type):
    """The top k documents of `mask` by (date in the direction, undated last, doc ascending) -> (docs int64, dates int64)."""
    secs = np.asarray(secs, dtype=np.int64)
    docs = np.nonzero(mask)[0].astype(np.int64)
    s = secs[docs]
    has = s != NONE
    # -s cannot overflow: NONE (the only value without a negation) is replaced by 0 first
    direction = np.where(has, s if order_type == ASC else -np.where(has, s, 0), 0)
    idx = np.lexsort((docs, direction, ~has))
    top = docs[idx][:k]
    return top, secs[top]


def search(n_docs, term_off, post_doc, terms, conj, alive, secs, k, order_type):
    """One ordered query: (docs, dates, total)."""
    mask = matched(n_docs, term_off, post_doc, terms, conj, alive)
    d, s = order_topk(mask, secs, k, order_type)
    return d, s, int(mask.sum())


def list_all(n_docs, alive, secs, k, order_type):
    """The empty body (AllQuery): (docs, dates, total alive)."""
    mask = alive_mask(n_docs, alive)
    d, s = order_topk(mask, secs, k, order_type)
    return d, s, int(mask.sum())


def literal_order(docs, secs, order_type):
    """The order rule as written, on Python ints: sorted() by (undated, date in the direction, doc)."""
    def key(d):
        s = int(secs[d])
        return (s == NONE, 0 if s == NONE else (s if order_type == ASC else -s), d)
    return sorted((int(d) for d in docs), key=key)
