"""A literal per-document restatement of SearchRequest.security, as nidx_text indexes and queries it.  No dictionaries, no ranges,
no bitsets: every check is made on the document's own group strings.

    indexing   nidx_text/src/resource_indexer.rs:49-62: a resource with a non-empty security.access_groups is indexed with
               groups_public = 0 and each group, with a '/' put in front when it lacks one, as a facet of groups_with_access; a
               resource without groups gets groups_public = 1.
    query      nidx_text/src/search_query.rs:63-87 (security_query): the union of groups_public = 1 and one facet term per requested
               group, again with a leading '/' added.  A facet term matches the facet and its descendants (tantivy indexes every
               ancestor of a facet path [recalled]), so group "/a" grants a resource of group "/a/b" but not one of "/ab".
    prefilter  nidx_text/src/reader.rs:147-160: the intersection of security_query and field_filter's query.
"""
from __future__ import annotations

import prefilter_model


def normalize(group: str) -> str:
    """The leading '/' both sides add (resource_indexer.rs:53-57, search_query.rs:76-80)."""
    return group if group.startswith("/") else "/" + group


def _under(path: str, f: str) -> bool:
    return f == "/" or path == f or path.startswith(f + "/")


def granted(doc_groups, access_groups) -> bool:
    """security_query on one document: public (no groups), or one of its groups lies at or under a requested group."""
    if not doc_groups:
        return True
    return any(_under(normalize(d), normalize(g)) for d in doc_groups for g in access_groups)


def matches(doc, access_groups=None, field_filter=None) -> bool:
    """TextReaderService::prefilter's query on one document: security (None: absent) AND field_filter (None: absent)."""
    if access_groups is not None and not granted(doc.groups, access_groups):
        return False
    return field_filter is None or prefilter_model.matches(field_filter, doc)


def bits(segments, access_groups=None, field_filter=None, alive=None):
    """segments: [[TextDoc]], alive: [[bool]] or None -> per segment [bool] matched and alive."""
    alive = alive if alive is not None else [[True] * len(s) for s in segments]
    return [[a and matches(d, access_groups, field_filter) for d, a in zip(docs, al)] for docs, al in zip(segments, alive)]


def visible(messages):
    """The sequence rule over a shard's index messages, oldest first: ("index", resource id, groups) or ("delete", resource id).
    Each message has the next sequence number; a message deletes its resource from every OLDER segment (the reference applies
    deletions to segments with a lower seq).  -> {resource id: groups} of the copies still alive."""
    out = {}
    for m in messages:
        out.pop(m[1], None)
        if m[0] == "index":
            out[m[1]] = tuple(m[2])
    return out


def eval_nodes(flat, doc_ords) -> bool:
    """The flat pre-order prefilter nodes of a security expression (OR, PUBLIC, GROUP) on one document's group ords."""
    def ev(i):
        kind, n, lo, hi, _ = flat[i]
        from nucliadb_b200 import _lib

        if kind == _lib.NIDX_P_PUBLIC:
            return not doc_ords, i + 1
        if kind == _lib.NIDX_P_GROUP:
            return any(lo <= o < hi for o in doc_ords), i + 1
        assert kind in (_lib.NIDX_P_OR, _lib.NIDX_P_AND)
        vals, j = [], i + 1
        for _ in range(n):
            v, j = ev(j)
            vals.append(v)
        return (any(vals) if kind == _lib.NIDX_P_OR else bool(vals) and all(vals)), j

    v, end = ev(0)
    assert end == len(flat)
    return v
