"""The relation index (reference: nidx/nidx_relation) and ``NidxSearcher.GraphSearch`` on the device.

Index (resource_indexer.rs): one document per IndexRelation of ``Resource.field_relations``: source and target (raw value, normalised
value, default tokens, type, subtype), relation type, label, metadata, ``resource_field_id`` = (resource, field key) and facets.

Query (graph_query_parser.rs) is restated by ``path_query`` / ``node_query`` as a tree of tantivy queries:
  ("bool", [(occur, q)])   occur MUST / SHOULD / MUST_NOT
  ("term", field, value)   fields src_norm dst_norm src_type dst_type src_sub dst_sub rel_type label facet
  ("termset", field, [tokens]), fields src_tok dst_tok
  ("fuzzy", field, term, distance, prefix)   on src_norm / dst_norm / src_tok / dst_tok
  ("all",), ("empty",)

Scoring, *recalled, unverifiable here* (tantivy is not in the tree; DESIGN 9 lists the rules):
  * a term leaf scores BM25 for a one-token field with tf = 1 over the index's alive documents (N) and the term's alive documents
    (df), in the f32 formula of the BM25 kernel: ``idf * (1 + K1) / (1 + K1)`` computed step by step;
  * a term set, a fuzzy term and the all query score 1.0;
  * a boolean sums its matched MUST clauses in order, then adds the sum of its matched SHOULD clauses (in order); MUST_NOT adds
    nothing; without MUST a SHOULD must match; with neither nothing matches;
  * a Some prefilter is a MUST clause scored 1.0 ahead of the query;
  * ties: PATH by document ascending, NODES / RELATIONS by key ascending (the reference's HashMap order is not fixed);
  * fuzzy: restricted Damerau-Levenshtein (a transposition costs one) on code points, distance <= 2; a prefix term matches an
    entry when some prefix of the entry is within the distance.

Normalisation (schema.rs:123-137): per whitespace-separated word, deunicode then ASCII lowercase, joined by one space.  deunicode is
restated exactly for ASCII and for Latin letters with diacritics (NFKD, combining marks dropped); other scripts keep their characters
(deunicode would transliterate them), a documented difference.
"""
from __future__ import annotations

import ctypes as C
import unicodedata
import uuid as _uuid
from dataclasses import dataclass
from typing import Optional, Sequence

import numpy as np

from . import _lib
from .text import facet_key, tokenize

MUST, SHOULD, MUST_NOT = "must", "should", "must_not"
PATH, NODES, RELATIONS = 0, 1, 2
MAX_TOP_K = 1024
K1, B = np.float32(1.2), np.float32(0.75)
META_FIELD = "a/metadata"

COLUMNS = {"src_norm": 0, "dst_norm": 1, "src_type": 2, "dst_type": 3, "src_sub": 4, "dst_sub": 5, "rel_type": 6, "label": 7}
SRC_NODE, DST_NODE, REL_KEY = 8, 9, 10


def _deunicode_word(w: str) -> str:
    out = []
    for ch in w:
        if ord(ch) < 128:
            out.append(ch)
            continue
        base = "".join(c for c in unicodedata.normalize("NFKD", ch) if not unicodedata.combining(c))
        out.append(base if base and all(ord(c) < 128 for c in base) else ch)
    return "".join(out)


def normalize(value: str) -> str:
    """Schema::normalize: deunicode every whitespace-separated word, ASCII-lowercase it, join with one space."""
    return " ".join(_deunicode_word(w).translate(_ASCII_LOWER) for w in value.split())


_ASCII_LOWER = {c: c + 32 for c in range(ord("A"), ord("Z") + 1)}


@dataclass
class GraphDoc:
    """One relation: source / target nodes as (value, type, subtype)."""
    rid: str
    field: str
    source: tuple
    target: tuple
    rel_type: int
    label: str
    metadata: Optional[bytes] = None
    facets: tuple = ()


def docs_from_resource(res) -> list:
    """Resource.field_relations -> [GraphDoc] (resource_indexer.rs:20-97)."""
    rid = _uuid.UUID(res.resource.uuid).hex
    out = []
    for fkey in sorted(res.field_relations):
        for ir in res.field_relations[fkey].relations:
            r = ir.relation
            if not r.HasField("source") or not r.HasField("to"):
                raise ValueError("Missing source" if not r.HasField("source") else "Missing target")
            out.append(GraphDoc(rid, fkey, (r.source.value, int(r.source.ntype), r.source.subtype), (r.to.value, int(r.to.ntype), r.to.subtype),
                                int(r.relation), r.relation_label, r.metadata.SerializeToString() if r.HasField("metadata") else None, tuple(ir.facets)))
    return out


def doc_terms(d: GraphDoc) -> dict:
    """field -> the document's terms (term and fuzzy leaves)."""
    return {"src_norm": [normalize(d.source[0])], "dst_norm": [normalize(d.target[0])], "src_tok": tokenize(d.source[0]), "dst_tok": tokenize(d.target[0]),
            "src_type": [d.source[1]], "dst_type": [d.target[1]], "src_sub": [d.source[2]], "dst_sub": [d.target[2]], "rel_type": [d.rel_type],
            "label": [d.label]}


def leaf_score(n_docs: int, df: int) -> np.float32:
    """BM25 of a one-token field at tf = 1, in f32 as the BM25 kernel computes it."""
    idf = np.float32(np.log(np.float32(1.0) + (np.float32(n_docs - df) + np.float32(0.5)) / (np.float32(df) + np.float32(0.5))))
    weight = np.float32(idf * (np.float32(1.0) + K1))
    norm = np.float32(K1 * (np.float32(1.0) - B + B * np.float32(1.0) / np.float32(1.0)))
    return np.float32(weight * np.float32(1.0) / np.float32(np.float32(1.0) + norm))


# ---- graph_query_parser.rs ------------------------------------------------------------------------------------------------------
_SIDE = {"src": ("src_norm", "src_tok", "src_type", "src_sub"), "dst": ("dst_norm", "dst_tok", "dst_type", "dst_sub")}


def _node_value(node, side: str):
    norm_f, tok_f = _SIDE[side][0], _SIDE[side][1]
    if not node.HasField("value"):
        return None
    v = node.value
    mk = node.WhichOneof("match_kind")
    if mk == "vector":
        raise NotImplementedError("semantic node matches (VectorMatch) are not supported")
    if v == "":
        return None
    loc = (node.exact.kind if mk == "exact" else node.fuzzy.kind) if mk else 0
    dist = int(node.fuzzy.distance) if mk == "fuzzy" else 0
    if mk == "fuzzy" and dist > 2:
        raise ValueError(f"fuzzy distance {dist} is above 2")
    if mk != "fuzzy" and loc == 0:
        return ("term", norm_f, normalize(v))
    if mk != "fuzzy" and loc == 2:
        return ("termset", tok_f, tokenize(v))
    prefix = loc in (1, 3)
    if loc in (0, 1):
        return ("fuzzy", norm_f, normalize(v), dist, prefix)
    toks = tokenize(v)
    if len(toks) == 1:
        return ("fuzzy", tok_f, toks[0], dist, prefix)
    return ("bool", [(MUST, ("fuzzy", tok_f, t, dist, prefix)) for t in toks])


def _has_node(node, side: str) -> list:
    if node is None:
        return []
    out = []
    q = _node_value(node, side)
    if q is not None:
        out.append(q)
    if node.HasField("node_type"):
        out.append(("term", _SIDE[side][2], int(node.node_type)))
    if node.HasField("node_subtype") and node.node_subtype:
        out.append(("term", _SIDE[side][3], node.node_subtype))
    return out


def _has_relation(rel) -> list:
    if rel is None:
        return []
    out = []
    if rel.HasField("value"):
        if rel.WhichOneof("match_kind") == "vector":
            raise NotImplementedError("semantic relation matches (VectorMatch) are not supported")
        out.append((MUST, ("term", "label", rel.value)))
    if rel.HasField("relation_type"):
        out.append((MUST, ("term", "rel_type", int(rel.relation_type))))
    return out


def _directed(src, rel, dst):
    subs = [(MUST, q) for q in _has_node(src, "src")] + _has_relation(rel) + [(MUST, q) for q in _has_node(dst, "dst")]
    if all(o == MUST_NOT for o, _ in subs):
        subs.append((MUST, ("all",)))
    return ("bool", subs)


def _facet(f: str):
    return ("term", "facet", f)


def path_query(pq):
    """GraphQuery.PathQuery -> the query tree of BoolGraphQuery + parse_bool (PATH and RELATIONS)."""
    kind = pq.WhichOneof("query")
    if kind is None:
        return ("bool", [(SHOULD, _directed(None, None, None)), (SHOULD, _directed(None, None, None))])
    if kind == "path":
        p = pq.path
        src = p.source if p.HasField("source") else None
        rel = p.relation if p.HasField("relation") else None
        dst = p.destination if p.HasField("destination") else None
        if p.undirected:
            return ("bool", [(SHOULD, _directed(src, rel, dst)), (SHOULD, _directed(dst, rel, src))])
        return _directed(src, rel, dst)
    if kind == "bool_not":
        return ("bool", [(MUST, ("all",)), (MUST_NOT, path_query(pq.bool_not))])
    if kind == "facet":
        return _facet(pq.facet.facet)
    occur = MUST if kind == "bool_and" else SHOULD
    return ("bool", [(occur, path_query(o)) for o in getattr(pq, kind).operands])


def node_query(pq, side: str):
    """GraphQuery.PathQuery -> the query tree of BoolNodeQuery + parse_bool_node for one side (NODES).  A path other than an
    undirected source-only one is a ValueError."""
    kind = pq.WhichOneof("query")
    if kind is None:
        return _directed(None, None, None)
    if kind == "path":
        p = pq.path
        if not (p.HasField("source") and not p.HasField("relation") and not p.HasField("destination") and p.undirected):
            raise ValueError("Invalid node query, we only expect a source for an undirected path")
        return _directed(p.source, None, None) if side == "src" else _directed(None, None, p.source)
    if kind == "bool_not":
        return ("bool", [(MUST, ("all",)), (MUST_NOT, node_query(pq.bool_not, side))])
    if kind == "facet":
        return _facet(pq.facet.facet)
    occur = MUST if kind == "bool_and" else SHOULD
    return ("bool", [(occur, node_query(o, side)) for o in getattr(pq, kind).operands])


def with_prefilter(q, some: bool):
    """apply_prefilter for a Some: intersection(TermSet(resource_field_ids), q); the term set scores 1.0."""
    return ("bool", [(MUST, ("prefilter",)), (MUST, q)]) if some else q


# ---- the index on the device ----------------------------------------------------------------------------------------------------
def _cp_dict(keys: list):
    cps = [np.frombuffer(k.encode("utf-32-le"), dtype=np.uint32) for k in keys]
    off = np.zeros(len(keys) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(c) for c in cps]) if keys else []
    return (np.concatenate(cps) if cps else np.zeros(0, dtype=np.uint32)).astype(np.uint32), off


def _facet_range(keys: list, f: str):
    k = facet_key(f)
    if k is None:
        return 0, 0
    import bisect

    lo = bisect.bisect_left(keys, k)
    hi = bisect.bisect_left(keys, k + b"\x01") if k else len(keys)
    return lo, hi


class GraphIndex:
    """The alive relations of a shard on one device: a text segment without terms (facets, resource / field ords) and the graph
    columns (nidx_graph_set_columns).  The dictionaries and document frequencies stay here."""

    def __init__(self, docs: Sequence[GraphDoc], device=0):
        from .segment import TextSegment

        self.docs, self.device, self.n_docs = list(docs), device, len(docs)
        terms = [doc_terms(d) for d in self.docs]
        self.values = sorted({t for ts in terms for t in ts["src_norm"] + ts["dst_norm"]})
        self.tokens = sorted({t for ts in terms for t in ts["src_tok"] + ts["dst_tok"]})
        self.subtypes = sorted({t for ts in terms for t in ts["src_sub"] + ts["dst_sub"]})
        self.labels = sorted({d.label for d in self.docs})
        self.node_keys = sorted({d.source for d in self.docs} | {d.target for d in self.docs})
        self.rel_keys = sorted({(d.rel_type, d.label) for d in self.docs})
        self.facet_keys = sorted({k for d in self.docs for k in map(facet_key, d.facets) if k is not None})
        self.df: dict = {}
        for d in self.docs:   # a facet term is every facet of the document and each of its ancestors
            valid = [k for k in map(facet_key, d.facets) if k is not None]
            for k in {k[:i] for k in valid for i in [j for j, c in enumerate(k) if c == 0] + [len(k)]} | ({b""} if valid else set()):
                self.df[("facet", k)] = self.df.get(("facet", k), 0) + 1
        for ts in terms:
            for f, vs in ts.items():
                for v in set(vs):
                    self.df[(f, v)] = self.df.get((f, v), 0) + 1
        ords = lambda xs: {x: i for i, x in enumerate(xs)}   # noqa: E731
        vo, to, so, lo, no, ro, fo = map(ords, (self.values, self.tokens, self.subtypes, self.labels, self.node_keys, self.rel_keys, self.facet_keys))
        n = self.n_docs
        u32 = lambda xs: np.asarray(xs, dtype=np.uint32)   # noqa: E731
        cols = [u32([vo[ts["src_norm"][0]] for ts in terms]), u32([vo[ts["dst_norm"][0]] for ts in terms]),
                u32([d.source[1] for d in self.docs]), u32([d.target[1] for d in self.docs]),
                u32([so[d.source[2]] for d in self.docs]), u32([so[d.target[2]] for d in self.docs]),
                u32([d.rel_type for d in self.docs]), u32([lo[d.label] for d in self.docs]),
                u32([no[d.source] for d in self.docs]), u32([no[d.target] for d in self.docs]), u32([ro[(d.rel_type, d.label)] for d in self.docs])]
        toks = []
        for side in ("src_tok", "dst_tok"):
            rows = [sorted({to[t] for t in ts[side]}) for ts in terms]
            off = np.zeros(n + 1, dtype=np.uint64)
            off[1:] = np.cumsum([len(r) for r in rows]) if n else []
            toks.append((off, u32([o for r in rows for o in r])))
        self.resource_ids = sorted({d.rid for d in self.docs})
        self.fields = sorted({d.field for d in self.docs})
        self.segment = TextSegment.create(n, 0, np.zeros(1, dtype=np.uint64), np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.uint32),
                                          np.zeros(n, dtype=np.uint8), device=device)
        self.graph = None
        try:
            frows = [sorted({fo[k] for k in map(facet_key, d.facets) if k is not None}) for d in self.docs]
            foff = np.zeros(n + 1, dtype=np.uint64)
            foff[1:] = np.cumsum([len(r) for r in frows]) if n else []
            self.segment.set_facets(self.facet_keys, foff, u32([o for r in frows for o in r]))
            rord, ford = ords(self.resource_ids), ords(self.fields)
            self.segment.set_doc_columns(u32([rord[d.rid] for d in self.docs]), u32([ford[d.field] for d in self.docs]))
            vcp, voff = _cp_dict(self.values)
            tcp, toff = _cp_dict(self.tokens)
            c = _lib.GraphColumns()
            for i, a in enumerate(cols):
                c.col[i] = a.ctypes.data
            for s in range(2):
                c.tok_off[s], c.tok_ord[s] = toks[s][0].ctypes.data, toks[s][1].ctypes.data
            self._keep = (cols, toks, vcp, voff, tcp, toff)
            c.n_values, c.value_cp, c.value_off = len(self.values), _lib.ptr(vcp), _lib.ptr(voff)
            c.n_tokens, c.token_cp, c.token_off = len(self.tokens), _lib.ptr(tcp), _lib.ptr(toff)
            c.n_node_keys, c.n_rel_keys = len(self.node_keys), len(self.rel_keys)
            h = C.c_void_p()
            L = _lib.load()
            _lib.check(L.nidx_graph_create(self.segment._h, C.byref(h)))
            self.graph = h
            _lib.check(L.nidx_graph_set_columns(self.graph, C.addressof(c)))
        except BaseException:
            self.close()
            raise
        self._value_ord, self._token_ord, self._sub_ord, self._label_ord = vo, to, so, lo

    def close(self):
        if self.graph is not None:
            _lib.load().nidx_graph_close(self.graph)
            self.graph = None
        if self.segment is not None:
            self.segment.close()
            self.segment = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- query tree -> pre-order nidx_graph_node ---------------------------------------------------------------------------------
    def compile(self, q, nodes: list, terms: list, keep: list):
        """Append q's nodes (and its automaton terms) in the scoring rules of the module docstring."""
        G = _lib
        kind = q[0]

        def node(k, n=0, arg=0, w=0.0, lo=0, hi=0, ords=None):
            nodes.append(G.GraphNode(k, n, arg, float(w), lo, hi, G.ptr(ords)))

        if kind == "all":
            node(G.NIDX_G_CONST, w=1.0, lo=1)
        elif kind == "prefilter":
            node(G.NIDX_G_CONST, w=1.0, lo=1)
        elif kind == "empty":
            node(G.NIDX_G_CONST, lo=0)
        elif kind == "term":
            f, v = q[1], q[2]
            w = leaf_score(self.n_docs, self.df_of(f, v))
            if f == "facet":
                lo, hi = _facet_range(self.facet_keys, v)
                if hi > lo:
                    node(G.NIDX_G_FACET, w=w, lo=lo, hi=hi)
                else:
                    node(G.NIDX_G_CONST, lo=0)
                return
            o = self._ord(f, v)
            if o is None:
                node(G.NIDX_G_CONST, lo=0)
            else:
                node(G.NIDX_G_EQ, arg=COLUMNS[f], w=w, lo=o)
        elif kind == "termset":
            found = np.asarray(sorted({self._token_ord[t] for t in q[2] if t in self._token_ord}), dtype=np.uint32)
            if len(found) == 0:
                node(G.NIDX_G_CONST, lo=0)
            else:
                keep.append(found)
                node(G.NIDX_G_TOKSET, n=len(found), arg=0 if q[1] == "src_tok" else 1, w=1.0, ords=found)
        elif kind == "fuzzy":
            f, term, dist, prefix = q[1:]
            cp = np.frombuffer(term.encode("utf-32-le"), dtype=np.uint32).copy()
            keep.append(cp)
            tok = f.endswith("_tok")
            terms.append(G.GraphTerm(G.NIDX_G_TERMS_TOKENS if tok else G.NIDX_G_TERMS_VALUES, int(dist), int(prefix), len(cp), G.ptr(cp)))
            if tok:
                node(G.NIDX_G_TOKBITS, arg=0 if f == "src_tok" else 1, w=1.0, lo=len(terms) - 1)
            else:
                node(G.NIDX_G_COLBITS, arg=COLUMNS[f], w=1.0, lo=len(terms) - 1)
        else:   # bool
            clauses = q[1]
            musts = [c for o, c in clauses if o == MUST]
            shoulds = [c for o, c in clauses if o == SHOULD]
            nots = [c for o, c in clauses if o == MUST_NOT]
            if not musts and not shoulds:
                node(G.NIDX_G_CONST, lo=0)
                return
            core = musts if musts else None
            n_and = (1 if core else 0) + len(nots) + (1 if musts and shoulds else 0)
            if not core:
                n_and += 1   # the SHOULD group is the core
            node(G.NIDX_G_AND, n=n_and)
            if core:
                node(G.NIDX_G_AND, n=len(musts))
                for c in musts:
                    self.compile(c, nodes, terms, keep)
            else:
                node(G.NIDX_G_OR, n=len(shoulds))
                for c in shoulds:
                    self.compile(c, nodes, terms, keep)
            for c in nots:
                node(G.NIDX_G_NOT, n=1)
                self.compile(c, nodes, terms, keep)
            if musts and shoulds:   # optional: OR(shoulds, an always-true clause scored 0)
                node(G.NIDX_G_OR, n=len(shoulds) + 1)
                for c in shoulds:
                    self.compile(c, nodes, terms, keep)
                node(G.NIDX_G_CONST, lo=1, w=0.0)

    def df_of(self, f: str, v) -> int:
        if f == "facet":
            k = facet_key(v)
            return 0 if k is None else self.df.get(("facet", k), 0)
        return self.df.get((f, v), 0)

    def _ord(self, f: str, v):
        if f in ("src_norm", "dst_norm"):
            o = self._value_ord.get(v)
        elif f in ("src_sub", "dst_sub"):
            o = self._sub_ord.get(v)
        elif f == "label":
            o = self._label_ord.get(v)
        else:
            o = int(v)
        return o if o is not None and self.df.get((f, v), 0) else None

    def search(self, trees: list, kind: int, k: int, mask=None):
        """The query tree(s) (NODES: source side, destination side) over alive AND mask (a torch CUDA int64 tensor of words, or
        None) -> [(id, score)]: document ords for PATH, node_keys / rel_keys ords otherwise."""
        if not 1 <= k <= MAX_TOP_K:
            raise ValueError(f"top_k must be in 1..{MAX_TOP_K}")
        nodes, terms, keep = [], [], []
        for t in trees:
            self.compile(t, nodes, terms, keep)
        arr = (_lib.GraphNode * len(nodes))(*nodes)
        tarr = (_lib.GraphTerm * max(len(terms), 1))(*terms)
        from .segment import _stage

        mem, stream, alloc = _stage(self.device, mask is not None)
        ids, scores, count = alloc(k, np.uint32), alloc(k, np.float32), alloc(1, np.int32)
        try:
            _lib.check(_lib.load().nidx_graph_search(self.graph, arr, len(nodes), tarr, len(terms), kind, k, _lib.ptr(mask), mem, _lib.ptr(ids),
                                                     _lib.ptr(scores), _lib.ptr(count), stream))
        except _lib.NidxError as e:
            if e.code == -1:
                raise ValueError(str(e)) from e
            raise
        if mask is not None:
            ids, scores, count = ids.cpu().numpy().view(np.uint32), scores.cpu().numpy(), count.cpu().numpy()
        c = int(count[0])
        return [(int(i), float(s)) for i, s in zip(ids[:c], scores[:c])]

    def last_times(self):
        ms = (C.c_float * 4)()
        _lib.check(_lib.load().nidx_graph_last_times(self.graph, ms))
        return list(ms)

    # ---- the prefilter: resource_field_id terms of a Some (reader.rs:52-95) --------------------------------------------------------
    def prefilter_mask(self, prefilter):
        """A device Some of TextSearcher.prefilter -> this index's document mask (nidx_txt_join_mask): a relation matches when the
        text document of its (resource, field) matched, or when its field is a/metadata and some document of its resource matched."""
        import torch

        ix, bits, _ = prefilter.device_bits
        dev = torch.device("cuda", self.device)
        key = getattr(self, "_join", None)
        if key is None or key[0] is not ix:
            pos, res_of = {}, {}
            for ts, off in zip(ix.searcher.segments, ix.word_off):
                for i, d in enumerate(ts.docs):
                    pos.setdefault((_uuid.UUID(d.uuid).hex, d.field.lstrip("/")), 64 * off + i)
            for o, r in enumerate(ix.resource_ids):
                try:
                    res_of.setdefault(_uuid.UUID(r).hex, o)
                except ValueError:
                    pass
            doc_join = np.asarray([pos.get((d.rid, d.field), _lib.NIL) for d in self.docs], dtype=np.uint32)
            res_join = np.asarray([res_of.get(d.rid, _lib.NIL) if d.field == META_FIELD else _lib.NIL for d in self.docs], dtype=np.uint32)
            up = lambda a: torch.from_numpy(a.view(np.int32)).to(dev)   # noqa: E731
            self._join = (ix, up(doc_join), up(res_join))
        _, doc_join, res_join = self._join
        n_res = len(ix.resource_ids)
        res_bits = torch.zeros(max((n_res + 63) // 64, 1), dtype=torch.int64, device=dev)
        for ts, off in zip(ix.searcher.segments, ix.word_off):
            res_bits |= ts._gpu.resource_bits(bits[off: off + (ts.n_docs + 63) // 64], n_res)
        mask, _ = self.segment.join_mask(None, bits, bits.numel() * 64, doc_join, res_bits, n_res, res_join, _lib.NIDX_F_OR)
        return mask


class GraphSearcher:
    """NidxSearcher.GraphSearch over one shard's GraphIndex (reader.rs graph_search)."""

    def __init__(self, index: GraphIndex):
        self.index = index

    def search(self, request, prefilter=None):
        """GraphSearchRequest + vector.PrefilterResult (None: All) -> GraphSearchResponse."""
        from . import nidx_protos as P

        resp = P.GraphSearchResponse()
        if not request.HasField("query") or not request.query.HasField("path"):
            return resp
        kind = int(request.kind)
        if prefilter is not None and prefilter.kind == "none":
            return resp
        some = prefilter is not None and prefilter.kind == "some"
        pq = request.query.path
        trees = [with_prefilter(node_query(pq, "src"), some), with_prefilter(node_query(pq, "dst"), some)] if kind == NODES else \
            [with_prefilter(path_query(pq), some)]
        k = int(request.top_k)
        if k == 0:
            return resp
        mask = self.index.prefilter_mask(prefilter) if some else None
        hits = self.index.search(trees, kind, k, mask)
        return self.response(kind, hits)

    def response(self, kind: int, hits: list):
        from . import nidx_protos as P

        ix = self.index
        resp = P.GraphSearchResponse()
        for i, score in hits:
            resp.scores.append(score)
            if kind == NODES:
                v, t, s = ix.node_keys[i]
                resp.nodes.add(value=v, ntype=t, subtype=s)
            elif kind == RELATIONS:
                t, label = ix.rel_keys[i]
                resp.relations.add(relation_type=t, label=label)
            else:
                d = ix.docs[i]
                src = len(resp.nodes)
                resp.nodes.add(value=d.source[0], ntype=d.source[1], subtype=d.source[2])
                resp.nodes.add(value=d.target[0], ntype=d.target[1], subtype=d.target[2])
                rel = len(resp.relations)
                resp.relations.add(relation_type=d.rel_type, label=d.label)
                p = resp.graph.add(source=src, relation=rel, destination=src + 1, resource_field_id=f"{d.rid}/{d.field}")
                if d.metadata is not None:
                    p.metadata.ParseFromString(d.metadata)
                p.facets.extend(d.facets)
        return resp
