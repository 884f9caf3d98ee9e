"""Host-side mirror of ``nidx_vector``'s public interface over the CUDA library.

Same names, argument meaning and error behaviour as the reference's Rust API for the search hot
path (``nidx/nidx_vector/src/lib.rs:65-148``):

* ``VectorConfig``            config.rs:102-124 (+ the HNSW constants of hnsw/params.rs as fields)
* ``VectorSearchRequest``     request_types.rs:18-35
* ``VectorSearcher.open / .search``   lib.rs:124-139 -> searcher.rs:241-343
* ``VectorIndexer.index_elems / .merge``  lib.rs:69-117 -> segment.rs:92-286 (Elem level; protobuf
  ``Resource`` decoding is outside the hot path)
* ``OpenSegment``             segment.rs:428-567

All arithmetic (similarities, top-k, graph walks, graph construction) runs in ``libnidx_b200.so`` on
the GPU; this module only keeps the per-paragraph metadata (ids, labels) the reference keeps in
``paragraphs.bin`` and evaluates filter formulas to bitsets (inverted_index/paragraph.rs:124-186).
"""
from __future__ import annotations

import ctypes as C
import enum
import os
import uuid as _uuid
from dataclasses import dataclass, field
from typing import Iterable, Optional, Sequence, Union

import numpy as np

from . import _lib
from ._lib import NidxError
from .segment import VectorSegment, normalize


class Similarity(enum.Enum):  # config.rs:33-37 (+ L2: an extension, the reference has no Euclidean similarity)
    Cosine = "Cosine"
    Dot = "Dot"
    L2 = "L2"


class VectorCardinality(enum.Enum):  # config.rs
    Single = "Single"
    Multi = "Multi"


class FilterOperator(enum.Enum):  # nidx_types/src/prefilter.rs
    And = "And"
    Or = "Or"


@dataclass
class VectorConfig:
    """config.rs:102-124.  ``m/m0/ef_construction/ef_search`` are the compile-time constants of
    hnsw/params.rs:34-46 made per-index (defaults = the reference's values)."""
    dimension: int
    similarity: Similarity = Similarity.Cosine
    normalize_vectors: bool = False
    vector_cardinality: VectorCardinality = VectorCardinality.Single
    flags: list = field(default_factory=list)
    m: int = 30
    m0: int = 60
    ef_construction: int = 100
    ef_search: int = 30
    device: int = 0

    def _segment_kw(self) -> dict:
        """VectorSegment.create / open's keyword arguments."""
        return dict(similarity={Similarity.Cosine: _lib.NIDX_SIM_COSINE, Similarity.Dot: _lib.NIDX_SIM_DOT, Similarity.L2: _lib.NIDX_SIM_L2}[self.similarity],
                    m=self.m, m0=self.m0, ef_construction=self.ef_construction, ef_search=self.ef_search, device=self.device,
                    multi_vector=self.vector_cardinality == VectorCardinality.Multi)


# ---- nidx_types::query_language::BooleanExpression ----------------------------------------------
@dataclass(frozen=True)
class Literal:
    value: str


@dataclass(frozen=True)
class Not:
    operand: "BooleanExpression"


@dataclass(frozen=True)
class Operation:
    operator: str  # "and" | "or"
    operands: tuple


BooleanExpression = Union[Literal, Not, Operation]


@dataclass(frozen=True)
class FieldId:  # nidx_types/src/prefilter.rs
    resource_id: _uuid.UUID
    field_id: Optional[str] = None  # e.g. "/a/title"


class PrefilterResult:
    """nidx_types/src/prefilter.rs: All | None | Some(fields).  A Some made on the device keeps its sets in HBM, in two parts: the
    text part `device_bits` (TextSearcher.prefilter: (the text index's prefilter state, the bits, the match count), or None) and the
    resource part `resources` (combine: (the JsonIndex, its resource bits), or None), combined under OR when `op_or`, else AND.
    Its `fields` are listed only when read; VectorSearcher.search and TextSearcher.json_masks hand the parts on without leaving
    the device."""

    def __init__(self, kind: str, fields: Sequence[FieldId] = (), device_bits=None, resources=None, op_or: bool = False):
        self.kind, self.device_bits, self.resources, self.op_or = kind, device_bits, resources, op_or
        self._fields = None if device_bits is not None or resources is not None else list(fields)

    @property
    def fields(self) -> list:
        if self._fields is None:
            index, bits, _ = self.device_bits
            self._fields = index.fields(bits)
        return self._fields

    @property
    def on_device(self) -> bool:
        """A Some whose sets are in HBM."""
        return self.kind == "some" and (self.device_bits is not None or self.resources is not None)

    @classmethod
    def from_device(cls, index, bits, matching: int):
        return cls("some", device_bits=(index, bits, matching))

    def combine(self, json_index, res_bits, found: int, op_or: bool) -> "PrefilterResult":
        """PrefilterResult::combine (nidx_types/src/prefilter.rs:49-92) of this text result with the resource set of a JSON prefilter
        (res_bits over json_index.resource_ids, in HBM, from `found` matched JSON documents) under OR (op_or) or AND.  A Some stays on
        the device: its text part, if any, and the resource part, which the hand-offs combine."""
        text = self.device_bits if self.kind == "some" else None
        if self.kind == "some" and text is None:
            raise ValueError("json_filter needs the device prefilter")
        if found == 0:   # an empty set: the text result under OR, None under AND
            return self if op_or else PrefilterResult.none()
        if (self.kind == "none" and not op_or) or (self.kind == "all" and op_or):
            return self
        # None under OR is the resource set alone; All under AND is the resource set ANDed with every field
        return PrefilterResult("some", device_bits=text, resources=(json_index, res_bits), op_or=op_or and text is not None)

    @classmethod
    def all(cls):
        return cls("all")

    @classmethod
    def none(cls):
        return cls("none")

    @classmethod
    def some(cls, fields):
        return cls("some", fields)


@dataclass
class VectorSearchRequest:  # request_types.rs:18-35 (Default: min_score 0.0, with_duplicates false)
    vector: Sequence[float] = ()
    result_per_page: int = 0
    with_duplicates: bool = False
    vector_set: str = ""
    min_score: float = 0.0
    filtering_formula: Optional[BooleanExpression] = None
    segment_filtering_formula: Optional[BooleanExpression] = None
    filter_operator: FilterOperator = FilterOperator.And


@dataclass
class DocumentScored:  # nodereader.proto:126-135
    doc_id: str
    score: float
    labels: list
    metadata: Optional[bytes]


@dataclass
class VectorSearchResponse:
    documents: list


@dataclass
class Elem:  # segment.rs Elem {key, vectors, metadata, labels}
    key: str
    vectors: Sequence[Sequence[float]]
    labels: Sequence[str] = ()
    metadata: Optional[bytes] = None


# ---- formula.rs ------------------------------------------------------------------------------------
@dataclass
class _KeyPrefixSet:
    keys: frozenset


def _map_expression(e):  # query_io.rs:20-50
    return e


def field_key(field_id: str) -> Optional[bytes]:
    """utils.rs:80-117 FieldKey::from_field_id: 16 raw uuid bytes [+ type + "/" + name]."""
    parts = field_id.split("/")
    try:
        rid = _uuid.UUID(parts[0])
    except ValueError:
        return None
    if len(parts) >= 2:
        if len(parts) >= 3:
            return rid.bytes + parts[1].encode() + b"/" + parts[2].encode()
        return None
    return rid.bytes


def _labels_key(label: str) -> str:  # inverted_index/paragraph.rs:64-66
    return label[1:] + "/"


class OpenSegment:
    """segment.rs OpenSegment: device-resident vectors + graph (``segment``, a VectorSegment; None for a host-only view),
    host-resident paragraph metadata."""

    def __init__(self, config: VectorConfig, segment: Optional[VectorSegment], keys, labels, metadata, first_vec, tags=frozenset()):
        self.config = config
        self.segment = segment
        self.keys, self.labels, self.metadata = list(keys), [tuple(l) for l in labels], list(metadata)
        self.first_vec = np.asarray(first_vec, dtype=np.uint32)  # [n_par + 1]
        self.records = len(self.keys)
        self.tags = frozenset(tags)
        self.alive = np.ones(self.records, dtype=bool)
        self._field_keys = [field_key(k) for k in self.keys]
        self._label_index: dict = {}
        for p, ls in enumerate(self.labels):
            for l in ls:
                self._label_index.setdefault(_labels_key(l), []).append(p)
        self._field_index: dict = {}
        for p, fk in enumerate(self._field_keys):
            if fk is not None:
                self._field_index.setdefault(fk, []).append(p)
        if segment is not None:   # the label and field indexes go to the library, so that filter formulas are evaluated on the device
            for which, index in ((_lib.NIDX_INV_LABELS, {k.encode(): v for k, v in self._label_index.items()}), (_lib.NIDX_INV_FIELDS, self._field_index)):
                keys = sorted(index)
                segment.set_inverted_index(which, keys, [sorted(index[k]) for k in keys])

    @property
    def _h(self):
        """The C handle of the owned VectorSegment, for callers that pass it to the C ABI themselves.  It stays owned by `segment`,
        which alone closes it."""
        return self.segment._h

    # -- filter formulas for the device (formula.rs:40-100 -> nidx_filter_node, pre-order) ----------
    def formula_nodes(self, clauses, operator_and=True):
        """-> (ctypes array of FilterNode, n, keep-alive list).  Literal -> LABEL(labels_key), _KeyPrefixSet -> KEYS(field keys),
        Not / Operation -> NOT / AND / OR; several clauses are wrapped in the formula's operator."""
        flat, keep = [], []

        def atom(kind, keys):
            bufs = [C.create_string_buffer(k, max(len(k), 1)) for k in keys]      # raw bytes: field keys start with 16 uuid bytes, NULs included
            arr = (C.c_void_p * max(len(keys), 1))(*[C.addressof(b) for b in bufs])
            lens = (C.c_uint32 * max(len(keys), 1))(*[len(k) for k in keys])
            keep.extend([arr, lens, bufs])
            flat.append((kind, len(keys), arr, lens))

        def walk(c):
            if isinstance(c, Literal):
                atom(_lib.NIDX_F_LABEL, [_labels_key(c.value).encode()])
            elif isinstance(c, _KeyPrefixSet):
                atom(_lib.NIDX_F_KEYS, [fk for fk in (field_key(f) for f in sorted(c.keys)) if fk is not None])
            elif isinstance(c, Not):
                flat.append((_lib.NIDX_F_NOT, 1, None, None))
                walk(c.operand)
            elif isinstance(c, Operation):
                flat.append((_lib.NIDX_F_AND if c.operator == "and" else _lib.NIDX_F_OR, len(c.operands), None, None))
                for o in c.operands:
                    walk(o)
            else:
                raise TypeError(f"unknown clause {c!r}")

        clauses = list(clauses)
        if len(clauses) != 1:
            flat.append((_lib.NIDX_F_AND if operator_and else _lib.NIDX_F_OR, len(clauses), None, None))
        for c in clauses:
            walk(c)
        nodes = (_lib.FilterNode * len(flat))()
        for i, (kind, n, arr, lens) in enumerate(flat):
            nodes[i].kind, nodes[i].n = kind, n
            if arr is not None:
                nodes[i].keys, nodes[i].key_len = arr, lens
        return nodes, len(flat), keep

    def device_filter(self, clauses, operator_and=True):
        """nidx_vec_filter: the formula's bitset AND the alive set, computed on the device -> (bool mask over paragraphs, matching)."""
        nodes, n, keep = self.formula_nodes(clauses, operator_and)
        words = np.zeros((self.records + 63) // 64, dtype=np.uint64)
        matching = self.segment.filter(nodes, n, words)
        return np.unpackbits(words.view(np.uint8), bitorder="little")[: self.records].astype(bool), matching

    # -- lifecycle -----------------------------------------------------------------------------
    @classmethod
    def create(cls, elems: Sequence[Elem], config: VectorConfig, tags=frozenset(), build_graph=True, seed=2, max_batch=4096):
        """segment::create (segment.rs:199-286): data store + HNSW (GPU build)."""
        _lib.require_device()
        dim = config.dimension
        vecs, par_of, first = [], [], [0]
        for p, e in enumerate(elems):
            if config.vector_cardinality == VectorCardinality.Single and len(e.vectors) != 1:
                raise NidxError(-1, "single-vector index got an element with several vectors")
            for v in e.vectors:
                if len(v) != dim:
                    raise NidxError(-1, f"InconsistentDimensions: index_config {dim}, vector {len(v)}")
                vecs.append(np.asarray(v, dtype=np.float32))
                par_of.append(p)
            first.append(len(vecs))
        arr = np.stack(vecs).astype(np.float32) if vecs else np.zeros((0, dim), dtype=np.float32)
        if config.normalize_vectors:  # indexer.rs:94-146 normalises at index time (utils.rs:20-23)
            normalize(arr, config.device)
        segment = VectorSegment.create(arr, dim, **config._segment_kw(), paragraph_of=np.asarray(par_of, dtype=np.uint32) if par_of else None)
        seg = cls(config, segment, [e.key for e in elems], [e.labels for e in elems], [e.metadata for e in elems], first, tags)
        seg.host_vectors = arr
        if build_graph and len(arr):
            segment.build_hnsw(seed, max_batch)
        return seg

    def save(self, directory: str):
        """Write the segment in the reference's data-store-v2 layout: vectors.bin, hnsw.graph, hnsw.edges (the library,
        segment_io.hpp) and paragraphs.bin / paragraphs.pos (paragraph_store.py).  The inverted indexes (index.map, field.fst,
        label.fst) are not written: `open` rebuilds them from the paragraphs, as the reference's `build_indexes` does
        (segment.rs:183)."""
        from . import paragraph_store as PS

        self.segment.save(directory)
        PS.write_paragraphs(directory, ((self.keys[p], self.labels[p], self.metadata[p], int(self.first_vec[p]), int(self.first_vec[p + 1] - self.first_vec[p]))
                                        for p in range(self.records)))

    @classmethod
    def open(cls, config: VectorConfig, directory: str, tags=frozenset()):
        """segment::open (segment.rs:39-90) for a data-store-v2 directory: vectors and graph go to the device, ids / labels /
        metadata of the paragraphs stay on the host."""
        from . import paragraph_store as PS

        _lib.require_device()
        paragraphs = PS.read_paragraphs(directory)
        first = [p[3] for p in paragraphs] + [paragraphs[-1][3] + paragraphs[-1][4] if paragraphs else 0]
        for i, p in enumerate(paragraphs):
            if p[3] + p[4] != first[i + 1]:
                raise NidxError(-1, f"paragraph {i} does not own a contiguous vector range")
        record = np.dtype([("vector", np.float32, (config.dimension,)), ("paragraph", np.uint32)])
        stored = np.fromfile(os.path.join(directory, "vectors.bin"), dtype=record)
        if len(stored) != first[-1]:
            raise NidxError(-1, f"vectors.bin holds {len(stored)} vectors, paragraphs.bin accounts for {first[-1]}")
        segment = VectorSegment.open(directory, config.dimension, **config._segment_kw())
        seg = cls(config, segment, [p[0] for p in paragraphs], [p[1] for p in paragraphs], [p[2] for p in paragraphs], first, tags)
        seg.host_vectors = np.ascontiguousarray(stored["vector"])
        return seg

    def close(self):
        if self.segment is not None:
            self.segment.close()

    # -- deletions (segment.rs:428-445, lib.rs:166-200) -------------------------------------------
    def apply_deletions(self, deleted_keys: Iterable[str]):
        for k in deleted_keys:
            fk = field_key(k)
            if fk is None:
                continue
            for stored, paragraphs in self._field_index.items():  # prefix match (ids_for_deletion_key)
                if stored.startswith(fk):
                    self.alive[paragraphs] = False
        bits = np.packbits(self.alive, bitorder="little")
        words = np.zeros((self.records + 63) // 64 * 8, dtype=np.uint8)
        words[: len(bits)] = bits
        self.segment.set_alive(words.view(np.uint64))

    # -- filters (inverted_index/paragraph.rs:124-186) ---------------------------------------------
    def _clause(self, clause) -> np.ndarray:
        out = np.zeros(self.records, dtype=bool)
        if isinstance(clause, Literal):
            prefix = _labels_key(clause.value)
            for k, ps in self._label_index.items():
                if k.startswith(prefix):
                    out[ps] = True
            return out
        if isinstance(clause, _KeyPrefixSet):
            for fid in clause.keys:
                fk = field_key(fid)
                if fk is not None and fk in self._field_index:  # exact get (fst_index.rs:71-73)
                    out[self._field_index[fk]] = True
            return out
        if isinstance(clause, Not):
            return ~self._clause(clause.operand)
        if isinstance(clause, Operation):
            parts = [self._clause(c) for c in clause.operands]
            acc = parts[0]
            for p in parts[1:]:
                acc = (acc & p) if clause.operator == "and" else (acc | p)
            return acc
        raise TypeError(f"unknown clause {clause!r}")

    def filter_bitset(self, clauses, operator_and=True) -> Optional[np.ndarray]:
        if not clauses:
            return None
        acc = self._clause(clauses[0])
        for c in clauses[1:]:
            acc = (acc & self._clause(c)) if operator_and else (acc | self._clause(c))
        return acc

    # -- search (segment.rs:477-567) ---------------------------------------------------------------
    def search(self, query, clauses, operator_and, with_duplicates, top_k, min_score, method=_lib.NIDX_METHOD_AUTO, ef=0):
        """-> (vector addrs [<=k], scores) for one query."""
        ids, scores, counts = self.search_batch(np.asarray(query, dtype=np.float32)[None, :], top_k, min_score, with_duplicates, clauses, operator_and,
                                                method, ef)
        c = int(counts[0])
        return ids[0, :c], scores[0, :c]

    def search_batch(self, queries: np.ndarray, top_k, min_score=0.0, with_duplicates=False, clauses=(), operator_and=True,
                     method=_lib.NIDX_METHOD_AUTO, ef=0):
        queries = np.ascontiguousarray(queries, dtype=np.float32)
        if queries.shape[1] != self.config.dimension:
            raise NidxError(-1, f"InconsistentDimensions: index_config {self.config.dimension}, vector {queries.shape[1]}")
        # a formula goes to the library as it is: postings -> bitset -> algebra -> AND alive -> count, all in HBM (segment.rs:516-534)
        clauses = list(clauses)
        nodes, _, keep = self.formula_nodes(clauses, operator_and) if clauses else (None, 0, None)
        return self.segment.search(queries, top_k, ef, min_score, with_duplicates, method, formula=nodes)

    def search_prefiltered(self, query, prefilter, formula, operator_and, with_duplicates, top_k, min_score, method=_lib.NIDX_METHOD_AUTO, ef=0):
        """search() restricted by a prefilter made on the device (a PrefilterResult with device_bits and / or resources) instead of a
        key set: the paragraphs of the text part's documents (through the text index's join table) and of the resource part's
        resources (every field of theirs, with or without a text document), combined under the result's operator, then with
        `formula` under the operator as search() combines its clauses (nidx_vec_prefilter_bits), go to the search as a bitset that
        never leaves the device."""
        import torch

        nodes, _, keep = self.formula_nodes([formula]) if formula is not None else (None, 0, None)
        doc_bits = join = res_bits = ranges = None
        n_docs = n_res = 0
        if prefilter.device_bits is not None:
            index, doc_bits, _ = prefilter.device_bits
            join, n_docs = index.join(self), index.n_docs_total()
        if prefilter.resources is not None:
            json_index, res_bits = prefilter.resources
            ranges, n_res = self.json_ranges(json_index), len(json_index.resource_ids)
        bits, matching = self.segment.prefilter_bits(doc_bits, join, n_docs, res_bits, ranges, n_res, self.records, nodes,
                                                     _lib.NIDX_F_AND if operator_and else _lib.NIDX_F_OR,
                                                     _lib.NIDX_F_OR if prefilter.op_or else _lib.NIDX_F_AND)
        if matching == 0:   # segment.rs:532-534: nothing can match
            return np.zeros(0, dtype=np.uint32), np.zeros(0, dtype=np.float32)
        q = torch.as_tensor(np.asarray(query, dtype=np.float32)[None, :]).to(torch.device("cuda", self.config.device))
        ids, scores, counts = self.segment.search(q, top_k, ef, min_score, with_duplicates, method, filter_bits=bits, filter_matching=matching)
        c = int(counts[0].item())
        return ids[0, :c].cpu().numpy().view(np.uint32), scores[0, :c].cpu().numpy()

    def json_ranges(self, json_index):
        """uint64 [n_res][2] on the device: the postings of the field index keys that start with each JSON resource's 16 uuid bytes
        (one contiguous run of the sorted keys), cached per JSON index."""
        import bisect

        import torch

        cached = getattr(self, "_json_ranges", None)
        if cached is not None and cached[0] is json_index:
            return cached[1]
        keys = sorted(self._field_index)
        post_off = np.zeros(len(keys) + 1, dtype=np.uint64)
        post_off[1:] = np.cumsum([len(self._field_index[k]) for k in keys])
        ranges = np.zeros((max(len(json_index.resource_ids), 1), 2), dtype=np.uint64)
        for r, rid in enumerate(json_index.resource_ids):
            try:
                prefix = _uuid.UUID(rid).bytes
            except ValueError:
                continue
            lo = bisect.bisect_left(keys, prefix)
            hi = bisect.bisect_left(keys, (int.from_bytes(prefix, "big") + 1).to_bytes(16, "big")) if prefix != b"\xff" * 16 else len(keys)
            ranges[r] = post_off[lo], post_off[hi]
        t = torch.from_numpy(ranges.view(np.int64)).to(torch.device("cuda", self.config.device))
        self._json_ranges = (json_index, t)
        return t

    def _raw_search(self, queries, k, filter_bits):
        """exact scan restricted to a paragraph bitset, no min_score: per (query, paragraph) the best vector's similarity."""
        return self.segment.search(queries, k, 0, float(np.finfo(np.float32).min), True, _lib.NIDX_METHOD_BRUTE, filter_bits=filter_bits)

    def paragraph_of(self, vector_addr: int) -> int:
        return int(np.searchsorted(self.first_vec, vector_addr, side="right") - 1)


def _segment_matches(expr, tags) -> bool:  # searcher.rs segment_matches
    if isinstance(expr, Literal):
        return expr.value in tags
    if isinstance(expr, Not):
        return not _segment_matches(expr.operand, tags)
    vals = [_segment_matches(o, tags) for o in expr.operands]
    return all(vals) if expr.operator == "and" else any(vals)


class _Fssc:
    """searcher.rs:150-199 fixed-size sorted collection keyed by paragraph id."""

    def __init__(self, size, with_duplicates):
        self.size, self.with_duplicates = size, with_duplicates
        self.seen, self.buff = set(), {}

    def add(self, pid, score, payload, vector_bytes):
        if not self.with_duplicates:
            if vector_bytes in self.seen:
                return
            self.seen.add(vector_bytes)
        if len(self.buff) == self.size:
            smaller = [(s, k) for k, (s, _) in self.buff.items() if score > s]
            if smaller:
                _, victim = min(smaller, key=lambda t: t[0])
                del self.buff[victim]
                self.buff.setdefault(pid, (score, payload))
        else:
            self.buff.setdefault(pid, (score, payload))

    def result(self):
        return sorted(((s, k, p) for k, (s, p) in self.buff.items()), key=lambda t: -t[0])


class VectorSearcher:
    """lib.rs:124-139 + searcher.rs:241-343."""

    def __init__(self, config: VectorConfig, segments: Sequence[OpenSegment]):
        self.config, self.open_segments = config, list(segments)

    @classmethod
    def open(cls, config: VectorConfig, segments: Sequence[tuple], deletions: Sequence[tuple] = ()):
        """segments: [(OpenSegment, seq)], deletions: [(key, seq)]; a deletion applies to a segment
        iff del.seq > segment.seq (lib.rs:188-199)."""
        _lib.require_device()
        opened = []
        for seg, seq in segments:
            dels = [k for k, dseq in deletions if dseq > seq]
            if dels:
                seg.apply_deletions(dels)
            opened.append(seg)
        return cls(config, opened)

    def search(self, request: VectorSearchRequest, prefilter: PrefilterResult = None, method=_lib.NIDX_METHOD_AUTO, ef=0) -> VectorSearchResponse:
        prefilter = prefilter or PrefilterResult.all()
        multi = self.config.vector_cardinality == VectorCardinality.Multi
        clauses = []
        if prefilter.kind == "some" and prefilter.resources is None and (multi or prefilter.device_bits is None):  # searcher.rs:300-314
            clauses.append(_KeyPrefixSet(frozenset(f"{f.resource_id.hex}{f.field_id}" if f.field_id else f.resource_id.hex for f in prefilter.fields)))
        if request.filtering_formula is not None:
            clauses.append(_map_expression(request.filtering_formula))
        operator_and = request.filter_operator == FilterOperator.And
        query = np.asarray(request.vector, dtype=np.float32)
        if self.config.normalize_vectors and self.config.vector_cardinality != VectorCardinality.Multi:  # searcher.rs:246-252, utils.rs:20-23
            query = normalize(query.copy(), self.config.device)
        if (len(query) != self.config.dimension) if not multi else (len(query) % self.config.dimension != 0 or len(query) == 0):
            raise NidxError(-1, f"InconsistentDimensions: index_config {self.config.dimension}, vector {len(query)}")
        k = request.result_per_page
        if self.config.vector_cardinality == VectorCardinality.Multi:
            if prefilter.resources is not None:
                raise ValueError("json_filter is not supported on a multi-vector vectorset")
            return self._search_multi_vector(request, clauses, operator_and, prefilter, method, ef)
        fssc = _Fssc(k, request.with_duplicates)
        if k > 0 and prefilter.kind != "none":
            for seg in self.open_segments:
                if request.segment_filtering_formula is not None and not _segment_matches(request.segment_filtering_formula, seg.tags):
                    continue
                if prefilter.on_device:
                    addrs, scores = seg.search_prefiltered(query, prefilter, request.filtering_formula, operator_and, request.with_duplicates, k,
                                                           request.min_score, method, ef)
                else:
                    addrs, scores = seg.search(query, clauses, operator_and, request.with_duplicates, k, request.min_score, method, ef)
                for a, s in zip(addrs, scores):
                    p = seg.paragraph_of(int(a))
                    vb = (id(seg), int(a)) if request.with_duplicates else self._vector_bytes(seg, int(a))
                    fssc.add(seg.keys[p], float(s), (seg, p), vb)
        docs = [DocumentScored(pid, score, list(seg.labels[p]), seg.metadata[p]) for score, pid, (seg, p) in fssc.result()]
        return VectorSearchResponse(docs)

    def _search_multi_vector(self, request, clauses, operator_and, prefilter, method, ef) -> VectorSearchResponse:
        """searcher.rs:345-394 + multivector.rs:34-46 (MaxSim).  Every query vector is searched on its own
        (duplicates allowed, no min_score, at least 10 results), the paragraphs found are re-scored with
        sum_q max(0, max_v sim(v, q)) -- the per-paragraph maxima come from one exact-scan call restricted to
        the candidate paragraphs -- then min_score (strict >), sort, truncate."""
        d = self.config.dimension
        k = request.result_per_page
        qv = np.asarray(request.vector, dtype=np.float32).reshape(-1, d)
        if self.config.normalize_vectors:
            qv = normalize(qv.copy(), self.config.device)
        if k <= 0 or prefilter.kind == "none":
            return VectorSearchResponse([])
        first_k = max(k, 10)
        scored = []
        for seg in self.open_segments:
            if request.segment_filtering_formula is not None and not _segment_matches(request.segment_filtering_formula, seg.tags):
                continue
            ids, _, counts = seg.search_batch(qv, first_k, float(np.finfo(np.float32).min), True, clauses, operator_and, method, ef)
            cand = sorted({seg.paragraph_of(int(a)) for qi in range(len(qv)) for a in ids[qi, : counts[qi]]})
            if not cand:
                continue
            mask = np.zeros(seg.records, dtype=bool)
            mask[cand] = True
            bits = np.zeros((seg.records + 63) // 64 * 8, dtype=np.uint8)
            pb = np.packbits(mask, bitorder="little")
            bits[: len(pb)] = pb
            rid, rsc, rcnt = seg._raw_search(qv, len(cand), bits.view(np.uint64))
            maxsim = {p: np.float32(0.0) for p in cand}
            for qi in range(len(qv)):
                best = {seg.paragraph_of(int(a)): np.float32(sc) for a, sc in zip(rid[qi, : rcnt[qi]], rsc[qi, : rcnt[qi]])}
                for p in cand:
                    maxsim[p] = np.float32(maxsim[p] + max(np.float32(0.0), best.get(p, np.float32(0.0))))
            scored += [(float(sc), seg, p) for p, sc in maxsim.items() if sc > request.min_score]
        scored.sort(key=lambda t: -t[0])
        docs = [DocumentScored(seg.keys[p], sc, list(seg.labels[p]), seg.metadata[p]) for sc, seg, p in scored[:k]]
        return VectorSearchResponse(docs)

    @staticmethod
    def _vector_bytes(seg: OpenSegment, addr: int) -> bytes:
        # Fssc's exact-duplicate test hashes the raw vector bytes (searcher.rs:175-183); the host copy
        # kept at create/open time plays the role of the reference's mmap of vectors.bin.
        return seg.host_vectors[addr].tobytes()


class VectorIndexer:
    """lib.rs:65-117 at Elem granularity."""

    @staticmethod
    def index_elems(elems: Sequence[Elem], config: VectorConfig, tags=frozenset(), **kw) -> OpenSegment:
        return OpenSegment.create(elems, config, tags, **kw)

    @staticmethod
    def merge(config: VectorConfig, segments: Sequence[tuple], deletions: Sequence[tuple] = (), **kw) -> OpenSegment:
        """lib.rs:97-117 + segment.rs:92-197: open the segments applying deletions by sequence (a deletion applies to a
        segment iff del.seq > segment.seq), copy the alive paragraphs -- segment with most stored records first -- into one
        data store.  If that first segment has no deletions its HNSW is reused (its vector addresses are a prefix of the
        merged store's) and only the other segments' vectors are inserted (merge_indexes, segment.rs:143-167); otherwise the
        graph is built from scratch.  Both on the GPU."""
        opened = []
        for seg, seq in segments:
            dels = [k for k, dseq in deletions if dseq > seq]
            if dels:
                seg.apply_deletions(dels)
            opened.append(seg)
        opened.sort(key=lambda s: -int(s.records))
        if any(s.tags != opened[0].tags for s in opened):
            raise NidxError(-1, "InconsistentMergeSegmentTags")
        elems = []
        for seg in opened:
            for p in np.nonzero(seg.alive)[0]:
                a, b = int(seg.first_vec[p]), int(seg.first_vec[p + 1])
                elems.append(Elem(seg.keys[p], [seg.host_vectors[i] for i in range(a, b)], seg.labels[p], seg.metadata[p]))
        merged_cfg = VectorConfig(**{**config.__dict__, "normalize_vectors": False})   # vectors were normalised when first indexed
        first = opened[0]
        reuse = bool(first.alive.all()) and len(first.host_vectors) > 0
        if reuse:
            try:
                g = first.segment.get_graph()
            except NidxError:                       # the first segment was created without a graph
                reuse = False
        if reuse:
            out = OpenSegment.create(elems, merged_cfg, frozenset(first.tags), build_graph=False)
            rows = max(int(g["upper_rows"]), 1)
            out.segment.extend_hnsw(len(first.host_vectors), g["level"], g["adj0"], g["adjU"][:rows], g["w0"], g["wU"][:rows], g["entry_node"], g["entry_layer"],
                                    seed=kw.get("seed", 2), max_batch=kw.get("max_batch", 4096))
        else:
            out = OpenSegment.create(elems, merged_cfg, frozenset(first.tags), **kw)
        out.config = config
        return out
