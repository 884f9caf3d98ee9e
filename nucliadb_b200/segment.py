"""Thin object wrappers over the C ABI handles (``include/nidx_b200.h``).

``VectorSegment``  = nidx_vec_segment: vectors + HNSW graph resident in HBM, exact scan / HNSW search /
                     GPU graph build.  Accepts numpy arrays (host path: copies inside the call) or torch
                     CUDA tensors (device path: zero copy, asynchronous on the current torch stream).
``TextSegment``    = nidx_txt_segment: postings resident in HBM, BM25 top-k.
torch is used for device memory and streams only.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import numpy as np

from . import _lib
from ._lib import NIL, NidxError, TxtSearchParams, VecConfig, VecSearchParams, check, ptr


def _is_torch(x) -> bool:
    return hasattr(x, "data_ptr") and hasattr(x, "is_cuda")


def _torch_stream(device: int):
    import torch

    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


_SIGNED = {"uint32": "int32", "uint64": "int64"}   # torch has no usable unsigned 32 / 64-bit tensors


def _stage(device: int, on_device: bool, stream: Optional[int] = None):
    """Where a call's buffers live -> (mem, stream, alloc).  On the device the call is asynchronous on the current torch stream and
    alloc(shape, numpy dtype) returns an uninitialised torch CUDA tensor of the same width (uint32 -> int32, uint64 -> int64).  On
    the host the call runs on `stream` (a cudaStream_t as int; None = the default stream) and alloc returns a numpy array, zeroed
    with zero=True (device outputs are left to the kernel: no fill is launched)."""
    if on_device:
        import torch

        def alloc(shape, dtype, zero=False):
            name = np.dtype(dtype).name
            return torch.empty(shape, dtype=getattr(torch, _SIGNED.get(name, name)), device=torch.device("cuda", device))

        return _lib.NIDX_MEM_DEVICE, _torch_stream(device), alloc
    return _lib.NIDX_MEM_HOST, C.c_void_p(stream) if stream else None, lambda shape, dtype, zero=False: (np.zeros if zero else np.empty)(shape, dtype)


def normalize(vectors: np.ndarray, device: int = 0) -> np.ndarray:
    """utils::normalize_vector (nidx_vector/src/utils.rs:20-23) through nidx_normalize_vectors, in place: one vector [d] or rows
    [n][d] of a C-contiguous float32 array.  The f32 fold runs sequentially on the device, bit-identical to the reference's."""
    assert vectors.dtype == np.float32 and vectors.flags.c_contiguous   # else the rows below would be a copy
    if vectors.size:
        rows = vectors.reshape(-1, vectors.shape[-1])
        check(_lib.require_device().nidx_normalize_vectors(device, ptr(rows), rows.shape[0], rows.shape[1], rows.shape[1], _lib.NIDX_MEM_HOST, None))
    return vectors


class VectorSegment:
    def __init__(self, handle, cfg: VecConfig):
        self._h, self.cfg = handle, cfg

    # ---- lifecycle ----------------------------------------------------------------------------------
    @classmethod
    def create(cls, vectors, dimension: int, similarity=_lib.NIDX_SIM_COSINE, m=30, m0=60, ef_construction=100, ef_search=30, device=0,
               multi_vector=False, paragraph_of: Optional[np.ndarray] = None) -> "VectorSegment":
        L = _lib.require_device()
        cfg = VecConfig(dimension, similarity, int(multi_vector), m, m0, ef_construction, ef_search, device)
        h = C.c_void_p()
        if _is_torch(vectors):
            assert vectors.is_cuda and vectors.is_contiguous() and vectors.dtype.is_floating_point
            n, ld = vectors.shape
            mem = _lib.NIDX_MEM_DEVICE
        else:
            vectors = np.ascontiguousarray(vectors, dtype=np.float32)
            n, ld = vectors.shape if vectors.ndim == 2 else (0, dimension)
            mem = _lib.NIDX_MEM_HOST
        par = None if paragraph_of is None else np.ascontiguousarray(paragraph_of, dtype=np.uint32)
        check(L.nidx_vec_create(C.byref(cfg), ptr(vectors) if n else None, n, ld, mem, ptr(par), C.byref(h)))
        return cls(h, cfg)

    @classmethod
    def open(cls, directory: str, dimension: int, similarity=_lib.NIDX_SIM_COSINE, m=30, m0=60, ef_construction=100, ef_search=30, device=0,
             multi_vector=False) -> "VectorSegment":
        L = _lib.require_device()
        cfg = VecConfig(dimension, similarity, int(multi_vector), m, m0, ef_construction, ef_search, device)
        h = C.c_void_p()
        check(L.nidx_vec_open(C.byref(cfg), directory.encode(), C.byref(h)))
        return cls(h, cfg)

    def save(self, directory: str):
        check(_lib.load().nidx_vec_save(self._h, directory.encode()))

    def close(self):
        if self._h is not None:
            _lib.load().nidx_vec_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __len__(self):
        return int(_lib.load().nidx_vec_len(self._h))

    # ---- graph ----------------------------------------------------------------------------------------
    def build_hnsw(self, seed=2, max_batch=4096):
        check(_lib.load().nidx_vec_build_hnsw(self._h, seed, max_batch, None))

    def extend_hnsw(self, n_existing, level, adj0, adjU, w0, wU, entry_node, entry_layer, seed=2, max_batch=4096):
        """Reuse the graph of the first n_existing vectors and insert the rest (segment.rs:143-167)."""
        level = np.ascontiguousarray(level, dtype=np.uint8)
        adj0 = np.ascontiguousarray(adj0, dtype=np.uint32)
        adjU = np.ascontiguousarray(adjU, dtype=np.uint32)
        w0 = np.ascontiguousarray(w0, dtype=np.float32)
        wU = np.ascontiguousarray(wU, dtype=np.float32)
        check(_lib.load().nidx_vec_extend_hnsw(self._h, n_existing, ptr(level), ptr(adj0), ptr(w0), ptr(adjU), ptr(wU), entry_node, entry_layer, seed,
                                               max_batch, None))

    def graph_dims(self):
        s0, su, rows, en, el = C.c_int32(), C.c_int32(), C.c_uint64(), C.c_uint32(), C.c_uint32()
        check(_lib.load().nidx_vec_graph_dims(self._h, C.byref(s0), C.byref(su), C.byref(rows), C.byref(en), C.byref(el)))
        return s0.value, su.value, rows.value, en.value, el.value

    def set_graph(self, level, adj0, adjU, w0=None, wU=None):
        level = np.ascontiguousarray(level, dtype=np.uint8)
        adj0 = np.ascontiguousarray(adj0, dtype=np.uint32)
        adjU = np.ascontiguousarray(adjU, dtype=np.uint32)
        w0 = None if w0 is None else np.ascontiguousarray(w0, dtype=np.float32)
        wU = None if wU is None else np.ascontiguousarray(wU, dtype=np.float32)
        check(_lib.load().nidx_vec_set_graph(self._h, ptr(level), ptr(adj0), ptr(w0), ptr(adjU), ptr(wU)))

    def get_graph(self):
        """-> dict(level, adj0, w0, adjU, wU, entry_node, entry_layer, s0, su)."""
        s0, su, rows, en, el = self.graph_dims()
        n = len(self)
        level = np.empty(n, dtype=np.uint8)
        adj0 = np.empty((n, s0), dtype=np.uint32)
        w0 = np.empty((n, s0), dtype=np.float32)
        adjU = np.full((max(rows, 1), su), NIL, dtype=np.uint32)
        wU = np.zeros((max(rows, 1), su), dtype=np.float32)
        check(_lib.load().nidx_vec_get_graph(self._h, ptr(level), ptr(adj0), ptr(w0), ptr(adjU), ptr(wU)))
        return dict(level=level, adj0=adj0, w0=w0, adjU=adjU, wU=wU, entry_node=en, entry_layer=el, s0=s0, su=su, upper_rows=rows)

    def set_alive(self, alive_bits: Optional[np.ndarray]):
        check(_lib.load().nidx_vec_set_alive(self._h, ptr(alive_bits), _lib.NIDX_MEM_HOST))

    def set_paragraph_keys(self, keys: Optional[np.ndarray]):
        """64-bit keys of the paragraph ids, for the cross-segment de-duplication of a sharded search (Fssc, searcher.rs:150-199)."""
        keys = None if keys is None else np.ascontiguousarray(keys, dtype=np.uint64)
        check(_lib.load().nidx_vec_set_paragraph_keys(self._h, ptr(keys)))

    # ---- filters (ParagraphInvertedIndexes, inverted_index/paragraph.rs) ----------------------------------
    def set_inverted_index(self, which, keys, postings):
        """ParagraphInvertedIndexes::build (inverted_index/paragraph.rs:74-106) for one index (_lib.NIDX_INV_*): keys (bytes) sorted
        bytewise as in the fst, and for each key its paragraphs, ascending.  The postings go to HBM, where filter formulas are
        evaluated."""
        key_bytes, key_off = _pack_keys(keys)
        post_off = np.zeros(len(keys) + 1, dtype=np.uint64)
        post_off[1:] = np.cumsum([len(p) for p in postings]) if len(keys) else []
        flat = np.asarray([p for ps in postings for p in ps] or [0], dtype=np.uint32)
        check(_lib.load().nidx_vec_set_inverted_index(self._h, which, len(keys), ptr(key_bytes), ptr(key_off), ptr(post_off), ptr(flat)))

    def filter(self, nodes, n, out_bits: Optional[np.ndarray] = None) -> int:
        """nidx_vec_filter: the formula (n FilterNodes in pre-order) AND the alive set, on the device -> the number of matching
        paragraphs; the bitset goes to out_bits (host uint64 words, (paragraphs + 63) // 64) when given."""
        matching = C.c_uint64()
        check(_lib.load().nidx_vec_filter(self._h, nodes, n, ptr(out_bits), _lib.NIDX_MEM_HOST, C.byref(matching), None))
        return matching.value

    def prefilter_bits(self, doc_bits, join, n_docs: int, res_bits, res_ranges, n_res: int, n_paragraphs: int, formula=None, op=_lib.NIDX_F_AND,
                       doc_op=_lib.NIDX_F_AND):
        """nidx_vec_prefilter_bits -> (paragraph bits, matching): the paragraphs of the text documents in doc_bits (uint64 words; join:
        uint32 [n_docs], each document's key in the field index, or NIL) and those of the resources in res_bits (res_ranges: uint64
        [n_res][2], each resource's postings in the field index), combined under doc_op when both are given (None: no such part),
        then with `formula` (a FilterNode array, or None) under `op`, AND alive.  numpy inputs -> numpy words; torch CUDA tensors ->
        a torch int64 tensor (device path)."""
        on_device = _is_torch(doc_bits if doc_bits is not None else res_bits)
        mem, stream, alloc = _stage(self.cfg.device, on_device)
        if not on_device:
            host = lambda a, dtype: None if a is None else np.ascontiguousarray(a, dtype=dtype)   # noqa: E731
            doc_bits, join, res_bits, res_ranges = host(doc_bits, np.uint64), host(join, np.uint32), host(res_bits, np.uint64), host(res_ranges, np.uint64)
        out = alloc((n_paragraphs + 63) // 64, np.uint64)
        matching = C.c_uint64()
        check(_lib.load().nidx_vec_prefilter_bits(self._h, ptr(doc_bits), n_docs, ptr(join), doc_op, ptr(res_bits), n_res, ptr(res_ranges), formula,
                                                  0 if formula is None else len(formula), op, ptr(out), mem, C.byref(matching), stream))
        return out, matching.value

    # ---- search ----------------------------------------------------------------------------------------
    def search(self, queries, k: int, ef: int = 0, min_score: float = -1.0, with_duplicates=True, method=_lib.NIDX_METHOD_AUTO,
               filter_bits=None, filter_matching: int = 0, formula=None, out=None, stream: Optional[int] = None):
        """Batch search.  numpy in -> numpy out (host path, synchronous); torch CUDA tensors in -> torch
        CUDA tensors out (device path, asynchronous on the current stream).  `stream` (a cudaStream_t as int) lets concurrent
        host-path callers overlap their copies with each other's kernels.  `formula` (a FilterNode array in pre-order) is a filter
        evaluated on the device (nidx_vec_search_formula) instead of filter_bits.  Returns (ids, scores, counts)."""
        mem, stream, alloc = _stage(self.cfg.device, _is_torch(queries), stream)
        if mem == _lib.NIDX_MEM_DEVICE:
            import torch

            assert queries.is_cuda and queries.is_contiguous() and queries.dtype == torch.float32
        else:
            queries = np.ascontiguousarray(np.atleast_2d(queries), dtype=np.float32)
            filter_bits = None if filter_bits is None else np.ascontiguousarray(filter_bits, dtype=np.uint64)
        nq, ldq = queries.shape
        out = out or (alloc((nq, k), np.uint32), alloc((nq, k), np.float32), alloc(nq, np.int32))
        p = VecSearchParams(k, ef, min_score, int(with_duplicates), method, ptr(filter_bits), filter_matching)
        L = _lib.load()
        fn, by_formula = (L.nidx_vec_search, ()) if formula is None else (L.nidx_vec_search_formula, (formula, len(formula)))
        check(fn(self._h, ptr(queries), nq, ldq, mem, C.byref(p), *by_formula, ptr(out[0]), ptr(out[1]), ptr(out[2]), stream))
        return out

    # ---- RaBitQ (vector_types/rabitq.rs) ----------------------------------------------------------------
    def rabitq_encode(self):
        check(_lib.load().nidx_vec_rabitq_encode(self._h, None))

    def rabitq_codes(self) -> np.ndarray:
        out = np.empty((len(self), self.cfg.dimension // 8 + 8), dtype=np.uint8)
        check(_lib.load().nidx_vec_rabitq_codes(self._h, ptr(out)))
        return out

    def rabitq_estimate(self, queries):
        queries = np.ascontiguousarray(np.atleast_2d(queries), dtype=np.float32)
        nq = queries.shape[0]
        est = np.empty((nq, len(self)), dtype=np.float32)
        err = np.empty((nq, len(self)), dtype=np.float32)
        check(_lib.load().nidx_vec_rabitq_estimate(self._h, ptr(queries), nq, queries.shape[1], _lib.NIDX_MEM_HOST, ptr(est), ptr(err), None))
        return est, err

    def last_kernel_ms(self) -> float:
        ms = C.c_float()
        check(_lib.load().nidx_vec_last_kernel_ms(self._h, C.byref(ms)))
        return ms.value

    def counters_ex(self):
        out = (C.c_uint64 * 6)()
        check(_lib.load().nidx_vec_counters_ex(self._h, out))
        return dict(similarities=out[0], expansions=out[1], overflows=out[2] + out[3], estimates=out[4], rerank_needed=out[5])

    def counters(self):
        out = (C.c_uint64 * 3)()
        check(_lib.load().nidx_vec_counters(self._h, out))
        return dict(similarities=out[0], expansions=out[1], overflows=out[2])

    def exact_rows(self) -> int:
        """f32 rows the last HNSW search / build read (<= counters()["similarities"]; the rest were settled on the fp16 copy)."""
        out = C.c_uint64()
        check(_lib.load().nidx_vec_exact_rows(self._h, C.byref(out)))
        return out.value

    def walk_reruns(self) -> int:
        """Queries the last dense HNSW walk ran a second time, on capacities that cannot overflow, because their first walk lost a
        neighbour or a candidate to its visited set or its closest_up_nodes list (0 when nothing overflowed)."""
        out = C.c_uint64()
        check(_lib.load().nidx_vec_walk_reruns(self._h, C.byref(out)))
        return out.value

    def scan_counters(self):
        """The last exhaustive scan's tensor-core filter: vectors re-scored as survivors, and queries scanned in full instead
        (both 0 when the scan did not use the filter)."""
        out = (C.c_uint64 * 2)()
        check(_lib.load().nidx_vec_scan_counters(self._h, out))
        return dict(survivors=out[0], full_scans=out[1])


def _merge_parts(entry, ids, scores, device, part_stride, out):
    n_parts, nq, k = ids.shape
    _, stream, alloc = _stage(device, True)
    out = out or (alloc((nq, k), np.uint32), alloc((nq, k), np.float32), alloc((nq, k), np.int32))
    check(getattr(_lib.load(), entry)(device, ptr(ids), ptr(scores), n_parts, part_stride, nq, k, ptr(out[0]), ptr(out[1]), ptr(out[2]), stream))
    return out


def merge_topk(ids, scores, device=0, part_stride=0, out=None):
    """The text merge (nidx_merge_topk): [n_parts, nq, k] torch CUDA tensors (each part sorted desc, NIL padded) -> merged
    (ids, scores, part) ranked (score desc, part asc, position asc).  ids / scores may be strided views of one all-gather buffer:
    part_stride = elements between parts."""
    return _merge_parts("nidx_merge_topk", ids, scores, device, part_stride, out)


def merge_vector_parts(ids, scores, device=0, part_stride=0, out=None):
    """The vector merge (nidx_merge_vector_parts): merge_vector_responses' kmerge_by(score >=) over the parts in the order given,
    same arguments and results as merge_topk."""
    return _merge_parts("nidx_merge_vector_parts", ids, scores, device, part_stride, out)


def _pack_keys(keys):
    """[bytes] -> (concatenated bytes as uint8, uint64 offsets [n + 1])."""
    off = np.zeros(len(keys) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(k) for k in keys]) if len(keys) else []
    return np.frombuffer(b"".join(keys) + b"\0", dtype=np.uint8).copy(), off


def _facet_request(facets):
    """-> (TxtFacetRequest, the arrays it points into: keep them alive for the call)."""
    kb, ko = _pack_keys(list(facets))
    return _lib.TxtFacetRequest(len(facets), ptr(kb), ptr(ko)), (kb, ko)


def _txt_params(k, mode=_lib.NIDX_BM25_OR, use_tf=True, min_score=0.0, after=None, docaddr_base=0):
    """nidx_txt_search_params; after = (score, mode, docaddr) with mode 1 Drop / 2 KeepAfter / 3 Keep (nidx_paragraph SearchAfter)."""
    p = TxtSearchParams(k, mode, int(use_tf), min_score, 0, 0.0, 0, docaddr_base)
    if after is not None:
        p.after_score, p.after_mode, p.after_docaddr = float(after[0]), int(after[1]), int(after[2])
    return p


class TextSegment:
    def __init__(self, handle, n_docs, n_terms, device):
        self._h, self.n_docs, self.n_terms, self.device = handle, n_docs, n_terms, device

    @classmethod
    def create(cls, n_docs, n_terms, term_off, post_doc, post_tf, fieldnorm_id, device=0) -> "TextSegment":
        L = _lib.require_device()
        term_off = np.ascontiguousarray(term_off, dtype=np.uint64)
        post_doc = np.ascontiguousarray(post_doc, dtype=np.uint32)
        post_tf = np.ascontiguousarray(post_tf, dtype=np.uint32)
        fieldnorm_id = np.ascontiguousarray(fieldnorm_id, dtype=np.uint8)
        h = C.c_void_p()
        check(L.nidx_txt_create(device, n_docs, n_terms, ptr(term_off), ptr(post_doc), ptr(post_tf), ptr(fieldnorm_id), C.byref(h)))
        return cls(h, n_docs, n_terms, device)

    def set_stats(self, total_docs: int, total_tokens: int, doc_freq: Optional[np.ndarray] = None):
        df = None if doc_freq is None else np.ascontiguousarray(doc_freq, dtype=np.uint64)
        check(_lib.load().nidx_txt_set_stats(self._h, total_docs, total_tokens, ptr(df)))

    def set_alive(self, alive_bits: Optional[np.ndarray]):
        check(_lib.load().nidx_txt_set_alive(self._h, ptr(alive_bits)))

    def _queries(self, query_terms, query_off):
        """-> (mem, stream, alloc, query_terms, query_off, nq): torch CUDA int32 -> device path, anything else -> host uint32."""
        mem, stream, alloc = _stage(self.device, _is_torch(query_terms))
        if mem == _lib.NIDX_MEM_DEVICE:
            return mem, stream, alloc, query_terms, query_off, query_off.numel() - 1
        query_off = np.ascontiguousarray(query_off, dtype=np.uint32)
        return mem, stream, alloc, np.ascontiguousarray(query_terms, dtype=np.uint32), query_off, len(query_off) - 1

    def search(self, query_terms, query_off, k, mode=_lib.NIDX_BM25_OR, use_tf=True, min_score=0.0, out=None, after=None, docaddr_base=0):
        """query i = query_terms[query_off[i]:query_off[i+1]].  numpy -> host path, torch CUDA int32 -> device path.
        Returns (docs, scores, counts, total)."""
        p = _txt_params(k, mode, use_tf, min_score, after, docaddr_base)
        mem, stream, alloc, query_terms, query_off, nq = self._queries(query_terms, query_off)
        out = out or (alloc((nq, k), np.uint32), alloc((nq, k), np.float32), alloc(nq, np.int32), alloc(nq, np.uint64))
        check(_lib.load().nidx_txt_search(self._h, ptr(query_terms), ptr(query_off), nq, mem, C.byref(p), *map(ptr, out), stream))
        return out

    # ---- facets (tantivy FacetCollector; keys in the encoded form of include/nidx_b200.h: segments joined by 0x00) -----------
    def set_facets(self, keys, doc_off, doc_ords):
        """keys: bytes, strictly ascending (facet order); document d carries doc_ords[doc_off[d]:doc_off[d + 1]] (ascending)."""
        kb, ko = _pack_keys(keys)
        doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
        doc_ords = np.ascontiguousarray(doc_ords, dtype=np.uint32)
        check(_lib.load().nidx_txt_set_facets(self._h, len(keys), ptr(kb), ptr(ko), ptr(doc_off), ptr(doc_ords)))

    def facet_buckets(self, facets):
        """facets: encoded facet keys -> (bucket_req, bucket_ord) uint32 arrays (include/nidx_b200.h nidx_txt_facet_buckets)."""
        req, _keep = _facet_request(facets)
        n = C.c_uint32()
        check(_lib.load().nidx_txt_facet_buckets(self._h, C.byref(req), None, None, 0, C.byref(n)))
        b_req, b_ord = np.empty(n.value, dtype=np.uint32), np.empty(n.value, dtype=np.uint32)
        check(_lib.load().nidx_txt_facet_buckets(self._h, C.byref(req), ptr(b_req), ptr(b_ord), n.value, C.byref(n)))
        return b_req, b_ord

    def search_faceted(self, query_terms, query_off, k, facets, mode=_lib.NIDX_BM25_OR, use_tf=True, min_score=0.0, after=None, docaddr_base=0):
        """search() + per-query facet bucket counts in the same pass: (docs, scores, counts, total, facet_counts[nq][n_buckets]).
        numpy -> host path, torch CUDA -> device path (as search())."""
        p = _txt_params(k, mode, use_tf, min_score, after, docaddr_base)
        nb = len(self.facet_buckets(facets)[0])
        req, _keep = _facet_request(facets)
        mem, stream, alloc, query_terms, query_off, nq = self._queries(query_terms, query_off)
        out = (alloc((nq, k), np.uint32), alloc((nq, k), np.float32), alloc(nq, np.int32), alloc(nq, np.uint64), alloc((nq, nb), np.uint32, zero=True))
        check(_lib.load().nidx_txt_search_faceted(self._h, ptr(query_terms), ptr(query_off), nq, mem, C.byref(p), C.byref(req), *map(ptr, out), stream))
        return out

    def facet_count_all(self, facets, device_out=False):
        """Bucket counts over every alive document (uint32 [n_buckets]; device_out: a torch CUDA int32 tensor, device path)."""
        nb = len(self.facet_buckets(facets)[0])
        req, _keep = _facet_request(facets)
        mem, stream, alloc = _stage(self.device, device_out)
        out = alloc(nb, np.uint32, zero=True)
        check(_lib.load().nidx_txt_facet_count_all(self._h, C.byref(req), mem, ptr(out), stream))
        return out

    # ---- order by date (TopDocs::order_by_fast_field; seconds, NIDX_DATE_NONE = no date) ----------------------------------------
    def set_dates(self, created, modified):
        """Every document's created / modified seconds (int64 [n_docs], _lib.NIDX_DATE_NONE = none)."""
        created = np.ascontiguousarray(created, dtype=np.int64)
        modified = np.ascontiguousarray(modified, dtype=np.int64)
        assert len(created) == self.n_docs and len(modified) == self.n_docs
        check(_lib.load().nidx_txt_set_dates(self._h, ptr(created), ptr(modified)))

    def search_ordered(self, query_terms, query_off, k, field=_lib.NIDX_ORDER_CREATED, order=_lib.NIDX_ORDER_DESC, mode=_lib.NIDX_BM25_OR, facets=None):
        """search() ordered by date: (docs, dates, counts, total) plus the facet counts [nq][n_buckets] when `facets` (encoded keys)
        is given.  numpy -> host path, torch CUDA -> device path (as search())."""
        p = TxtSearchParams(k, mode, 0, 0.0, 0, 0.0, 0, 0)
        o = _lib.TxtOrder(field, order)
        req, _keep = _facet_request(facets) if facets is not None else (None, None)
        mem, stream, alloc, query_terms, query_off, nq = self._queries(query_terms, query_off)
        out = (alloc((nq, k), np.uint32), alloc((nq, k), np.int64), alloc(nq, np.int32), alloc(nq, np.uint64))
        if facets is not None:
            out += (alloc((nq, len(self.facet_buckets(facets)[0])), np.uint32, zero=True),)
        check(_lib.load().nidx_txt_search_ordered(self._h, ptr(query_terms), ptr(query_off), nq, mem, C.byref(p), C.byref(o),
                                                  C.byref(req) if req is not None else None, *map(ptr, out[:4]), ptr(out[4]) if facets is not None else None,
                                                  stream))
        return out

    # ---- exact phrases (tantivy PhraseQuery, slop 0: include/nidx_b200.h nidx_txt_search_phrases) ------------------------------
    def set_positions(self, positions):
        """Every posting's token positions in posting order (uint32; per posting its tf of them, strictly ascending)."""
        positions = np.ascontiguousarray(positions, dtype=np.uint32)
        check(_lib.load().nidx_txt_set_positions(self._h, ptr(positions), len(positions)))

    def search_phrases(self, query_terms, query_off, phrases, k, mode=_lib.NIDX_BM25_OR, use_tf=True, min_score=0.0, after=None, docaddr_base=0,
                       order=None, facets=None):
        """search() / search_faceted() / search_ordered() with phrase clauses: phrases = [(query index, [term ids])] (host lists).
        order = (field, type) orders by date (dates in place of scores).  Returns (docs, scores or dates, counts, total) plus the
        facet counts [nq][n_buckets] when `facets` (encoded keys) is given."""
        p = _txt_params(k, mode, use_tf, min_score, after, docaddr_base)
        terms = np.asarray([t for _, ts in phrases for t in ts], dtype=np.uint32)
        poff = np.zeros(len(phrases) + 1, dtype=np.uint32)
        poff[1:] = np.cumsum([len(ts) for _, ts in phrases])
        pq = np.asarray([q for q, _ in phrases], dtype=np.uint32)
        ph = _lib.TxtPhrases(ptr(terms), ptr(poff), ptr(pq), len(phrases))
        o = _lib.TxtOrder(*order) if order is not None else None
        req, _keep = _facet_request(facets) if facets is not None else (None, None)
        nb = len(self.facet_buckets(facets)[0]) if facets is not None else 0
        mem, stream, alloc, query_terms, query_off, nq = self._queries(query_terms, query_off)
        out = (alloc((nq, k), np.uint32), alloc((nq, k), np.int64 if order is not None else np.float32), alloc(nq, np.int32), alloc(nq, np.uint64))
        if facets is not None:
            out += (alloc((nq, nb), np.uint32, zero=True),)
        scores, dates = (None, out[1]) if order is not None else (out[1], None)
        check(_lib.load().nidx_txt_search_phrases(self._h, ptr(query_terms), ptr(query_off), nq, mem, C.byref(p), C.addressof(ph),
                                                  C.byref(o) if o is not None else None, C.byref(req) if req is not None else None,
                                                  ptr(out[0]), ptr(scores), ptr(dates), ptr(out[2]), ptr(out[3]),
                                                  ptr(out[4]) if facets is not None else None, stream))
        return out

    def list_ordered(self, k, field=_lib.NIDX_ORDER_CREATED, order=_lib.NIDX_ORDER_DESC, device_out=False):
        """The empty body ordered by date: the top k alive documents -> (docs [k], dates [k], count, total alive); with device_out
        all four are torch CUDA tensors (count and total of one element), on the device path."""
        o = _lib.TxtOrder(field, order)
        mem, stream, alloc = _stage(self.device, device_out)
        out = (alloc(k, np.uint32), alloc(k, np.int64), alloc(1, np.int32, zero=True), alloc(1, np.uint64, zero=True))
        check(_lib.load().nidx_txt_list_ordered(self._h, C.byref(o), k, mem, *map(ptr, out), stream))
        return out if device_out else (out[0], out[1], int(out[2][0]), int(out[3][0]))

    # ---- prefilter (TextReaderService::prefilter: include/nidx_b200.h nidx_txt_prefilter) ---------------------------------------
    def set_doc_columns(self, resource_ord, field_ord):
        """Every document's resource ord and field ord (uint32 [n_docs]) in the caller's dictionaries."""
        resource_ord = np.ascontiguousarray(resource_ord, dtype=np.uint32)
        field_ord = np.ascontiguousarray(field_ord, dtype=np.uint32)
        assert len(resource_ord) == self.n_docs and len(field_ord) == self.n_docs
        check(_lib.load().nidx_txt_set_doc_columns(self._h, ptr(resource_ord), ptr(field_ord)))

    def set_doc_groups(self, keys, doc_off, doc_ords):
        """The access group dictionary (encoded facet keys, strictly ascending) and every document's group ords (as set_facets);
        a document without ords is public."""
        kb, ko = _pack_keys(keys)
        doc_off = np.ascontiguousarray(doc_off, dtype=np.uint64)
        doc_ords = np.ascontiguousarray(doc_ords, dtype=np.uint32)
        check(_lib.load().nidx_txt_set_doc_groups(self._h, len(keys), ptr(kb), ptr(ko), ptr(doc_off), ptr(doc_ords)))

    def view(self, mask) -> "TextSegment":
        """This segment under a document mask (nidx_txt_view): every search of the returned segment runs over alive AND mask, with
        this segment's statistics.  mask: uint64 words [(n_docs + 63) // 64], numpy (host) or a torch CUDA int64 tensor (device
        path, current torch stream).  The view keeps this segment open; close it when done."""
        mem, stream, _ = _stage(self.device, _is_torch(mask))
        h = C.c_void_p()
        check(_lib.load().nidx_txt_view(self._h, ptr(mask), mem, C.byref(h), stream))
        v = TextSegment(h, self.n_docs, self.n_terms, self.device)
        v._parent = self
        return v

    def prefilter(self, nodes, out=None):
        """The expression (a PrefilterNode array in pre-order) AND alive -> (bits, matching): bits = uint64 words [(n_docs + 63) // 64]
        in a new numpy array, or written into `out` (a torch CUDA int64 tensor of that many words: device path)."""
        on_device = out is not None and _is_torch(out)
        mem, stream, alloc = _stage(self.device, on_device)
        if out is None:
            out = alloc((self.n_docs + 63) // 64, np.uint64)
        matching = C.c_uint64()
        check(_lib.load().nidx_txt_prefilter(self._h, C.addressof(nodes), len(nodes), ptr(out), mem, C.byref(matching), stream))
        return out, matching.value

    def resource_bits(self, doc_bits, n_resources: int):
        """nidx_txt_resource_bits: document bits -> the bits of their resource ords (uint64 words [(n_resources + 63) // 64]); a torch
        CUDA tensor in -> a torch int64 tensor out (device path), numpy -> numpy."""
        on_device = _is_torch(doc_bits)
        mem, stream, alloc = _stage(self.device, on_device)
        if not on_device:
            doc_bits = np.ascontiguousarray(doc_bits, dtype=np.uint64)
        out = alloc(max((n_resources + 63) // 64, 1), np.uint64)
        check(_lib.load().nidx_txt_resource_bits(self._h, ptr(doc_bits), n_resources, ptr(out), mem, stream))
        return out

    def join_mask(self, and_bits, doc_bits, n_doc_bits: int, doc_join, res_bits, n_res: int, res_join, op=_lib.NIDX_F_AND):
        """nidx_txt_join_mask: bit d = and_bits[d] AND op(doc_bits[doc_join[d]], res_bits[res_join[d]]) (and_bits / doc_bits None:
        all set) -> (mask words, matching).  torch CUDA res_bits -> device path (every input a device tensor), numpy -> host path."""
        on_device = _is_torch(res_bits)
        mem, stream, alloc = _stage(self.device, on_device)
        if not on_device:
            res_bits, res_join = np.ascontiguousarray(res_bits, dtype=np.uint64), np.ascontiguousarray(res_join, dtype=np.uint32)
            if and_bits is not None:
                and_bits = np.ascontiguousarray(and_bits, dtype=np.uint64)
            if doc_bits is not None:
                doc_bits, doc_join = np.ascontiguousarray(doc_bits, dtype=np.uint64), np.ascontiguousarray(doc_join, dtype=np.uint32)
        out = alloc(max((self.n_docs + 63) // 64, 1), np.uint64)
        matching = C.c_uint64()
        check(_lib.load().nidx_txt_join_mask(self._h, ptr(and_bits), ptr(doc_bits), n_doc_bits if doc_bits is not None else 0, ptr(doc_join),
                                             ptr(res_bits), n_res, ptr(res_join), op, ptr(out), mem, C.byref(matching), stream))
        return out, matching.value

    # ---- suggest (include/nidx_b200.h nidx_txt_set_repeated / nidx_txt_suggest_mask / nidx_txt_suggest_fuzzy) -----------------
    def set_repeated(self, repeated: Optional[np.ndarray]):
        """The paragraphs repeated in their field: a bool per document (None: none)."""
        words = None
        if repeated is not None:
            words = np.zeros((self.n_docs + 63) // 64 * 8, dtype=np.uint8)
            packed = np.packbits(np.asarray(repeated, dtype=bool), bitorder="little")
            words[: len(packed)] = packed
            words = words.view(np.uint64)
        check(_lib.load().nidx_txt_set_repeated(self._h, ptr(words)))

    def suggest_mask(self, sec_bits, pf_bits, joined_bits, op=_lib.NIDX_F_AND):
        """NOT repeated AND sec_bits AND op(pf_bits, joined_bits), a None operand dropped -> (mask words, matching).  Torch CUDA operands
        -> device path (a torch int64 mask), numpy or all None -> host path."""
        ops = [b for b in (sec_bits, pf_bits, joined_bits) if b is not None]
        on_device = any(_is_torch(b) for b in ops)
        mem, stream, alloc = _stage(self.device, on_device)
        if not on_device:
            sec_bits, pf_bits, joined_bits = (None if b is None else np.ascontiguousarray(b, dtype=np.uint64) for b in (sec_bits, pf_bits, joined_bits))
        out = alloc(max((self.n_docs + 63) // 64, 1), np.uint64)
        matching = C.c_uint64()
        check(_lib.load().nidx_txt_suggest_mask(self._h, ptr(sec_bits), ptr(pf_bits), ptr(joined_bits), op, ptr(out), mem, C.byref(matching), stream))
        return out, matching.value

    def suggest_fuzzy(self, clauses, exp_bits, n_exp_rows: int, n_dict: int, phrases, k: int, match_hits: int = 10, match_cap: int = 4096):
        """The fuzzy pass: clauses = [(NIDX_SG_* kind, arg)], exp_bits = SuggestDict.expand's torch tensor (None without fuzzy
        clauses), phrases = [[term ids]] -> (ids, scores, count, matches) with matches = sorted (hit, clause, term id) triples (host
        path: the call returns when they are in place)."""
        cl = (_lib.SuggestClause * len(clauses))(*[_lib.SuggestClause(kind, arg) for kind, arg in clauses])
        terms = np.asarray([t for p in phrases for t in p], dtype=np.uint32)
        poff = np.zeros(len(phrases) + 1, dtype=np.uint32)
        poff[1:] = np.cumsum([len(p) for p in phrases])
        pq = np.zeros(len(phrases), dtype=np.uint32)
        ph = _lib.TxtPhrases(ptr(terms), ptr(poff), ptr(pq), len(phrases))
        while True:
            ids, scores, count = np.empty(k, np.uint32), np.empty(k, np.float32), np.zeros(1, np.int32)
            matches, n_matches = np.empty(max(match_cap, 1), np.uint64), np.zeros(1, np.uint32)
            check(_lib.load().nidx_txt_suggest_fuzzy(self._h, C.addressof(cl), len(clauses), ptr(exp_bits), n_exp_rows, n_dict,
                                                     C.addressof(ph) if phrases else None, k, match_hits, _lib.NIDX_MEM_HOST, ptr(ids), ptr(scores),
                                                     ptr(count), ptr(matches), match_cap, ptr(n_matches), None))
            if int(n_matches[0]) <= match_cap:
                break
            match_cap = int(n_matches[0])   # a larger list than expected: run again with room for all of it
        m = np.sort(matches[: int(n_matches[0])])
        trip = [(int(x >> 40), int((x >> 32) & 0xFF), int(x & 0xFFFFFFFF)) for x in m]
        c = int(count[0])
        return ids[:c], scores[:c], c, trip

    def suggest_last_times(self):
        """(bitsets, scored pass, top-k, matches) ms of the last fuzzy pass."""
        ms = (C.c_float * 4)()
        check(_lib.load().nidx_txt_suggest_last_times(self._h, ms))
        return list(ms)

    def set_doc_keys(self, keys: Optional[np.ndarray]):
        """Caller keys of the documents (paragraph ids) for rank fusion; None = the document number."""
        k = None if keys is None else np.ascontiguousarray(keys, dtype=np.uint64)
        check(_lib.load().nidx_txt_set_doc_keys(self._h, ptr(k)))

    def last_kernel_ms(self) -> float:
        ms = C.c_float()
        check(_lib.load().nidx_txt_last_kernel_ms(self._h, C.byref(ms)))
        return ms.value

    def close(self):
        if self._h is not None:
            _lib.load().nidx_txt_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class SuggestDict:
    """nidx_suggest_dict: a paragraph index's vocabulary as code points in HBM, for the fuzzy expansion of NidxSearcher.Suggest."""

    def __init__(self, terms, device=0):
        L = _lib.require_device()
        cps = [np.frombuffer(t.encode("utf-32-le"), dtype=np.uint32) for t in terms]
        off = np.zeros(len(terms) + 1, dtype=np.uint64)
        off[1:] = np.cumsum([len(c) for c in cps]) if terms else []
        cp = np.concatenate(cps).astype(np.uint32) if cps else np.zeros(1, dtype=np.uint32)
        self.n_terms, self.device, self._h = len(terms), device, None
        h = C.c_void_p()
        check(L.nidx_suggest_dict_create(device, len(terms), ptr(cp), ptr(off), C.byref(h)))
        self._h = h

    def expand(self, terms):
        """[(term, distance, prefix)] -> (torch CUDA int64 bitsets [len(terms)][(n_terms + 63) // 64], expanded terms per row)."""
        import torch

        cps = [np.frombuffer(t.encode("utf-32-le"), dtype=np.uint32).copy() for t, _, _ in terms]
        arr = (_lib.GraphTerm * max(len(terms), 1))(*[_lib.GraphTerm(0, int(d), int(p), len(c), ptr(c)) for c, (_, d, p) in zip(cps, terms)])
        bits = torch.empty((max(len(terms), 1), max((self.n_terms + 63) // 64, 1)), dtype=torch.int64, device=torch.device("cuda", self.device))
        counts = np.zeros(max(len(terms), 1), dtype=np.uint64)
        check(_lib.load().nidx_suggest_expand(self._h, arr, len(terms), ptr(bits), ptr(counts), _torch_stream(self.device)))
        return bits, counts[: len(terms)]

    def last_ms(self) -> float:
        ms = C.c_float()
        check(_lib.load().nidx_suggest_last_ms(self._h, C.byref(ms)))
        return ms.value

    def close(self):
        if self._h is not None:
            _lib.load().nidx_suggest_dict_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
