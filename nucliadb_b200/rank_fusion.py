"""Rank fusion and the fused shard search, host mirror of the reference's interface over the C ABI.

    ReciprocalRankFusion(k, window=, weights=).fuse(sources)     nucliadb/src/nucliadb/search/search/rank_fusion.py:106-186
    shard_search(...)                                            nidx/src/searcher/shard_search.rs:176-241 (run_index_searches)

`fuse` takes {source name: [(key, score), ...]} with 64-bit integer keys (the paragraph id's table index or hash) and returns
[(key, score, score_type), ...] exactly like the reference's merged list: fused by `nidx_rank_fusion_rrf` on the device (IEEE
double arithmetic in the reference's association), never on the host.
"""
from __future__ import annotations

import ctypes as C
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

from . import _lib
from ._lib import RrfSource, ShardSearchRequest, ShardSearchResponse, TxtSearchParams, VecSearchParams, check, ptr

KEYWORD, SEMANTIC, GRAPH = "keyword", "semantic", "graph"      # IndexSource (rank_fusion.py:54-57)
_TYPE_OF = {KEYWORD: "BM25", SEMANTIC: "VECTOR", GRAPH: "RELATION_RELEVANCE"}      # SCORE_TYPE of a retriever's items


class ReciprocalRankFusion:
    def __init__(self, k: float = 60.0, *, window: int, weights: Optional[Dict[str, float]] = None, default_weight: float = 1.0, device: int = 0):
        self._k, self._window, self._weights, self._default_weight, self.device = float(k), window, dict(weights or {}), float(default_weight), device

    @property
    def window(self) -> int:
        return self._window

    def fuse(self, sources: Dict[str, Sequence[Tuple[int, float]]]) -> List[Tuple[int, float, str]]:
        L = _lib.require_device()
        names = list(sources)
        if not names or len(names) > 4:
            raise _lib.NidxError(-1, "rank fusion takes 1..4 sources")
        arrs, structs = [], (RrfSource * len(names))()
        cap = 0
        for i, name in enumerate(names):
            # every source sorted by its own score, descending and stable (rank_fusion.py:151-154)
            items = sorted(sources[name], key=lambda t: t[1], reverse=True)
            kk = max(1, len(items))
            keys = np.full((1, kk), np.uint64(0xFFFFFFFFFFFFFFFF), dtype=np.uint64)
            scores = np.zeros((1, kk), dtype=np.float32)
            for j, (key, sc) in enumerate(items):
                keys[0, j], scores[0, j] = key, sc
            cnt = np.asarray([len(items)], dtype=np.int32)
            arrs.append((keys, scores, cnt))
            structs[i] = RrfSource(keys.ctypes.data, scores.ctypes.data, cnt.ctypes.data, kk, self._weights.get(name, self._default_weight))
            cap += kk
        out_keys, out_scores = np.empty((1, cap), dtype=np.uint64), np.empty((1, cap), dtype=np.float64)
        out_refs, out_counts = np.empty((1, cap), dtype=np.uint32), np.empty(1, dtype=np.int32)
        check(L.nidx_rank_fusion_rrf(self.device, structs, len(names), 1, self._k, _lib.NIDX_MEM_HOST, ptr(out_keys), ptr(out_scores), ptr(out_refs),
                                     ptr(out_counts), None))
        fused = []
        types = [_TYPE_OF.get(name, "RELATION_RELEVANCE") for name in names]
        for j in range(int(out_counts[0])):
            ref = int(out_refs[0, j])
            first, mask = types[ref >> 28], (ref >> 24) & 0xF
            joined = {t for i, t in enumerate(types) if mask >> i & 1}
            # rank_fusion.py:166-174: the surviving (first) item becomes BOTH when a BM25 and a VECTOR item meet; other types are kept
            st = "BOTH" if first in ("BM25", "VECTOR") and {"BM25", "VECTOR"} <= joined else first
            fused.append((int(out_keys[0, j]), float(out_scores[0, j]), st))
        return fused


def shard_search(nq, *, vec=None, queries=None, vec_params: Optional[VecSearchParams] = None, par=None, par_terms=None, par_off=None,
                 par_params: Optional[TxtSearchParams] = None, doc=None, doc_terms=None, doc_off=None, doc_params: Optional[TxtSearchParams] = None,
                 rrf_k: float = 0.0, weight_keyword: float = 1.0, weight_semantic: float = 1.0, semantic_first: bool = False):
    """run_index_searches (shard_search.rs:176-241) for a batch of nq requests with host (numpy) buffers: the vector, paragraph and
    document searches of the batch run concurrently on the device; rrf_k > 0 fuses the paragraph (keyword) and vector (semantic)
    lists on the device.  `vec` is a VectorSegment, `par` / `doc` TextSegments.  Returns a dict of numpy arrays."""
    L = _lib.require_device()
    rq, rs, keep, out = ShardSearchRequest(), ShardSearchResponse(), [], {}
    rq.nq = nq

    def host(a, dtype):
        a = np.ascontiguousarray(a, dtype=dtype)
        keep.append(a)
        return a.ctypes.data

    def alloc(name, shape, dtype):
        out[name] = np.empty(shape, dtype=dtype)
        return out[name].ctypes.data

    kv = kp = 0
    if vec is not None:
        q = np.ascontiguousarray(queries, dtype=np.float32)
        keep.append(q)
        kv = vec_params.k
        rq.vec, rq.queries, rq.ldq, rq.vec_params = vec._h, q.ctypes.data, q.shape[1], C.pointer(vec_params)
        rs.vec_ids, rs.vec_scores, rs.vec_counts = alloc("vec_ids", (nq, kv), np.uint32), alloc("vec_scores", (nq, kv), np.float32), alloc("vec_counts", nq, np.int32)
    if par is not None:
        kp = par_params.k
        rq.par, rq.par_terms, rq.par_off, rq.par_params = par._h, host(par_terms, np.uint32), host(par_off, np.uint32), C.pointer(par_params)
        rs.par_docs, rs.par_scores = alloc("par_docs", (nq, kp), np.uint32), alloc("par_scores", (nq, kp), np.float32)
        rs.par_counts, rs.par_total = alloc("par_counts", nq, np.int32), alloc("par_total", nq, np.uint64)
    if doc is not None:
        kd = doc_params.k
        rq.doc, rq.doc_terms, rq.doc_off, rq.doc_params = doc._h, host(doc_terms, np.uint32), host(doc_off, np.uint32), C.pointer(doc_params)
        rs.doc_docs, rs.doc_scores = alloc("doc_docs", (nq, kd), np.uint32), alloc("doc_scores", (nq, kd), np.float32)
        rs.doc_counts, rs.doc_total = alloc("doc_counts", nq, np.int32), alloc("doc_total", nq, np.uint64)
    rq.rrf_k, rq.weight_keyword, rq.weight_semantic, rq.semantic_first = rrf_k, weight_keyword, weight_semantic, int(semantic_first)
    if rrf_k > 0 and vec is not None and par is not None:
        rs.fused_keys, rs.fused_scores = alloc("fused_keys", (nq, kv + kp), np.uint64), alloc("fused_scores", (nq, kv + kp), np.float64)
        rs.fused_refs, rs.fused_counts = alloc("fused_refs", (nq, kv + kp), np.uint32), alloc("fused_counts", nq, np.int32)
    check(L.nidx_shard_search(C.byref(rq), C.byref(rs), _lib.NIDX_MEM_HOST, None))
    return out
