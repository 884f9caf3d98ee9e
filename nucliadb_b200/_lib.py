"""ctypes loader for ``libnidx_b200.so`` (the C ABI in ``include/nidx_b200.h``).

The CUDA library is the product: if it is missing or no CUDA device is usable the package fails
loudly -- there is no CPU fallback anywhere in ``nucliadb_b200``.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# NIDX_B200_LIB names another build of the same library next to this file (A/B runs of two builds)
LIB_PATH = os.path.join(_HERE, os.path.basename(os.environ.get("NIDX_B200_LIB", "libnidx_b200.so")))

NIDX_MEM_HOST, NIDX_MEM_DEVICE = 0, 1
NIDX_SIM_DOT, NIDX_SIM_COSINE, NIDX_SIM_L2 = 0, 1, 2
NIDX_METHOD_AUTO, NIDX_METHOD_HNSW, NIDX_METHOD_BRUTE, NIDX_METHOD_BRUTE_RABITQ, NIDX_METHOD_HNSW_RABITQ = 0, 1, 2, 3, 4
NIDX_BM25_OR, NIDX_BM25_AND = 0, 1
NIDX_ORDER_CREATED, NIDX_ORDER_MODIFIED = 0, 1   # OrderBy.OrderField
NIDX_ORDER_DESC, NIDX_ORDER_ASC = 0, 1           # OrderBy.OrderType
NIDX_DATE_NONE = -(1 << 63)                      # a document without a date
NIL = 0xFFFFFFFF

# every symbol include/nidx_b200.h declares (tests check the .so exports exactly these)
SYMBOLS = [
    "nidx_last_error", "nidx_device_count", "nidx_launch_count",
    "nidx_vec_create", "nidx_vec_open", "nidx_vec_save", "nidx_vec_close", "nidx_vec_len", "nidx_vec_device_vectors",
    "nidx_use_hnsw", "nidx_hnsw_levels", "nidx_normalize_vectors", "nidx_vec_build_hnsw", "nidx_vec_extend_hnsw", "nidx_vec_graph_dims", "nidx_vec_set_graph", "nidx_vec_get_graph", "nidx_vec_set_alive",
    "nidx_vec_set_inverted_index", "nidx_vec_filter", "nidx_vec_search_formula",
    "nidx_vec_search", "nidx_merge_topk", "nidx_merge_vector_parts", "nidx_vec_counters", "nidx_vec_counters_ex", "nidx_vec_exact_rows", "nidx_vec_scan_counters", "nidx_vec_last_kernel_ms",
    "nidx_vec_rabitq_encode", "nidx_vec_rabitq_codes", "nidx_vec_rabitq_estimate",
    "nidx_txt_create", "nidx_txt_set_stats", "nidx_txt_set_alive", "nidx_txt_close", "nidx_txt_search", "nidx_txt_last_kernel_ms",
    "nidx_txt_set_facets", "nidx_txt_facet_buckets", "nidx_txt_search_faceted", "nidx_txt_facet_count_all",
    "nidx_txt_set_dates", "nidx_txt_search_ordered", "nidx_txt_list_ordered",
    "nidx_shard_unique_id", "nidx_shard_init", "nidx_shard_destroy", "nidx_vec_set_paragraph_keys", "nidx_vec_search_sharded",
    "nidx_vec_shard_record", "nidx_shard_merge", "nidx_txt_search_sharded",
    "nidx_txt_set_doc_keys", "nidx_rank_fusion_rrf", "nidx_shard_search",
]


class NidxError(RuntimeError):
    """Mirror of the reference's anyhow::Error / VectorErr (nidx_vector/src/lib.rs:203-232)."""

    def __init__(self, code: int, message: str):
        super().__init__(f"nidx_b200 error {code}: {message}")
        self.code = code


class VecConfig(C.Structure):
    _fields_ = [("dimension", C.c_int32), ("similarity", C.c_int32), ("multi_vector", C.c_int32), ("m", C.c_int32), ("m0", C.c_int32),
                ("ef_construction", C.c_int32), ("ef_search", C.c_int32), ("device", C.c_int32)]


class VecSearchParams(C.Structure):
    _fields_ = [("k", C.c_int32), ("ef", C.c_int32), ("min_score", C.c_float), ("with_duplicates", C.c_int32), ("method", C.c_int32),
                ("filter_bits", C.c_void_p), ("filter_matching", C.c_uint64)]


class FilterNode(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n", C.c_int32), ("keys", C.POINTER(C.c_void_p)), ("key_len", C.POINTER(C.c_uint32))]   # keys are raw bytes (may hold NULs)


NIDX_INV_LABELS, NIDX_INV_FIELDS = 0, 1
NIDX_F_LABEL, NIDX_F_KEYS, NIDX_F_AND, NIDX_F_OR, NIDX_F_NOT = 0, 1, 2, 3, 4


class TxtSearchParams(C.Structure):
    _fields_ = [("k", C.c_int32), ("mode", C.c_int32), ("use_tf", C.c_int32), ("min_score", C.c_float), ("after_mode", C.c_int32),
                ("after_score", C.c_float), ("after_docaddr", C.c_uint64), ("docaddr_base", C.c_uint64)]


class TxtFacetRequest(C.Structure):
    _fields_ = [("n", C.c_int32), ("key_bytes", C.c_void_p), ("key_off", C.c_void_p)]


class TxtOrder(C.Structure):
    _fields_ = [("field", C.c_int32), ("type", C.c_int32)]


class RrfSource(C.Structure):
    _fields_ = [("keys", C.c_void_p), ("scores", C.c_void_p), ("counts", C.c_void_p), ("k", C.c_int32), ("weight", C.c_double)]


class ShardSearchRequest(C.Structure):
    _fields_ = [("nq", C.c_int32),
                ("vec", C.c_void_p), ("queries", C.c_void_p), ("ldq", C.c_int32), ("vec_params", C.POINTER(VecSearchParams)),
                ("formula", C.POINTER(FilterNode)), ("n_formula", C.c_int32),
                ("par", C.c_void_p), ("par_terms", C.c_void_p), ("par_off", C.c_void_p), ("par_params", C.POINTER(TxtSearchParams)),
                ("doc", C.c_void_p), ("doc_terms", C.c_void_p), ("doc_off", C.c_void_p), ("doc_params", C.POINTER(TxtSearchParams)),
                ("rrf_k", C.c_double), ("weight_keyword", C.c_double), ("weight_semantic", C.c_double), ("semantic_first", C.c_int32)]


class ShardSearchResponse(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in ("vec_ids", "vec_scores", "vec_counts", "par_docs", "par_scores", "par_counts", "par_total",
                                           "doc_docs", "doc_scores", "doc_counts", "doc_total", "fused_keys", "fused_scores", "fused_refs", "fused_counts")]


_lib = None


def load():
    """Load the shared library (raises if it has not been built: run ``__graft_entry__.build()``)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                          "(nvcc, sm_90a). nucliadb_b200 has no CPU fallback.")
    L = C.CDLL(LIB_PATH)
    L.nidx_last_error.restype = C.c_char_p
    L.nidx_launch_count.restype = C.c_uint64
    L.nidx_vec_len.restype = C.c_uint64
    L.nidx_vec_device_vectors.restype = C.c_void_p
    L.nidx_vec_close.restype = None
    L.nidx_txt_close.restype = None
    L.nidx_shard_destroy.restype = None
    _lib = L
    return L


def check(rc: int):
    if rc != 0:
        raise NidxError(rc, load().nidx_last_error().decode("utf-8", "replace"))


def require_device():
    L = load()
    if L.nidx_device_count() <= 0:
        raise NidxError(-2, "no CUDA device available; nucliadb_b200 has no CPU fallback")
    return L


def ptr(a):
    """void* of a numpy array / torch tensor / None / int."""
    if a is None:
        return None
    if isinstance(a, int):
        return C.c_void_p(a)
    if hasattr(a, "data_ptr"):
        return C.c_void_p(a.data_ptr())
    return a.ctypes.data_as(C.c_void_p)
