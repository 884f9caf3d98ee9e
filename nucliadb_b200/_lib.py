"""ctypes loader for ``libnidx_b200.so`` (the C ABI in ``include/nidx_b200.h``).

The CUDA library is the product: if it is missing or no CUDA device is usable the package fails
loudly -- there is no CPU fallback anywhere in ``nucliadb_b200``.

``SIGNATURES`` declares every function of the header once: name -> (restype, argtypes), applied to the library by ``load()``.
Scalars take their exact width (``int`` = ``int32_t``); data buffers, handles, out-handles and streams are ``void*``; pointers to
the ABI's own structs are typed, so passing the wrong struct raises.  ctypes then converts plain Python values at every call
site and rejects too few arguments or a wrong type.  It does not catch extra trailing arguments, and it does not range-check
integers (``-1`` passed for a ``uint64_t`` arrives as 2^64 - 1).
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


class PrefilterNode(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n", C.c_int32), ("lo", C.c_int64), ("hi", C.c_int64), ("terms", C.c_void_p)]


NIDX_P_FACET, NIDX_P_FIELD, NIDX_P_RESOURCE, NIDX_P_DATE, NIDX_P_KEYWORD, NIDX_P_ALL, NIDX_P_AND, NIDX_P_OR, NIDX_P_NOT, NIDX_P_PUBLIC, NIDX_P_GROUP = range(11)
NIDX_PREFILTER_MAX_DEPTH = 64


class GraphColumns(C.Structure):
    _fields_ = [("col", C.c_void_p * 11), ("tok_off", C.c_void_p * 2), ("tok_ord", C.c_void_p * 2), ("n_values", C.c_uint32), ("value_cp", C.c_void_p),
                ("value_off", C.c_void_p), ("n_tokens", C.c_uint32), ("token_cp", C.c_void_p), ("token_off", C.c_void_p), ("n_node_keys", C.c_uint32),
                ("n_rel_keys", C.c_uint32)]


class GraphNode(C.Structure):
    _fields_ = [("kind", C.c_int32), ("n", C.c_int32), ("arg", C.c_int32), ("w", C.c_float), ("lo", C.c_int64), ("hi", C.c_int64), ("ords", C.c_void_p)]


class GraphTerm(C.Structure):
    _fields_ = [("dict", C.c_int32), ("distance", C.c_int32), ("prefix", C.c_int32), ("n_cp", C.c_int32), ("cp", C.c_void_p)]


(NIDX_G_EQ, NIDX_G_COLBITS, NIDX_G_TOKBITS, NIDX_G_TOKSET, NIDX_G_FACET, NIDX_G_CONST, NIDX_G_AND, NIDX_G_OR, NIDX_G_NOT,
 NIDX_G_CONST_SCORE) = range(10)
NIDX_G_TERMS_VALUES, NIDX_G_TERMS_TOKENS = 0, 1
NIDX_G_PATH, NIDX_G_NODES, NIDX_G_RELATIONS = 0, 1, 2


class SuggestClause(C.Structure):
    _fields_ = [("kind", C.c_int32), ("arg", C.c_uint32)]


NIDX_SG_FUZZY, NIDX_SG_TERM, NIDX_SG_PHRASE = 0, 1, 2
NIDX_SG_MAX_CLAUSES, NIDX_SG_MAX_HITS = 64, 16


class TxtSearchParams(C.Structure):
    _fields_ = [("k", C.c_int32), ("mode", C.c_int32), ("use_tf", C.c_int32), ("min_score", C.c_float), ("after_mode", C.c_int32),
                ("after_score", C.c_float), ("after_docaddr", C.c_uint64), ("docaddr_base", C.c_uint64)]


class TxtFacetRequest(C.Structure):
    _fields_ = [("n", C.c_int32), ("key_bytes", C.c_void_p), ("key_off", C.c_void_p)]


class TxtOrder(C.Structure):
    _fields_ = [("field", C.c_int32), ("type", C.c_int32)]


class TxtPhrases(C.Structure):
    _fields_ = [("terms", C.c_void_p), ("off", C.c_void_p), ("query", C.c_void_p), ("n", C.c_int32)]


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


# every function include/nidx_b200.h declares (tests check the table against the header and the .so's exports)
i32, u32, i64, u64, f64, P = C.c_int32, C.c_uint32, C.c_int64, C.c_uint64, C.c_double, C.c_void_p
CFG, VSP, NODES, TSP = C.POINTER(VecConfig), C.POINTER(VecSearchParams), C.POINTER(FilterNode), C.POINTER(TxtSearchParams)
REQ, ORDER, RRF = C.POINTER(TxtFacetRequest), C.POINTER(TxtOrder), C.POINTER(RrfSource)
SIGNATURES = {
    "nidx_last_error": (C.c_char_p, []),
    "nidx_device_count": (i32, []),
    "nidx_launch_count": (u64, []),
    "nidx_vec_create": (i32, [CFG, P, u64, i32, i32, P, P]),
    "nidx_vec_open": (i32, [CFG, C.c_char_p, P]),
    "nidx_vec_save": (i32, [P, C.c_char_p]),
    "nidx_vec_close": (None, [P]),
    "nidx_vec_len": (u64, [P]),
    "nidx_vec_device_vectors": (P, [P, P]),
    "nidx_vec_build_hnsw": (i32, [P, u64, i32, P]),
    "nidx_hnsw_levels": (i32, [u64, i32, u64, P]),
    "nidx_normalize_vectors": (i32, [i32, P, u64, i32, i32, i32, P]),
    "nidx_use_hnsw": (i32, [u64, u64, u64, i32, i32]),
    "nidx_vec_extend_hnsw": (i32, [P, u64, P, P, P, P, P, u32, u32, u64, i32, P]),
    "nidx_vec_graph_dims": (i32, [P, P, P, P, P, P]),
    "nidx_vec_set_graph": (i32, [P, P, P, P, P, P]),
    "nidx_vec_get_graph": (i32, [P, P, P, P, P, P]),
    "nidx_vec_set_alive": (i32, [P, P, i32]),
    "nidx_vec_search": (i32, [P, P, i32, i32, i32, VSP, P, P, P, P]),
    "nidx_vec_set_inverted_index": (i32, [P, i32, u32, P, P, P, P]),
    "nidx_vec_filter": (i32, [P, NODES, i32, P, i32, P, P]),
    "nidx_vec_search_formula": (i32, [P, P, i32, i32, i32, VSP, NODES, i32, P, P, P, P]),
    "nidx_merge_topk": (i32, [i32, P, P, i32, i64, i32, i32, P, P, P, P]),
    "nidx_merge_vector_parts": (i32, [i32, P, P, i32, i64, i32, i32, P, P, P, P]),
    "nidx_vec_counters": (i32, [P, P]),
    "nidx_vec_counters_ex": (i32, [P, P]),
    "nidx_vec_exact_rows": (i32, [P, P]),
    "nidx_vec_scan_counters": (i32, [P, P]),
    "nidx_vec_walk_reruns": (i32, [P, P]),
    "nidx_vec_rabitq_encode": (i32, [P, P]),
    "nidx_vec_rabitq_codes": (i32, [P, P]),
    "nidx_vec_rabitq_estimate": (i32, [P, P, i32, i32, i32, P, P, P]),
    "nidx_vec_last_kernel_ms": (i32, [P, P]),
    "nidx_txt_create": (i32, [i32, u32, u32, P, P, P, P, P]),
    "nidx_txt_set_stats": (i32, [P, u64, u64, P]),
    "nidx_txt_set_alive": (i32, [P, P]),
    "nidx_txt_close": (None, [P]),
    "nidx_txt_view": (i32, [P, P, i32, P, P]),
    "nidx_txt_search": (i32, [P, P, P, i32, i32, TSP, P, P, P, P, P]),
    "nidx_txt_last_kernel_ms": (i32, [P, P]),
    "nidx_txt_set_facets": (i32, [P, u32, P, P, P, P]),
    "nidx_txt_facet_buckets": (i32, [P, REQ, P, P, u32, P]),
    "nidx_txt_search_faceted": (i32, [P, P, P, i32, i32, TSP, REQ, P, P, P, P, P, P]),
    "nidx_txt_facet_count_all": (i32, [P, REQ, i32, P, P]),
    "nidx_txt_set_dates": (i32, [P, P, P]),
    "nidx_txt_search_ordered": (i32, [P, P, P, i32, i32, TSP, ORDER, REQ, P, P, P, P, P, P]),
    "nidx_txt_list_ordered": (i32, [P, ORDER, i32, i32, P, P, P, P, P]),
    "nidx_txt_set_positions": (i32, [P, P, u64]),
    "nidx_txt_search_phrases": (i32, [P, P, P, i32, i32, TSP, P, ORDER, REQ, P, P, P, P, P, P, P]),
    "nidx_txt_set_doc_columns": (i32, [P, P, P]),
    "nidx_txt_set_doc_groups": (i32, [P, u32, P, P, P, P]),
    "nidx_txt_prefilter": (i32, [P, P, i32, P, i32, P, P]),   # nodes: an array of PrefilterNode
    "nidx_vec_prefilter_bits": (i32, [P, P, u64, P, i32, P, u64, P, NODES, i32, i32, P, i32, P, P]),
    "nidx_txt_resource_bits": (i32, [P, P, u64, P, i32, P]),
    "nidx_txt_join_mask": (i32, [P, P, P, u64, P, P, u64, P, i32, P, i32, P, P]),
    "nidx_graph_create": (i32, [P, P]),
    "nidx_graph_set_columns": (i32, [P, P]),   # cols: a GraphColumns
    "nidx_graph_close": (None, [P]),
    "nidx_graph_search": (i32, [P, P, i32, P, i32, i32, i32, P, i32, P, P, P, P]),
    "nidx_graph_last_times": (i32, [P, P]),
    "nidx_suggest_dict_create": (i32, [i32, u32, P, P, P]),
    "nidx_suggest_dict_close": (None, [P]),
    "nidx_suggest_expand": (i32, [P, P, i32, P, P, P]),   # terms: an array of GraphTerm
    "nidx_suggest_last_ms": (i32, [P, P]),
    "nidx_txt_set_repeated": (i32, [P, P]),
    "nidx_txt_suggest_mask": (i32, [P, P, P, P, i32, P, i32, P, P]),
    "nidx_txt_suggest_fuzzy": (i32, [P, P, i32, P, i32, u64, P, i32, i32, i32, P, P, P, P, u32, P, P]),   # clauses: SuggestClause, phrases: TxtPhrases
    "nidx_txt_suggest_last_times": (i32, [P, P]),
    "nidx_shard_unique_id": (i32, [P]),
    "nidx_shard_init": (i32, [P, i32, i32, i32, P]),
    "nidx_shard_destroy": (None, [P]),
    "nidx_vec_set_paragraph_keys": (i32, [P, P]),
    "nidx_vec_search_sharded": (i32, [P, P, P, i32, i32, i32, VSP, i32, P, P, P, P, P]),
    "nidx_vec_shard_record": (i32, [P, P, i32, i32, i32, VSP, i32, i32, P, P]),
    "nidx_shard_merge": (i32, [i32, P, i32, i32, i32, i32, i32, i32, P, P, P, P, P]),
    "nidx_txt_search_sharded": (i32, [P, P, P, P, i32, i32, TSP, P, P, P, P, P, P]),
    "nidx_txt_set_doc_keys": (i32, [P, P]),
    "nidx_rank_fusion_rrf": (i32, [i32, RRF, i32, i32, f64, i32, P, P, P, P, P]),
    "nidx_shard_search": (i32, [C.POINTER(ShardSearchRequest), C.POINTER(ShardSearchResponse), i32, P]),
}
SYMBOLS = list(SIGNATURES)

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
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(L, name)
        fn.restype, fn.argtypes = restype, argtypes
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
