"""The C-ABI library loads and exports exactly what include/nidx_b200.h declares; without a CUDA device
every entry point fails loudly (no CPU fallback).  CPU only: no compute calls."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from nucliadb_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_functions():
    text = open(os.path.join(ROOT, "include", "nidx_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(nidx_[a-z0-9_]+)\s*\(", text)))


def header_prototypes():
    """-> {name: (return type, [parameter declarations])} of every function include/nidx_b200.h declares."""
    text = open(os.path.join(ROOT, "include", "nidx_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = "\n".join(l for l in text.splitlines() if not l.lstrip().startswith("#"))
    protos = {}
    for stmt in text.split(";"):
        stmt = stmt.split("{")[-1].split("}")[-1]
        m = re.fullmatch(r"\s*(.+?)\s*\b(nidx_\w+)\s*\((.*)\)\s*", stmt, flags=re.S)
        if m:
            params = [p.strip() for p in m.group(3).split(",")]
            protos[m.group(2)] = (m.group(1), [] if params == ["void"] else params)
    return protos


def ctype_of(decl):
    """The ctypes type _lib.SIGNATURES gives a C declaration: scalars by exact width, `const char*` as c_char_p, pointers to the
    ABI's structs typed, every other pointer or array (buffers, handles, out-handles, streams) void*; void -> None."""
    structs = {"nidx_vec_config": _lib.VecConfig, "nidx_vec_search_params": _lib.VecSearchParams, "nidx_filter_node": _lib.FilterNode,
               "nidx_txt_search_params": _lib.TxtSearchParams, "nidx_txt_facet_request": _lib.TxtFacetRequest, "nidx_txt_order": _lib.TxtOrder,
               "nidx_rrf_source": _lib.RrfSource, "nidx_shard_search_request": _lib.ShardSearchRequest,
               "nidx_shard_search_response": _lib.ShardSearchResponse}
    scalars = {"int": C.c_int32, "int32_t": C.c_int32, "uint32_t": C.c_uint32, "int64_t": C.c_int64, "uint64_t": C.c_uint64, "float": C.c_float,
               "double": C.c_double}
    base = re.findall(r"\w+", re.sub(r"\bconst\b", " ", decl))[0]
    if "*" in decl or "[" in decl:
        return C.c_char_p if base == "char" else C.POINTER(structs[base]) if base in structs else C.c_void_p
    return None if base == "void" else scalars[base]


def test_signature_table_matches_the_header():
    """Every prototype of include/nidx_b200.h against _lib.SIGNATURES, parameter by parameter (a scalar of the wrong width, or
    a missing parameter, reaches the library as a wrong value without an error)."""
    protos = header_prototypes()
    assert len(protos) == len(header_functions())
    assert sorted(_lib.SIGNATURES) == sorted(protos)
    for name, (ret, params) in protos.items():
        restype, argtypes = _lib.SIGNATURES[name]
        assert restype is ctype_of(ret), (name, ret, restype)
        assert len(argtypes) == len(params), (name, params, argtypes)
        for i, (decl, t) in enumerate(zip(params, argtypes)):
            assert t is ctype_of(decl), (name, i, decl, t)
    L = _lib.load()
    assert L.nidx_vec_search.argtypes == _lib.SIGNATURES["nidx_vec_search"][1] and L.nidx_vec_len.restype is C.c_uint64


def test_wrappers_agree_with_the_signature_table():
    """Every VectorSegment / TextSegment wrapper that reaches its ABI call with numpy inputs, driven over a NULL handle: the
    library refuses it (NidxError).  A ctypes.ArgumentError or TypeError would mean a call site disagrees with the table.
    Not driven here (the GPU suite covers them): create / open (require_device first), close / len (no refusal to see), and
    the torch device path."""
    from nucliadb_b200.segment import TextSegment, VectorSegment

    vec = VectorSegment(None, _lib.VecConfig(8, _lib.NIDX_SIM_DOT, 0, 0, 0, 0, 0, 0))
    txt = TextSegment(None, 4, 3, 0)
    txt.facet_buckets = lambda facets: (np.zeros(2, np.uint32), np.zeros(2, np.uint32))   # reach the faceted calls themselves
    nodes = (_lib.FilterNode * 1)(_lib.FilterNode(_lib.NIDX_F_NOT, 0, None, None))
    q = np.zeros((2, 8), np.float32)
    qt, qoff = np.array([0, 1], np.uint32), np.array([0, 1, 2], np.uint32)
    level, adj = np.zeros(2, np.uint8), np.zeros((2, 4), np.uint32)
    calls = {
        "VectorSegment.save": lambda: vec.save("/nonexistent"),
        "VectorSegment.build_hnsw": lambda: vec.build_hnsw(seed=3, max_batch=64),
        "VectorSegment.extend_hnsw": lambda: vec.extend_hnsw(1, level, adj, adj, adj, adj, 0, 0, seed=3, max_batch=64),
        "VectorSegment.graph_dims": vec.graph_dims,
        "VectorSegment.get_graph": vec.get_graph,
        "VectorSegment.set_graph": lambda: vec.set_graph(level, adj, adj, adj, adj),
        "VectorSegment.set_alive": lambda: vec.set_alive(np.ones(1, np.uint64)),
        "VectorSegment.set_paragraph_keys": lambda: vec.set_paragraph_keys(np.arange(2)),
        "VectorSegment.set_inverted_index": lambda: vec.set_inverted_index(_lib.NIDX_INV_LABELS, [b"a", b"b"], [[0], [0, 1]]),
        "VectorSegment.filter": lambda: vec.filter(nodes, 1, np.zeros(1, np.uint64)),
        "VectorSegment.search": lambda: vec.search(q, 3, ef=16, min_score=0.5, with_duplicates=False, method=_lib.NIDX_METHOD_BRUTE),
        "VectorSegment.search(filter_bits)": lambda: vec.search(q, 3, filter_bits=np.ones(1, np.uint64), filter_matching=2),
        "VectorSegment.search(formula)": lambda: vec.search(q, 3, formula=nodes),
        "VectorSegment.rabitq_encode": vec.rabitq_encode,
        "VectorSegment.rabitq_codes": vec.rabitq_codes,
        "VectorSegment.rabitq_estimate": lambda: vec.rabitq_estimate(q),
        "VectorSegment.last_kernel_ms": vec.last_kernel_ms,
        "VectorSegment.counters": vec.counters,
        "VectorSegment.counters_ex": vec.counters_ex,
        "VectorSegment.exact_rows": vec.exact_rows,
        "VectorSegment.scan_counters": vec.scan_counters,
        "VectorSegment.walk_reruns": vec.walk_reruns,
        "TextSegment.set_stats": lambda: txt.set_stats(4, 10, np.ones(3)),
        "TextSegment.set_alive": lambda: txt.set_alive(np.ones(1, np.uint64)),
        "TextSegment.search": lambda: txt.search(qt, qoff, 3, mode=_lib.NIDX_BM25_AND, use_tf=False, min_score=0.1, after=(1.0, 2, 5), docaddr_base=1 << 32),
        "TextSegment.set_facets": lambda: txt.set_facets([b"a", b"a\0b"], np.zeros(5), np.zeros(0)),
        "TextSegment.facet_buckets": lambda: TextSegment.facet_buckets(txt, [b"a"]),
        "TextSegment.search_faceted": lambda: txt.search_faceted(qt, qoff, 3, [b"a"], after=(1.0, 1, 0)),
        "TextSegment.facet_count_all": lambda: txt.facet_count_all([b"a"]),
        "TextSegment.set_dates": lambda: txt.set_dates(np.zeros(4), np.zeros(4)),
        "TextSegment.search_ordered": lambda: txt.search_ordered(qt, qoff, 3, field=_lib.NIDX_ORDER_MODIFIED, order=_lib.NIDX_ORDER_ASC),
        "TextSegment.search_ordered(facets)": lambda: txt.search_ordered(qt, qoff, 3, facets=[b"a"]),
        "TextSegment.list_ordered": lambda: txt.list_ordered(3),
        "TextSegment.set_doc_keys": lambda: txt.set_doc_keys(np.arange(4)),
        "TextSegment.last_kernel_ms": txt.last_kernel_ms,
    }
    for name, call in calls.items():
        with pytest.raises(_lib.NidxError):
            call()
            pytest.fail(f"{name} was not refused")


def test_library_exports_every_header_symbol():
    L = _lib.load()
    names = header_functions()
    assert names, "no functions parsed from the header"
    for n in names:
        assert hasattr(L, n), f"libnidx_b200.so does not export {n}"
    assert sorted(_lib.SYMBOLS) == names


def test_library_does_not_link_the_oracle():
    out = os.popen(f"nm -D --defined-only {_lib.LIB_PATH}").read()
    assert "oracle_" not in out
    for f in ("vector.py", "text.py", "segment.py", "dist.py", "_lib.py", "__init__.py"):
        src = open(os.path.join(ROOT, "nucliadb_b200", f)).read()
        assert "import oracle" not in src and "from oracle" not in src


def test_no_device_fails_loudly():
    L = _lib.load()
    if L.nidx_device_count() > 0:
        pytest.skip("a CUDA device is present")
    cfg = _lib.VecConfig(8, _lib.NIDX_SIM_COSINE, 0, 0, 0, 0, 0, 0)
    h = C.c_void_p()
    v = np.zeros((4, 8), dtype=np.float32)
    rc = L.nidx_vec_create(C.byref(cfg), _lib.ptr(v), C.c_uint64(4), C.c_int32(8), _lib.NIDX_MEM_HOST, None, C.byref(h))
    assert rc == -2 and b"no CUDA device" in L.nidx_last_error()
    out = (C.c_uint64 * 2)()
    assert L.nidx_vec_scan_counters(None, out) != 0 and b"null" in L.nidx_last_error()
    with pytest.raises(_lib.NidxError):
        _lib.require_device()
    from nucliadb_b200.segment import VectorSegment
    with pytest.raises(_lib.NidxError):
        VectorSegment.create(v, 8)


def test_cost_model_is_a_host_function_equal_to_the_oracle():
    """nidx_use_hnsw (segment.rs:626-660) needs no device; same decisions as the oracle's restatement on a grid, with and
    without RaBitQ, including SURVEY F6's known point (100 k unfiltered vectors, k = 10 => HNSW)."""
    import ctypes as C

    import oracle as O

    L = _lib.load()
    call =lambda t, mt, k, rq, m=30: bool(L.nidx_use_hnsw(C.c_uint64(t), C.c_uint64(mt), C.c_uint64(k), C.c_int(int(rq)), C.c_int(m)))
    assert call(100_000, 100_000, 10, False) and not call(100_000, 500, 10, False)
    for total in (1, 7, 640, 5_000, 100_000, 10_000_000):
        for frac in (1.0, 0.3, 0.01, 0.0001):
            matching = max(1, int(total * frac))
            for k in (1, 5, 10, 100):
                for rq in (False, True):
                    for m in (16, 30):
                        assert call(total, matching, k, rq, m) == O.use_hnsw(total, matching, k, has_rabitq=rq, M=m), (total, matching, k, rq, m)


def test_ctypes_structures_have_the_header_layout(tmp_path):
    """sizeof / offsetof of every struct of include/nidx_b200.h, as gcc lays it out, against the ctypes mirrors in nucliadb_b200/_lib.py
    (a drift here corrupts arguments silently)."""
    import ctypes as C
    import subprocess

    from nucliadb_b200 import _lib as L

    pairs = [("nidx_vec_config", L.VecConfig), ("nidx_vec_search_params", L.VecSearchParams), ("nidx_txt_search_params", L.TxtSearchParams),
             ("nidx_filter_node", L.FilterNode), ("nidx_rrf_source", L.RrfSource), ("nidx_shard_search_request", L.ShardSearchRequest),
             ("nidx_shard_search_response", L.ShardSearchResponse)]
    lines = ['#include <stdio.h>', '#include <stddef.h>', f'#include "{os.path.join(ROOT, "include", "nidx_b200.h")}"', "int main(void) {"]
    for cname, ct in pairs:
        lines.append(f'printf("{cname} %zu", sizeof({cname}));')
        for fname, _ in ct._fields_:
            lines.append(f'printf(" %zu", offsetof({cname}, {fname}));')
        lines.append('printf("\\n");')
    lines += ["return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c11", "-o", str(exe), str(src)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.strip().splitlines()
    for (cname, ct), line in zip(pairs, out):
        got = [int(x) for x in line.split()[1:]]
        want = [C.sizeof(ct)] + [getattr(ct, f).offset for f, _ in ct._fields_]
        assert got == want, (cname, got, want)
