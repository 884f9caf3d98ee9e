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
    L.nidx_use_hnsw.restype = C.c_int
    call = lambda t, mt, k, rq, m=30: bool(L.nidx_use_hnsw(C.c_uint64(t), C.c_uint64(mt), C.c_uint64(k), C.c_int(int(rq)), C.c_int(m)))
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
