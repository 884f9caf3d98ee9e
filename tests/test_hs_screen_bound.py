"""CPU check of the HNSW walk's fp16 screen: the error bound it adds to the fp16 dot must make the screened similarity rank at or
above the exact f32 similarity for every row it may reject, or the walk would drop a neighbour the f32 walk admits.  The encoder,
both dots and the test are restated in the kernels' order in tests/host/hs_screen_host.cpp (compiled with g++)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
SIM_DOT, SIM_COSINE, SIM_L2 = 0, 1, 2


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("hs_screen") / "hs_screen_host.so")
    subprocess.run(["g++", "-O1", "-std=c++17", "-frounding-math", "-ffp-contract=off", "-shared", "-fPIC", "-o", so,
                    os.path.join(HERE, "host", "hs_screen_host.cpp")], check=True)
    return C.CDLL(so)


def run(host, v, q, sim):
    v = np.ascontiguousarray(v, dtype=np.float32)
    q = np.ascontiguousarray(q, dtype=np.float32)
    n, ld = v.shape
    out = [np.zeros(n, np.float32) for _ in range(4)]
    scr = np.zeros(n, np.int32)
    p = lambda a: a.ctypes.data_as(C.c_void_p)
    bad = host.screen_rows(p(v), C.c_int(n), C.c_int(ld), p(q), C.c_int(sim), *[p(a) for a in out], p(scr))
    return bad, out, scr.astype(bool)


def pad(x, d):
    ld = (d + 3) // 4 * 4
    out = np.zeros((x.shape[0], ld), np.float32)
    out[:, :d] = x[:, :d]
    return out


def rows(rng, n, d):
    """Random rows, rows scaled by 1e-20 .. 1e20, rows whose elements span that range, fp16-subnormal elements, near copies."""
    g = rng.standard_normal((n, d)).astype(np.float32)
    unit = g / np.linalg.norm(g, axis=1, keepdims=True)
    scaled = unit * (10.0 ** rng.uniform(-20, 20, (n, 1))).astype(np.float32)
    spread = g * (10.0 ** rng.uniform(-20, 20, (n, d))).astype(np.float32)
    sub = unit.copy()
    sub[:, ::3] *= np.float32(1e-6)                     # below 2^-14 of the row's max after scaling: fp16 subnormals or zero
    near = unit[:1] + rng.normal(0, 1e-7, (n, d)).astype(np.float32)
    return np.concatenate([unit, scaled, spread, sub, near]).astype(np.float32)


@pytest.mark.parametrize("sim", [SIM_DOT, SIM_COSINE, SIM_L2])
@pytest.mark.parametrize("d", [96, 100, 384, 768, 1024])
def test_screen_bound_never_under_the_exact_score(host, sim, d):
    rng = np.random.default_rng(d * 3 + sim)
    v = pad(rows(rng, 40, d), d)
    queries = pad(np.concatenate([rows(rng, 2, d)[[0, 2, 4, 6, 8]], np.zeros((1, d), np.float32)]), d)
    for q in queries:
        bad, (s, s_up, ab, ab_up), scr = run(host, v, q, sim)
        assert bad == 0
        if np.abs(q).max() > 0:
            assert scr.sum() >= len(v) // 2               # most rows are screenable
    # unit rows against a unit query: the bound is tight enough to be useful
    bad, (s, s_up, ab, ab_up), scr = run(host, v[:40], queries[0], sim)
    assert bad == 0 and scr.all() and np.max(ab_up - ab) < 2e-3


@pytest.mark.parametrize("sim", [SIM_DOT, SIM_COSINE, SIM_L2])
def test_zero_and_nonfinite_rows(host, sim):
    d = 128
    rng = np.random.default_rng(1)
    v = rng.standard_normal((6, d)).astype(np.float32)
    v[0] = 0.0
    v[1, 3] = np.nan
    v[2, 4] = np.inf
    v[3, 5] = -np.inf
    v[4] = np.float32(3e38)                             # every element near FLT_MAX: the exact dot overflows
    q = rng.standard_normal(d).astype(np.float32)
    bad, (s, s_up, ab, ab_up), scr = run(host, v, q, sim)
    assert bad == 0
    assert scr[0] and scr[5]                            # a zero row and an ordinary one are screened
    assert not scr[1:5].any()                           # non-finite elements, and a dot that could overflow: always exact
    for bad_q in (np.full(d, np.nan, np.float32), np.full(d, np.inf, np.float32), np.full(d, 1e30, np.float32)):
        bad, _, scr = run(host, v, bad_q, sim)
        assert bad == 0 and not scr[1:5].any()
