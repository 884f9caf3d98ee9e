"""Rows and queries at the numeric edges of the RaBitQ estimator (vector_types/rabitq.rs:75-218), shared by the CPU model test
(test_rabitq_edge_models.py, which pins the oracle to a numpy transcription of the reference on exactly these inputs) and the GPU
test (test_gpu_rabitq_edges.py, which compares the kernels with the oracle on them)."""
import numpy as np

from conftest import make_queries, make_vectors

f32 = np.float32


def edge_rows(n, d, seed, nonfinite=True):
    """[n][d] Dot rows: unit rows scaled by 10^U(-3, 3) per row (so that about half have dot_quant_original > 1 and a NaN error
    bound), with a zero row, an all-negative row, an all-positive row and -- when `nonfinite` -- rows holding a NaN, a +inf or a
    -inf among finite elements.  The special rows sit at fixed places spread over the segment."""
    v = make_vectors(n, d, seed=seed)
    rng = np.random.default_rng(seed + 1)
    v *= (10.0 ** rng.uniform(-3, 3, n)).astype(f32)[:, None]
    v = v.astype(f32)
    at = [int(x) for x in np.linspace(0, n - 1, 7 if nonfinite else 4).round()]
    v[at[0]] = 0.0                                                  # dqo = 0: estimate +-inf (or NaN), error +inf
    v[at[1]] = -np.abs(v[at[1]]) - f32(1e-3)                        # sum_bits = 0
    v[at[2]] = np.abs(v[at[2]]) + f32(1e-3)                         # sum_bits = d
    if nonfinite:
        v[at[4], d // 3] = np.nan
        v[at[5], d // 2] = np.inf
        v[at[6], 1] = -np.inf
    return v


def edge_queries(v, d, seed, nonfinite=True):
    """Queries at the edges of QueryVector::from_vector, one per row, with a name each:
    near-data and random-normal queries; constant queries below and at magnitude 256 (delta = 0.00001 / 16, and delta = 0 where
    every (q - low) / delta is 0 / 0 = NaN and `as u64` gives 0); a query whose maximum is >= 256 (it quantises to 16, which no bit
    plane holds); elements spread over the subnormals; and -- when `nonfinite` -- +-inf elements (delta = inf) and NaN as the
    first element (low = hi = NaN) and as a later one (the min / max fold skips it)."""
    rng = np.random.default_rng(seed)
    qs = {
        "near": make_queries(np.nan_to_num(v[:64], posinf=0, neginf=0), 1, seed=seed)[0],
        "normal": rng.standard_normal(d).astype(f32),
        "const_3": np.full(d, 3.0, f32),
        "const_-3": np.full(d, -3.0, f32),
        "const_255": np.full(d, 255.0, f32),
        "const_256": np.full(d, 256.0, f32),
        "const_-300": np.full(d, -300.0, f32),
        "max_300": rng.standard_normal(d).astype(f32),
        "subnormal": (rng.standard_normal(d) * 1e-39).astype(f32),
    }
    qs["max_300"][d // 5] = 300.0
    if nonfinite:
        qs["plus_inf"] = rng.standard_normal(d).astype(f32)
        qs["plus_inf"][7] = np.inf
        qs["minus_inf"] = rng.standard_normal(d).astype(f32)
        qs["minus_inf"][d - 1] = -np.inf
        qs["nan_first"] = rng.standard_normal(d).astype(f32)
        qs["nan_first"][0] = np.nan
        qs["nan_later"] = rng.standard_normal(d).astype(f32)
        qs["nan_later"][d // 2 + 1] = np.nan
    names = list(qs)
    return names, np.stack([qs[k] for k in names]).astype(f32)


def same_bits(a, b):
    """Bitwise equality of two float32 arrays, a NaN equal to any NaN (the sign and payload of a NaN produced by arithmetic are not
    pinned: x86 produces 0xFFC00000, CUDA 0x7FFFFFFF)."""
    a, b = np.asarray(a, f32), np.asarray(b, f32)
    nan = np.isnan(a)
    return a.shape == b.shape and bool(np.array_equal(nan, np.isnan(b)) and np.array_equal(a.view(np.uint32)[~nan], b.view(np.uint32)[~nan]))


def same_codes(a, b):
    """vectors.quant records equal byte for byte, except that a NaN dot_quant_original equals any NaN."""
    a, b = np.asarray(a, np.uint8), np.asarray(b, np.uint8)
    return a.shape == b.shape and same_bits(a[:, :4].copy().view(f32), b[:, :4].copy().view(f32)) and bool(np.array_equal(a[:, 4:], b[:, 4:]))
