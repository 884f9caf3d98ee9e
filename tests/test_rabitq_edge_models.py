"""The oracle's RaBitQ (oracle/rabitq.hpp) against a numpy float32 transcription of the reference (vector_types/rabitq.rs:75-244,
segment.rs:581-608) on the numeric edges the GPU tests feed: rows with dot_quant_original > 1, zero rows, rows with sum_bits = 0
or d, rows holding NaN or +-inf, and constant, >= 256, +-inf, NaN and subnormal queries.  Every float operation is written out
in the reference's order; Rust's `as u64` is written out by hand (NaN -> 0, negative -> 0, truncation, saturation at u64::MAX),
which `astype(np.uint64)` is not.  This pins the oracle that test_gpu_rabitq_edges.py compares the kernels with."""
import heapq
import math

import numpy as np
import pytest

import oracle as O
from rabitq_edge_inputs import edge_queries, edge_rows, f32, same_bits, same_codes

U64_MAX = (1 << 64) - 1


def as_u64(x):
    """Rust's `f32 as u64`: NaN -> 0, values <= 0 -> 0, truncation toward zero, saturation at u64::MAX (inf included)."""
    x = float(x)
    if math.isnan(x) or x <= 0.0:
        return 0
    if x >= 2.0 ** 64:
        return U64_MAX
    return int(x)


def test_as_u64_is_rusts_saturating_cast():
    assert [as_u64(x) for x in (np.nan, -np.nan, -1.5, -0.0, 0.0, 0.999, 1.0, 15.99, 16.0, 2.0 ** 63, 2.0 ** 64, np.inf, -np.inf)] == \
        [0, 0, 0, 0, 0, 0, 1, 15, 16, 1 << 63, U64_MAX, U64_MAX, 0]


def model_encode(v):
    """rabitq.rs:75-106.  dot(v, v_repr) in the oracle's lane-blocked order (distance.hpp dot_ordered: acc[i % 128] by fma in
    increasing i, then (a0 + a1) + (a2 + a3) per lane and the 32-lane butterfly).  With d a power of four, 1 / sqrt(d) is a power
    of two, so every product is exact and each fma is one float32 add."""
    n, d = v.shape
    assert d in (64, 256, 1024, 4096)
    root_dim = f32(np.sqrt(f32(d)))
    pos, neg = f32(f32(1.0) / root_dim), f32(f32(-1.0) / root_dim)
    bits = v > f32(0.0)
    repr_ = np.where(bits, pos, neg).astype(f32)
    with np.errstate(all="ignore"):
        prod = (v * repr_).astype(f32)
        acc = np.zeros((n, 128), f32)
        for i in range(0, d, 128):
            blk = prod[:, i : i + 128]
            acc[:, : blk.shape[1]] = acc[:, : blk.shape[1]] + blk
        lanes = ((acc[:, 0::4] + acc[:, 1::4]) + (acc[:, 2::4] + acc[:, 3::4])).astype(f32)
        off = 16
        while off >= 1:
            lanes[:, :off] = lanes[:, :off] + lanes[:, off : 2 * off]
            off //= 2
    dqo = lanes[:, 0].copy()
    sum_bits = bits.sum(1).astype(np.uint32)
    words = np.packbits(bits, axis=1, bitorder="little")              # u64 little-endian words: bit i % 64 of word i / 64
    return np.concatenate([dqo.view(np.uint8).reshape(n, 4), sum_bits.view(np.uint8).reshape(n, 4), words], axis=1), dqo, sum_bits, bits


def model_query(q):
    """rabitq.rs:124-157: the sequential min / max fold from q[0] (a NaN is never `<` or `>`: NaN first sticks, NaN later is
    skipped), hi += 0.00001, delta = (hi - low) / 16, wq = ((q_i - low) / delta) as u64, four bit planes (wq / 2^p) % 2, and
    sum_quantized = (sum of wq as u64) as u32."""
    d = q.size
    low, hi = q[0], q[0]
    for x in q:
        low = x if x < low else low
        hi = x if x > hi else hi
    with np.errstate(all="ignore"):
        hi = f32(hi + f32(0.00001))
        delta = f32(f32(hi - low) / f32(16.0))
        wq = [as_u64(f32(f32(x - low) / delta)) for x in q]
    planes = np.zeros((4, d // 64), np.uint64)
    for p in range(4):
        for i, w in enumerate(wq):
            planes[p, i // 64] += np.uint64(((w >> p) % 2) << (i % 64))
    return planes, f32(low), delta, (sum(wq) % (1 << 64)) % (1 << 32), wq


def model_similarity(wq, low, delta, sum_q, dqo, sum_bits, bits, d):
    """rabitq.rs:166-218 for every row: the weighted popcount, then the estimate and the error bound in float32, in order."""
    root_dim = f32(np.sqrt(f32(d)))
    w = np.array(wq, dtype=np.int64)
    dot = np.array([sum(int(((w >> p) & 1)[bits[i]].sum()) << p for p in range(4)) for i in range(len(bits))], np.int64)
    with np.errstate(all="ignore"):
        t1 = f32(f32(f32(2.0) * delta) / root_dim) * dot.astype(f32)
        t2 = (f32(f32(2.0) * low) * sum_bits.astype(f32)) / root_dim
        t3 = f32(f32(delta * f32(sum_q)) / root_dim)
        t4 = f32(low * root_dim)
        dqq = ((t1 + t2).astype(f32) - t3).astype(f32) - t4
        est = (dqq.astype(f32) / dqo).astype(f32)
        d2 = (dqo * dqo).astype(f32)
        err = ((np.sqrt(((f32(1.0) - d2) / d2).astype(f32)).astype(f32) * f32(1.9)).astype(f32) / root_dim).astype(f32)
    return est, err


def _ordered(score):
    """f32::total_cmp as an integer (the oracle's ordered_bits): with the lower id first on equal scores."""
    u = int(np.float32(score).view(np.uint32))
    return (~u & 0xFFFFFFFF) if u & 0x80000000 else (u | 0x80000000)


def model_scan(v, est, err, q, k, min_score):
    """segment.rs:581-608 + rabitq.rs:222-244: upper_bound = estimate + error, candidates with upper_bound >= min_score in address
    order, rerank_top evaluating the exact similarity iff `best.len() < k || best_k < upper_bound`."""
    best, best_k, n_exact = [], f32(0.0), 0                          # min-heap of (rank, id) = BinaryHeap<Reverse<Cnx>>
    with np.errstate(all="ignore"):
        up = (est + err).astype(f32)
    for addr in range(len(v)):
        if not up[addr] >= f32(min_score):
            continue
        if len(best) < k or best_k < up[addr]:
            real = f32(O.dot(v[addr], q))
            n_exact += 1
            if real >= f32(min_score) and (len(best) < k or best_k < real):
                heapq.heappush(best, ((_ordered(real), -addr), addr, real))
                if len(best) > k:
                    heapq.heappop(best)
                best_k = best[0][2]
    want = sorted(best, reverse=True)
    return [x[1] for x in want], [x[2] for x in want], n_exact


@pytest.mark.parametrize("d", [64, 256])
def test_oracle_encode_query_and_estimate_equal_the_transcription_at_the_edges(d):
    v = edge_rows(300, d, seed=d)
    names, q = edge_queries(v, d, seed=d + 5)
    enc = O.rabitq_encode(v)
    want, dqo, sum_bits, bits = model_encode(v)
    assert same_codes(enc, want)
    assert (dqo[np.isfinite(dqo)] > 1).sum() > 50                    # rows whose error bound is NaN are well represented
    est_all, err_all = O.rabitq_estimate(enc, d, q)
    for qi, name in enumerate(names):
        planes, low, delta, sum_q, wq = model_query(q[qi])
        oplanes, olow, odelta, osum = O.rabitq_query(q[qi])
        assert np.array_equal(oplanes, planes), name
        assert same_bits(f32(olow), low) and same_bits(f32(odelta), delta) and osum == sum_q, name
        est, err = model_similarity(wq, low, delta, sum_q, dqo, sum_bits, bits, d)
        assert same_bits(est_all[qi], est) and same_bits(err_all[qi], err), name
        if name == "max_300":
            assert max(wq) == 16                                     # counted in sum_quantized, in no bit plane
        if name == "const_256":
            assert delta == 0 and sum_q == 0
        if name == "const_255":
            assert delta > 0 and sum_q == 0


@pytest.mark.parametrize("d", [64, 256])
def test_oracle_scan_equals_the_transcription_at_the_edges(d):
    n = 300
    v = edge_rows(n, d, seed=d + 1)
    names, q = edge_queries(v, d, seed=d + 6)
    enc = O.rabitq_encode(v)
    est, err = O.rabitq_estimate(enc, d, q)
    for k, ms in ((1, -1.0), (10, -1.0), (10, 0.0), (n + 3, -np.inf), (10, 1e30)):
        ids, sc, cnt, evals = O.rabitq_brute_force(v, enc, q, k, min_score=ms)
        for qi, name in enumerate(names):
            wi, ws, wn = model_scan(v, est[qi], err[qi], q[qi], k, ms)
            assert cnt[qi] == len(wi) and evals[qi] == wn, (name, k, ms)
            assert ids[qi, : cnt[qi]].tolist() == wi and same_bits(sc[qi, : cnt[qi]], np.array(ws, f32)), (name, k, ms)
