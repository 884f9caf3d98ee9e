"""CPU check of the tensor-core filter of the exhaustive scan (scan_tc2.cuh).

1. The bound: a model of the filter's approximate score -- operands truncated to tf32, the f32 sum taken as a sequential sum
   rounded toward zero (the worst case the header comment allows for the tensor cores' undocumented order), the cosine epilogue
   with frcp_rn -- stays within eps(ld) of the exact lane-blocked score (the oracle's), on random and adversarial rows.
2. The selection: a restatement of the lists, tau, the survivors, the overflow test and the survivor cap, with the kernel's
   assignment of vectors to lists, fed approximations perturbed adversarially within +-eps: every true top-k member survives,
   or the query is flagged for the exact scan.
"""
import numpy as np
import pytest

import oracle as O

TC2_L, TC2_CHUNK, TC2_N, TC2_LISTS, TC2_SURV_CAP = 24, 2048, 128, 2, 512


def tc2_eps(ld):
    """tc2_eps() in f32, as the kernel computes it."""
    return max(np.float32(2.2e-3), np.float32(np.float32(2.0 ** -9 + 2.0 ** -20) + np.float32((ld + 64) * 2.0 ** -23)))


def tf32(x):
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)


def add_rz(a, b):
    """f32 a + b rounded toward zero (elementwise, exact: two-sum in f64, then the f32 neighbour towards zero)."""
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    s = a64 + b64
    bb = s - a64
    err = (a64 - (s - bb)) + (b64 - bb)
    r = s.astype(np.float32)
    below = ((s - r.astype(np.float64)) + err)        # sign of (exact - r)
    toward = ((r > 0) & (below < 0)) | ((r < 0) & (below > 0))
    return np.where(toward, np.nextafter(r, np.float32(0)), r).astype(np.float32)


def approx_dots(q, V):
    """The filter's tf32 dot of q with every row of V, accumulated sequentially in f32 with round-toward-zero."""
    p = tf32(V) * tf32(q)[None, :]                      # products of tf32 operands are exact in f32
    acc = np.zeros(V.shape[0], np.float32)
    for i in range(V.shape[1]):
        acc = add_rz(acc, p[:, i])
    return acc


def rcp_rn(x):
    return (1.0 / np.asarray(x, np.float64)).astype(np.float32)


def approx_scores(q, V, sim):
    a = approx_dots(q, V)
    if sim == O.SIM_DOT:
        return a
    qn, vn = O.norms(q[None, :])[0], O.norms(V)
    return (a * rcp_rn(qn)) * rcp_rn(vn)               # sc * inv_qn * ivn, f32 products


def exact_scores(q, V, sim):
    f = O.dot if sim == O.SIM_DOT else O.cosine
    return np.asarray([f(q, v) for v in V], np.float32)


def low_bits_set(x):
    """Every element loses the most to tf32 truncation: its 13 low mantissa bits set."""
    return (np.ascontiguousarray(x, np.float32).view(np.uint32) | np.uint32(0x1FFF)).view(np.float32)


def absorption(ld):
    """q = v = (x, e, ..., e), x = 1 + 2^-10 - 2^-23 (truncates to 1), e a tf32 value with e^2 just below 2^-23: each e^2 is
    absorbed by a round-toward-zero sum at 1, and the operand error adds 2^-9 on top."""
    e = np.float32(1.4140625 * 2.0 ** -12)
    v = np.full(ld, e, np.float32)
    v[0] = np.float32(1 + 2.0 ** -10 - 2.0 ** -23)
    return v


def rows(rng, n, ld):
    g = rng.standard_normal((n, ld)).astype(np.float32)
    unit = g / np.linalg.norm(g, axis=1, keepdims=True)
    scaled = unit * (10.0 ** rng.uniform(-15, 15, (n, 1))).astype(np.float32)
    spread = g * (10.0 ** rng.uniform(-6, 6, (n, ld))).astype(np.float32)
    return np.concatenate([unit, scaled, spread, low_bits_set(np.abs(unit)), low_bits_set(unit)]).astype(np.float32)


@pytest.mark.parametrize("sim", [O.SIM_DOT, O.SIM_COSINE])
@pytest.mark.parametrize("ld", [64, 384, 768, 1024, 1536, 2048, 3072, 4096])
def test_approximate_score_is_within_eps_of_the_exact_score(sim, ld):
    rng = np.random.default_rng(ld + sim)
    V = np.concatenate([rows(rng, 6, ld), absorption(ld)[None, :]])
    g = rng.standard_normal(ld).astype(np.float32)
    queries = [g / np.linalg.norm(g), low_bits_set(np.abs(g / np.linalg.norm(g))), absorption(ld), g * np.float32(1e6)]
    eps = tc2_eps(ld)
    vn = O.norms(V).astype(np.float64)
    for q in queries:
        err = np.abs(approx_scores(q, V, sim).astype(np.float64) - exact_scores(q, V, sim))
        bound = eps if sim == O.SIM_COSINE else eps * O.norms(q[None, :])[0].astype(np.float64) * vn
        assert (err <= bound).all(), (ld, np.max(err / bound))


@pytest.mark.parametrize("sim", [O.SIM_DOT, O.SIM_COSINE])
def test_a_fixed_eps_of_2_2e_3_fails_at_4096_dimensions(sim):
    """What eps(ld) adds: the accumulation term.  At ld = 4096 the absorption input is off by 2.43e-3 of |q||v|, above the
    2.2e-3 that was enough up to ld ~ 2000 (eps(ld) equals 2.2e-3 there) and below eps(4096)."""
    v = absorption(4096)
    err = abs(float(approx_scores(v, v[None, :], sim)[0]) - float(exact_scores(v, v[None, :], sim)[0]))
    scale = 1.0 if sim == O.SIM_COSINE else float(O.norms(v[None, :])[0]) ** 2
    assert 2.2e-3 * scale < err <= tc2_eps(4096) * scale
    assert tc2_eps(1984) == np.float32(2.2e-3) and tc2_eps(384) == np.float32(2.2e-3)


# ---- 2. the selection -----------------------------------------------------------------------------------------------------

def list_of(n, slots):
    """(slot, column half) list index of every vector: CTA slot s walks chunks s, s + slots, ...; thread = (row, column half)."""
    v = np.arange(n)
    return ((v // TC2_CHUNK) % slots) * TC2_LISTS + (v % TC2_N) // (TC2_N // TC2_LISTS)


def filter_lists(approx, elig, slots):
    """scan_tc_filter_kernel's lists for one query: each list sees its vectors in increasing id order and keeps the best TC2_L
    (a candidate enters when it beats the smallest entry; when full it replaces the first smallest entry)."""
    lists = []
    owner = list_of(len(approx), slots)
    for l in range(slots * TC2_LISTS):
        ls, li = [-np.inf] * TC2_L, [None] * TC2_L
        cnt, minpos, thr = 0, 0, -np.inf
        for v in np.nonzero((owner == l) & elig)[0]:
            sc = approx[v]
            if sc > thr:
                pos = cnt if cnt < TC2_L else minpos
                ls[pos], li[pos] = sc, int(v)
                cnt = min(cnt + 1, TC2_L)
                if cnt == TC2_L:
                    minpos = int(np.argmin(ls))
                    thr = ls[minpos]
        lists.append((ls, li))
    return lists


def refine(lists, k, eps):
    """scan_tc_refine_kernel's selection: (survivor ids, flagged for the exact scan)."""
    entries = [(s, i) for ls, li in lists for s, i in zip(ls, li) if i is not None]
    scores = sorted((s for s, _ in entries), reverse=True)
    tau = np.float32(scores[k - 1]) if len(scores) >= k else np.float32(-np.inf)
    margin = np.float32(2) * np.float32(eps)
    lo = np.float32(tau - margin)
    if tau == np.inf or np.isnan(lo):
        return set(), True
    overflow = any(all(i is not None for i in li) and min(ls) >= lo for ls, li in lists)
    surv = {i for s, i in entries if s >= lo}
    return surv, overflow or len(surv) > TC2_SURV_CAP


def exact_topk(exact, elig, k):
    ids = np.nonzero(elig)[0]
    order = sorted(ids, key=lambda v: (-exact[v], v))
    return set(int(v) for v in order[:k])


def check_selection(exact, elig, k, eps, slots, rng):
    top = exact_topk(exact, elig, k)
    flagged_any, ran = False, False
    perturbations = {
        "top_down": lambda: np.where(np.isin(np.arange(len(exact)), list(top)), -eps, eps),
        "random": lambda: rng.uniform(-eps, eps, len(exact)),
        "zero": lambda: np.zeros(len(exact)),
    }
    for name, pert in perturbations.items():
        approx = (exact.astype(np.float64) + pert()).astype(np.float32)
        approx = np.clip(approx, exact - np.float32(eps), exact + np.float32(eps))     # f32 rounding stays within eps
        surv, flagged = refine(filter_lists(approx, elig, slots), k, eps)
        assert flagged or top <= surv, (name, sorted(top - surv))
        flagged_any |= flagged
        ran |= not flagged
    return flagged_any, ran


@pytest.mark.parametrize("k", [1, 10, 16])
@pytest.mark.parametrize("slots", [1, 3])
def test_every_true_top_k_member_survives_or_the_query_is_flagged(k, slots):
    rng = np.random.default_rng(k * 7 + slots)
    eps = tc2_eps(384)
    n = 3 * TC2_CHUNK + 77
    for case in range(6):
        exact = rng.uniform(-0.2, 0.8, n).astype(np.float32)
        if case == 1:       # a crowd within 2 eps of the k-th score, spread over every list
            exact[rng.choice(n, 300, replace=False)] = np.float32(0.9) + rng.uniform(-2 * eps, 2 * eps, 300).astype(np.float32)
        if case == 2:       # the crowd packed into one list: it must overflow or keep the top
            crowd = np.arange(64, 64 + 40 * 128, 128)[:40]
            exact[crowd] = np.float32(0.9) + rng.uniform(-eps, eps, len(crowd)).astype(np.float32)
        if case == 3:       # exact ties at the top
            exact[rng.choice(n, 50, replace=False)] = np.float32(0.95)
        if case == 4:       # fewer eligible vectors than k in some lists, and overall close to k
            exact[:] = -1.0
            exact[rng.choice(n, k + 3, replace=False)] = rng.uniform(0, 1, k + 3).astype(np.float32)
        if case == 5:       # near-ties in every list, each holding fewer than TC2_L of them: no list overflows
            exact[:] = rng.uniform(-0.2, 0.5, n).astype(np.float32)
            per_list = 20
            owner = list_of(n, slots)
            for l in range(slots * TC2_LISTS):
                members = np.nonzero(owner == l)[0][:per_list]
                exact[members] = np.float32(0.9) + rng.uniform(-0.5 * eps, 0.5 * eps, len(members)).astype(np.float32)
        elig = rng.random(n) < 0.9
        flagged_any, ran = check_selection(exact, elig, k, eps, slots, rng)
        if case == 5:       # built so that no list overflows and the survivors stay under the cap: the filter's selection serves them
            assert ran and not flagged_any


def test_the_survivor_cap_flags_without_an_overflowing_list():
    """22 lists x 24 > 512: with 23 near-ties in each of 24 lists (12 slots) no list overflows, but the survivors exceed the cap."""
    slots, k, eps = 12, 10, tc2_eps(384)
    n = slots * TC2_CHUNK
    exact = np.full(n, -0.5, np.float32)
    owner = list_of(n, slots)
    for l in range(slots * TC2_LISTS):
        exact[np.nonzero(owner == l)[0][:23]] = np.float32(0.9)
    lists = filter_lists(exact, np.ones(n, bool), slots)
    assert not any(all(i is not None for i in li) and min(ls) >= 0.9 - 2 * eps for ls, li in lists)
    surv, flagged = refine(lists, k, eps)
    assert len(surv) == 23 * 24 > TC2_SURV_CAP and flagged


def test_non_finite_tau_is_flagged():
    eps = tc2_eps(384)
    n = TC2_CHUNK
    for bad in (np.inf, np.nan):
        approx = np.zeros(n, np.float32)
        approx[5] = np.float32(bad) if bad == np.inf else np.float32(0)
        e = np.float32(eps) if bad == np.inf else np.float32(np.nan)
        surv, flagged = refine(filter_lists(approx, np.ones(n, bool), 1), 1, e)
        assert flagged
