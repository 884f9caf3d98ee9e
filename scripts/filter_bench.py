"""Paragraph filters on the device: nidx_vec_filter per formula shape, nidx_vec_search_formula (batch 16, BRUTE and HNSW) and the
prefilter hand-off nidx_vec_prefilter_bits with and without a formula, on vector segments of 1 M and 10 M paragraphs with a label
index (1 000 labels of Zipf popularity, 3 per paragraph, a tenth of them with a sub-label) and a field index (4 paragraphs per field).

Each call is timed on the host around the call, which returns after a synchronise.  Given several builds of the library (--libs, file
names next to nucliadb_b200/_lib.py), one process per build and round runs the same seeded cases, the builds alternating round by
round; the outputs (bits, counts, ids, scores) must be byte-identical across builds, and the spread of one build's round medians is
reported beside the medians.  One JSON line, with the card's name and power limit.

    python scripts/filter_bench.py [--libs libnidx_b200.so,...] [--paragraphs 1000000,10000000] [--rounds 3] [--steps 20] [--warmup 3]
"""
import argparse
import hashlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

N_LABELS, LABELS_PER_PAR, PARS_PER_FIELD, DIM, NQ, K = 1000, 3, 4, 16, 16, 10


def label_key(i, sub=False):
    return b"/l/%04d%s" % (i, b"/s" if sub else b"")


def build_indexes(seg, n, rng):
    """-> the label and field keys; the postings go to the segment"""
    from nucliadb_b200 import _lib

    ranks = np.arange(1, N_LABELS + 1, dtype=np.float64) ** -1.07
    lab = rng.choice(N_LABELS, (n, LABELS_PER_PAR), p=ranks / ranks.sum())
    sub = rng.random((n, LABELS_PER_PAR)) < 0.1
    codes = np.unique(np.stack([np.repeat(np.arange(n), LABELS_PER_PAR), (lab * 2 + sub).ravel()], 1), axis=0)   # (paragraph, key code)
    order = np.lexsort((codes[:, 0], codes[:, 1]))
    par, code = codes[order, 0].astype(np.uint32), codes[order, 1]
    used = np.unique(code)
    keys = [label_key(c // 2, bool(c % 2)) for c in used]                   # /l/NNNN sorts before /l/NNNN/s: code order is key order
    counts = np.searchsorted(code, used, side="right") - np.searchsorted(code, used, side="left")
    set_index(seg, _lib.NIDX_INV_LABELS, keys, counts, par)
    n_fields = (n + PARS_PER_FIELD - 1) // PARS_PER_FIELD
    fkeys = [b"%016d" % i for i in range(n_fields)]
    fcounts = np.full(n_fields, PARS_PER_FIELD)
    fcounts[-1] = n - PARS_PER_FIELD * (n_fields - 1)
    set_index(seg, _lib.NIDX_INV_FIELDS, fkeys, fcounts, np.arange(n, dtype=np.uint32))
    return fkeys


def set_index(seg, which, keys, counts, post):
    from nucliadb_b200 import _lib

    key_off = np.zeros(len(keys) + 1, dtype=np.uint64)
    key_off[1:] = np.cumsum([len(k) for k in keys])
    post_off = np.zeros(len(keys) + 1, dtype=np.uint64)
    post_off[1:] = np.cumsum(counts)
    key_bytes = np.frombuffer(b"".join(keys), dtype=np.uint8)
    _lib.check(_lib.load().nidx_vec_set_inverted_index(seg._h, which, len(keys), _lib.ptr(key_bytes), _lib.ptr(key_off), _lib.ptr(post_off),
                                                       _lib.ptr(np.ascontiguousarray(post))))


def set_random_graph(seg, n, rng, m0=16):
    """A one-layer graph of m0 random neighbours per node: the walk's cost without a graph build of 10 M nodes"""
    adj0 = np.full((n, (m0 + 31) // 32 * 32), 0xFFFFFFFF, dtype=np.uint32)   # rows padded to the segment's stride with NIL
    adj0[:, :m0] = rng.integers(0, n, (n, m0), dtype=np.uint32)
    seg.set_graph(np.zeros(n, dtype=np.uint8), adj0, np.zeros((1, 1), np.uint32))


def formulas(fkeys, rng):
    L = lambda i: ("label", label_key(i))   # noqa: E731
    keys = lambda m: ("keys", [fkeys[int(i)] for i in rng.integers(0, len(fkeys), m)])   # noqa: E731
    deep = L(3)
    for d in range(1, 8):
        sib = L(int(rng.integers(0, 200))) if d % 2 else keys(50)
        deep = (("and", "or", "not")[d % 3], [deep, sib])
    return {
        "one_label": L(2),
        "or_64_labels": ("or", [L(i) for i in range(10, 74)]),
        "and_3_atoms": ("and", [L(1), ("label", b"/l/00"), keys(2000)]),
        "not_and_2": ("not", [L(1), L(5)]),
        "mixed_8_deep": deep,
    }


def nodes_of(t, keep):
    import ctypes as C

    from nucliadb_b200 import _lib

    flat = []

    def walk(t):
        kind, arg = t
        if kind in ("label", "keys"):
            ks = [arg] if kind == "label" else list(arg)
            bufs = [C.create_string_buffer(k, len(k)) for k in ks]
            arr = (C.c_void_p * len(ks))(*[C.addressof(b) for b in bufs])
            lens = (C.c_uint32 * len(ks))(*[len(k) for k in ks])
            keep.extend([arr, lens, bufs])
            flat.append((_lib.NIDX_F_LABEL if kind == "label" else _lib.NIDX_F_KEYS, len(ks), arr, lens))
            return
        flat.append(({"and": _lib.NIDX_F_AND, "or": _lib.NIDX_F_OR, "not": _lib.NIDX_F_NOT}[kind], len(arg), None, None))
        for c in arg:
            walk(c)

    walk(t)
    nodes = (_lib.FilterNode * len(flat))()
    for i, (kind, n, arr, lens) in enumerate(flat):
        nodes[i].kind, nodes[i].n = kind, n
        if arr is not None:
            nodes[i].keys, nodes[i].key_len = arr, lens
    return nodes, len(flat)


def timed(fn, warmup, steps):
    for _ in range(warmup):
        fn()
    ms = []
    for _ in range(steps):
        t0 = time.perf_counter()
        fn()
        ms.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ms))


def worker(a):
    """One build: every case on every segment size -> {case: median ms}, {case: sha256 of the outputs}"""
    import ctypes as C

    from nucliadb_b200 import _lib
    from nucliadb_b200.segment import VectorSegment

    L = _lib.require_device()
    times, digests = {}, {}
    for n in a.paragraphs:
        rng = np.random.default_rng(n)
        seg = VectorSegment.create(rng.standard_normal((n, DIM)).astype(np.float32), DIM, similarity=_lib.NIDX_SIM_DOT, m=8, m0=16)
        fkeys = build_indexes(seg, n, rng)
        set_random_graph(seg, n, rng)
        alive = np.packbits(rng.random(((n + 63) // 64) * 64) < 0.97, bitorder="little").view(np.uint64).copy()
        seg.set_alive(alive)
        words = (n + 63) // 64
        keep = []
        out = np.empty(words, dtype=np.uint64)
        m = C.c_uint64()
        for name, t in formulas(fkeys, rng).items():
            nodes, nn = nodes_of(t, keep)
            fn = lambda: _lib.check(L.nidx_vec_filter(seg._h, nodes, nn, _lib.ptr(out), _lib.NIDX_MEM_HOST, C.byref(m), None))   # noqa: E731
            times[f"{n}/filter/{name}"] = timed(fn, a.warmup, a.steps)
            digests[f"{n}/filter/{name}"] = hashlib.sha256(out.tobytes() + bytes(m)).hexdigest()
        q = rng.standard_normal((NQ, DIM)).astype(np.float32)
        ids, sc, cnt = np.empty((NQ, K), np.uint32), np.empty((NQ, K), np.float32), np.empty(NQ, np.int32)
        mixed, nm = nodes_of(formulas(fkeys, np.random.default_rng(1))["mixed_8_deep"], keep)
        for method, mname in ((_lib.NIDX_METHOD_BRUTE, "brute"), (_lib.NIDX_METHOD_HNSW, "hnsw")):
            p = _lib.VecSearchParams(K, 64, -1e30, 1, method, None, 0)
            fn = lambda: _lib.check(L.nidx_vec_search_formula(seg._h, _lib.ptr(q), NQ, DIM, _lib.NIDX_MEM_HOST, C.byref(p), mixed, nm,   # noqa: E731
                                                              _lib.ptr(ids), _lib.ptr(sc), _lib.ptr(cnt), None))
            times[f"{n}/search_formula/{mname}"] = timed(fn, a.warmup, a.steps)
            digests[f"{n}/search_formula/{mname}"] = hashlib.sha256(ids.tobytes() + sc.tobytes() + cnt.tobytes()).hexdigest()
        n_docs = (n + PARS_PER_FIELD - 1) // PARS_PER_FIELD
        doc_bits = np.packbits(rng.random(((n_docs + 63) // 64) * 64) < 0.3, bitorder="little").view(np.uint64).copy()
        join = np.arange(n_docs, dtype=np.uint32)
        for name, (f, nf) in (("no_formula", (None, 0)), ("formula", (mixed, nm))):
            fn = lambda: _lib.check(L.nidx_vec_prefilter_bits(seg._h, _lib.ptr(doc_bits), n_docs, _lib.ptr(join), _lib.NIDX_F_AND, None, 0, None,   # noqa: E731
                                                              f, nf, _lib.NIDX_F_AND, _lib.ptr(out), _lib.NIDX_MEM_HOST, C.byref(m), None))
            times[f"{n}/prefilter_bits/{name}"] = timed(fn, a.warmup, a.steps)
            digests[f"{n}/prefilter_bits/{name}"] = hashlib.sha256(out.tobytes() + bytes(m)).hexdigest()
        seg.close()
    print(json.dumps(dict(times=times, digests=digests)))


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--libs", default="libnidx_b200.so", help="comma-separated builds of the library, file names next to nucliadb_b200/_lib.py")
    ap.add_argument("--paragraphs", default="1000000,10000000")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    a.paragraphs = [int(x) for x in a.paragraphs.split(",")]
    if a.worker:
        return worker(a)
    libs = a.libs.split(",")
    runs = {lib: [] for lib in libs}
    for _ in range(a.rounds):
        for lib in libs:
            env = dict(os.environ, NIDX_B200_LIB=lib)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", "--paragraphs", ",".join(map(str, a.paragraphs)), "--steps",
                                str(a.steps), "--warmup", str(a.warmup)], env=env, capture_output=True, text=True)
            if r.returncode:
                sys.exit(f"{lib}: worker failed\n{r.stderr[-4000:]}")
            runs[lib].append(json.loads(r.stdout.strip().splitlines()[-1]))
    ref = runs[libs[0]][0]["digests"]
    identical = all(run["digests"] == ref for lib in libs for run in runs[lib])
    out = {"identical_outputs": identical, "rounds": a.rounds, "steps": a.steps}
    for lib in libs:
        out[lib] = {case: dict(median_ms=round(float(np.median([r["times"][case] for r in runs[lib]])), 4),
                               spread_ms=round(float(np.ptp([r["times"][case] for r in runs[lib]])), 4)) for case in ref}
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    out["gpu"] = q.stdout.strip()
    print(json.dumps(out))
    if not identical:
        sys.exit("outputs differ between builds")


if __name__ == "__main__":
    main()
