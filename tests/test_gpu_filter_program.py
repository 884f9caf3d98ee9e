"""Paragraph formulas as prefilter programs (nidx_vec_filter / nidx_vec_search_formula / nidx_vec_prefilter_bits): the device bits,
padding words included, and the counts against a literal host model of ParagraphInvertedIndexes::filter (inverted_index/paragraph.rs:
124-186) ANDed with the alive set, at the word edges of the paragraph space, at nesting depths past the bit stack, for wide formulas,
at the program limit, and with the launch count of a call."""
import bisect
import ctypes as C

import numpy as np
import pytest

from nucliadb_b200 import _lib
from nucliadb_b200 import vector as V
from nucliadb_b200.segment import VectorSegment

pytestmark = pytest.mark.gpu

N_LABELS, N_FIELDS = 6000, 2000


class Index:
    """A vector segment of n paragraphs with a label index (keys /l/NNNN and /l/NNNN/s, two labels per paragraph) and a field
    index (16-byte keys, one per paragraph), and the host model of a formula over them."""

    def __init__(self, n, seed=5):
        rng = np.random.default_rng(seed)
        self.n = n
        self.seg = VectorSegment.create(rng.standard_normal((n, 8)).astype(np.float32), 8, similarity=_lib.NIDX_SIM_DOT)
        labels = sorted([b"/l/%04d" % i for i in range(N_LABELS)] + [b"/l/%04d/s" % i for i in range(0, N_LABELS, 7)])
        self.labels = self._index(_lib.NIDX_INV_LABELS, labels, rng.integers(0, len(labels), (n, 2)))
        self.fields = self._index(_lib.NIDX_INV_FIELDS, [b"%016d" % i for i in range(N_FIELDS)], rng.integers(0, N_FIELDS, (n, 1)))
        self.alive = np.ones(n, dtype=bool)
        self.label_keys = labels
        self._atoms = {}

    def _index(self, which, keys, of_par):
        par = np.repeat(np.arange(self.n), of_par.shape[1])
        key = of_par.ravel()
        order = np.lexsort((par, key))
        counts = np.bincount(key, minlength=len(keys))
        post = np.split(par[order].astype(np.uint32), np.cumsum(counts)[:-1])
        post = [np.unique(p) for p in post]
        self.seg.set_inverted_index(which, keys, post)
        return dict(zip(keys, post))

    def set_alive(self, kind, rng):
        self.alive = {"all": np.ones(self.n, bool), "none": np.zeros(self.n, bool), "random": rng.random(self.n) < 0.6}[kind]
        words = np.zeros((self.n + 63) // 64 * 8, dtype=np.uint8)
        pb = np.packbits(self.alive, bitorder="little")
        words[: len(pb)] = pb
        if self.n % 64:
            words[len(pb) - 1] |= (0xFF << (self.n % 8)) & 0xFF
            words[len(pb):] = 0xFF   # the padding bits of the last word are set: they must not reach the result
        self.seg.set_alive(words.view(np.uint64))

    def model(self, t):
        kind, arg = t
        m = np.zeros(self.n, dtype=bool)
        if kind == "label":   # get_prefix: every key that starts with the label
            if arg not in self._atoms:
                i = bisect.bisect_left(self.label_keys, arg)
                while i < len(self.label_keys) and self.label_keys[i].startswith(arg):
                    m[self.labels[self.label_keys[i]]] = True
                    i += 1
                self._atoms[arg] = m
            return self._atoms[arg]
        if kind == "keys":    # get: the exact keys
            for k in arg:
                if k in self.fields:
                    m[self.fields[k]] = True
        else:
            parts = [self.model(c) for c in arg]
            acc = parts[0].copy()
            for p in parts[1:]:
                acc = acc | p if kind == "or" else acc & p
            m = ~acc if kind == "not" else acc   # NOT: the complement of the intersection (paragraph.rs:160-178)
        return m

    def expected(self, t):
        want = self.model(t) & self.alive
        words = np.zeros((self.n + 63) // 64 * 8, dtype=np.uint8)
        pb = np.packbits(want, bitorder="little")
        words[: len(pb)] = pb
        return words.view(np.uint64), int(want.sum())


def nodes_of(t):
    """A tree ('label', key) / ('keys', [keys]) / ('and' | 'or' | 'not', [operands]) -> (FilterNode array, n, keep-alive)."""
    flat, keep = [], []

    def walk(t):
        kind, arg = t
        if kind in ("label", "keys"):
            keys = [arg] if kind == "label" else list(arg)
            bufs = [C.create_string_buffer(k, max(len(k), 1)) for k in keys]
            arr = (C.c_void_p * max(len(keys), 1))(*[C.addressof(b) for b in bufs])
            lens = (C.c_uint32 * max(len(keys), 1))(*[len(k) for k in keys])
            keep.extend([arr, lens, bufs])
            flat.append((_lib.NIDX_F_LABEL if kind == "label" else _lib.NIDX_F_KEYS, len(keys), arr, lens))
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
    return nodes, len(flat), keep


def device_filter(ix, t, on_device=False):
    nodes, n, _keep = nodes_of(t)
    words = (ix.n + 63) // 64
    matching = C.c_uint64()
    L = _lib.load()
    if not on_device:
        out = np.full(words, 0xA5A5A5A5A5A5A5A5, dtype=np.uint64)
        _lib.check(L.nidx_vec_filter(ix.seg._h, nodes, n, _lib.ptr(out), _lib.NIDX_MEM_HOST, C.byref(matching), None))
        return out, matching.value
    import torch

    out = torch.full((words,), -0x5A5A5A5A5A5A5A5B, dtype=torch.int64, device="cuda")
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    _lib.check(L.nidx_vec_filter(ix.seg._h, nodes, n, C.c_void_p(out.data_ptr()), _lib.NIDX_MEM_DEVICE, C.byref(matching), stream))
    torch.cuda.synchronize()
    return out.cpu().numpy().view(np.uint64), matching.value


def check_filter(ix, t, on_device=False):
    got, matching = device_filter(ix, t, on_device)
    want, count = ix.expected(t)
    assert np.array_equal(got, want), t if len(repr(t)) < 300 else t[0]
    assert matching == count


def L(i):
    return ("label", b"/l/%04d" % i)


def K(*ids):
    return ("keys", [b"%016d" % i for i in ids])


def chain(depth, rng):
    """depth levels: each AND / OR / NOT over the level below and a sibling atom"""
    t = L(int(rng.integers(N_LABELS)))
    for d in range(1, depth):
        sib = L(int(rng.integers(N_LABELS))) if d % 2 else K(*rng.integers(0, N_FIELDS, 40))
        t = (("and", "or", "not")[d % 3], [t, sib] if d % 4 < 2 else [sib, t])
    return t


FORMULAS = [
    L(7),
    ("label", b"/l/00"),                                            # a prefix of many keys
    ("or", [L(1), L(2), K(3, 4, 5), ("label", b"/none")]),
    ("and", [("label", b"/l/0"), ("not", [L(11)]), K(*range(0, 2000, 3))]),
    ("not", [("label", b"/l/1"), ("label", b"/l/1"), ("or", [L(3), ("label", b"/l/10")])]),
    ("or", [("label", b"/none"), K(999999)]),                      # atoms that match nothing
]


@pytest.mark.parametrize("n", [1, 63, 64, 65, 4097, 262145])
def test_paragraph_edges_alive_sets_and_mem_paths(n):
    ix = Index(n)
    rng = np.random.default_rng(n)
    for alive in ("all", "none", "random"):
        ix.set_alive(alive, rng)
        for t in FORMULAS + [chain(5, rng)]:
            for on_device in (False, True):
                check_filter(ix, t, on_device)


@pytest.mark.parametrize("depth", [1, 2, 63, 64, 65, 200])
def test_nesting_chains(depth):
    ix = Index(4097)
    rng = np.random.default_rng(depth)
    ix.set_alive("random", rng)
    for _ in range(3):
        check_filter(ix, chain(depth, rng))


def test_wide_formulas():
    ix = Index(65537)
    rng = np.random.default_rng(1)
    ix.set_alive("random", rng)
    check_filter(ix, ("or", [L(int(i)) for i in rng.integers(0, N_LABELS + 500, 5000)]))              # some past the last key
    check_filter(ix, ("and", [("label", b"/l/") if i % 2 else ("label", b"/l") for i in range(500)]))
    check_filter(ix, ("and", [("label", b"/l/%d" % (i % 6)) if i % 3 else K(*range(i, 2000, 2)) for i in range(500)]))
    check_filter(ix, ("or", [L(3), ("and", [("label", b"/l/"), ("label", b"/none")])]))
    check_filter(ix, K(*rng.integers(0, N_FIELDS * 3 // 2, 1000)))                                      # a third missing
    check_filter(ix, ("not", [("label", b"/l/0"), ("label", b"/l/00"), ("not", [L(5)])]))


def test_program_limit():
    ix = Index(4097)
    atoms = [L(i) for i in range(2048)]
    check_filter(ix, ("not", [("and", atoms)]))                # 2048 leaves + 2047 ANDs + NOT = 4096 instructions
    nodes, n, _keep = nodes_of(("not", [("not", [("and", atoms)])]))
    m = C.c_uint64()
    with pytest.raises(_lib.NidxError):
        _lib.check(_lib.load().nidx_vec_filter(ix.seg._h, nodes, n, None, _lib.NIDX_MEM_HOST, C.byref(m), None))


def test_launches_per_call_do_not_grow_with_the_formula():
    ix = Index(4097)
    rng = np.random.default_rng(3)
    L_ = _lib.load()
    for t in (L(9), ("or", [L(i) for i in range(64)]), ("and", [L(1), ("label", b"/l/"), K(1, 2)]), ("not", [("and", [L(1), L(2)])]),
              chain(8, rng), chain(200, rng), ("and", [L(i) if i % 2 else K(i) for i in range(500)])):
        before = L_.nidx_launch_count()
        check_filter(ix, t)
        assert L_.nidx_launch_count() - before <= 2, t[0]


def has_postings(ix, t):
    kind, arg = t
    return bool(ix.model(t).any()) if kind in ("label", "keys") else any(has_postings(ix, c) for c in arg)


def test_prefilter_bits_text_and_resource_parts_with_and_without_a_formula():
    """The hand-off's text part (documents joined to field keys), resource part (runs of field keys) or both under doc_op, with and
    without a formula under op, against the host model; and its launches: one per part, one to scatter the formula's postings, and
    and_bits_kernel or the program's pass."""
    ix = Index(4097)
    rng = np.random.default_rng(8)
    ix.set_alive("random", rng)
    n_docs = 3000
    doc = rng.random(n_docs) < 0.3
    doc_words = np.zeros((n_docs + 63) // 64 * 8, dtype=np.uint8)
    pb = np.packbits(doc, bitorder="little")
    doc_words[: len(pb)] = pb
    keys = sorted(ix.fields)
    join = rng.integers(0, N_FIELDS + 100, n_docs).astype(np.uint32)   # some past the last key: no paragraphs
    join[rng.random(n_docs) < 0.1] = 0xFFFFFFFF
    joined = np.zeros(ix.n, dtype=bool)
    for d in np.flatnonzero(doc):
        if join[d] < N_FIELDS:
            joined[ix.fields[keys[join[d]]]] = True
    # resource r's paragraphs: the postings of the field keys [lo, hi) (a resource's fields are one run of keys; some runs are empty)
    n_res = 300
    runs = np.sort(rng.integers(0, N_FIELDS + 1, (n_res, 2)), axis=1)
    post_off = np.concatenate([[0], np.cumsum([len(ix.fields[k]) for k in keys])]).astype(np.uint64)
    res = rng.random(n_res) < 0.2
    res_words = np.zeros((n_res + 63) // 64 * 8, dtype=np.uint8)
    pr = np.packbits(res, bitorder="little")
    res_words[: len(pr)] = pr
    res_joined = np.zeros(ix.n, dtype=bool)
    for r in np.flatnonzero(res):
        for j in range(*runs[r]):
            res_joined[ix.fields[keys[j]]] = True
    L_ = _lib.load()
    for text, resources, doc_op in ((True, False, _lib.NIDX_F_AND), (False, True, _lib.NIDX_F_AND), (True, True, _lib.NIDX_F_AND),
                                    (True, True, _lib.NIDX_F_OR)):
        parts = dict(doc_bits=doc_words.view(np.uint64) if text else None, join=join if text else None, n_docs=n_docs if text else 0,
                     res_bits=res_words.view(np.uint64) if resources else None, res_ranges=post_off[runs] if resources else None,
                     n_res=n_res if resources else 0)
        matched = joined if not resources else res_joined if not text else joined & res_joined if doc_op == _lib.NIDX_F_AND else joined | res_joined
        for t in (None, L(4), chain(9, rng), ("or", [L(i) for i in range(40)])):
            for op in (_lib.NIDX_F_AND, _lib.NIDX_F_OR):
                nodes = None if t is None else nodes_of(t)
                before = L_.nidx_launch_count()
                bits, matching = ix.seg.prefilter_bits(**parts, n_paragraphs=ix.n, formula=None if t is None else nodes[0], op=op, doc_op=doc_op)
                launches = L_.nidx_launch_count() - before
                want = matched.copy()
                if t is not None:
                    want = want & ix.model(t) if op == _lib.NIDX_F_AND else want | ix.model(t)
                want &= ix.alive
                ww = np.zeros((ix.n + 63) // 64 * 8, dtype=np.uint8)
                pw = np.packbits(want, bitorder="little")
                ww[: len(pw)] = pw
                assert np.array_equal(bits, ww.view(np.uint64)), (t, op, text, resources, doc_op)
                assert matching == int(want.sum())
                assert launches == text + resources + (t is not None and has_postings(ix, t)) + 1, (t, op, text, resources)


def _open_segment():
    rng = np.random.default_rng(6)
    dim = 64
    cfg = V.VectorConfig(dimension=dim, similarity=V.Similarity.Dot)
    rids = [f"{i:032x}" for i in range(1, 41)]
    pool = ["/l/a", "/l/ab", "/l/a/x", "/l/b", "/k/c", "/k/c/deep", "/e/PERSON/one", "/e/PERSON/two"]
    elems = []
    for i in range(3000):
        labels = [lab for lab in pool if rng.random() < 0.25]
        field = rng.choice(["a/title", "a/summary", "f/file1", "t/text"])
        v = rng.standard_normal(dim).astype(np.float32)
        elems.append(V.Elem(f"{rids[i % len(rids)]}/{field}/{i}-{i + 1}", [v / np.linalg.norm(v)], labels=labels))
    return V.VectorIndexer.index_elems(elems, cfg), rids


def test_search_formula_equals_search_with_the_host_bitset():
    seg, rids = _open_segment()
    seg.apply_deletions([f"{rids[0]}/a/title"])
    rng = np.random.default_rng(2)
    q = rng.standard_normal((16, 64)).astype(np.float32)
    deep = V.Literal("/l/a")
    for d in range(70):
        sib = V.Literal(["/l/b", "/k/c", "/e/PERSON", "/l/a/x"][d % 4])
        deep = V.Not(V.Operation("and", (deep, sib))) if d % 3 == 0 else V.Operation("or" if d % 3 == 1 else "and", (sib, deep))
    for clauses in ([V.Literal("/l/a")], [V.Operation("or", tuple(V.Literal(p) for p in ["/l/b", "/k/c", "/none", "/e/PERSON/one"]))],
                    [V.Operation("and", (V.Literal("/l"), V._KeyPrefixSet(frozenset(f"{r}/a/title" for r in rids[:9])))), V.Not(V.Literal("/k/c"))],
                    [deep]):
        for method in (_lib.NIDX_METHOD_AUTO, _lib.NIDX_METHOD_BRUTE, _lib.NIDX_METHOD_HNSW):
            ids, sc, cnt = seg.search_batch(q, 10, min_score=-1.0, with_duplicates=True, clauses=clauses, method=method)
            mask = seg.filter_bitset(clauses, True) & seg.alive
            words = np.zeros((seg.records + 63) // 64 * 8, dtype=np.uint8)
            pb = np.packbits(mask, bitorder="little")
            words[: len(pb)] = pb
            p = _lib.VecSearchParams(10, 0, -1.0, 1, method, words.ctypes.data, int(mask.sum()))
            i2, s2, c2 = np.empty_like(ids), np.empty_like(sc), np.empty_like(cnt)
            _lib.check(_lib.load().nidx_vec_search(seg.segment._h, _lib.ptr(q), C.c_int32(len(q)), C.c_int32(64), _lib.NIDX_MEM_HOST, C.byref(p),
                                                   _lib.ptr(i2), _lib.ptr(s2), _lib.ptr(c2), None))
            assert (cnt == c2).all() and (ids == i2).all() and np.array_equal(sc, s2), (method, len(clauses))
