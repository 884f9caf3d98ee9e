"""TEST INFRASTRUCTURE: a stand-in for libnidx_b200.so backed by the oracle, so that the Python mirror of the reference
interface (nucliadb_b200/vector.py, text.py: filters, Fssc, MaxSim re-scoring, deletions by sequence, merges, directory round
trip) can be exercised on a machine without a GPU.  It takes the same ctypes arguments as the C ABI (include/nidx_b200.h) and
restates api.cu's HOST-side decisions (alive AND filter, the AUTO method choice, ef defaults, the insertion schedule); every number
it returns comes from oracle/.  It is not a fallback: nothing in the product can reach it (tests monkeypatch `_lib._lib`)."""
import ctypes as C
import os

import numpy as np

import oracle as O
from oracle import disk_v2
from nucliadb_b200 import _lib

NIL = 0xFFFFFFFF


def _v(x):
    return x.value if hasattr(x, "value") else x


def _addr(p):
    if p is None:
        return 0
    return _v(p) or 0


def _arr(p, dtype, count):
    a = _addr(p)
    if not a or count == 0:
        return None if not a else np.zeros(0, dtype)
    nbytes = int(count) * np.dtype(dtype).itemsize
    return np.frombuffer((C.c_char * nbytes).from_address(a), dtype=dtype)


def _deref(byref_arg):
    return byref_arg._obj


class _Vec:
    def __init__(self, cfg, vecs, par_of):
        self.d, self.sim = cfg.dimension, {_lib.NIDX_SIM_COSINE: O.SIM_COSINE, _lib.NIDX_SIM_DOT: O.SIM_DOT, _lib.NIDX_SIM_L2: O.SIM_L2}[cfg.similarity]
        self.multi, self.m, self.m0, self.efc, self.ef = bool(cfg.multi_vector), cfg.m, cfg.m0, cfg.ef_construction, cfg.ef_search
        self.v = np.ascontiguousarray(vecs, dtype=np.float32).reshape(-1, self.d)
        self.n = len(self.v)
        self.par_of = None if par_of is None else np.array(par_of, dtype=np.uint32)
        if self.par_of is not None and len(self.par_of):
            self.n_par = int(self.par_of.max()) + 1
            first = np.searchsorted(self.par_of, np.arange(self.n_par + 1)).astype(np.uint32)
            self.first, self.num = first[:-1].copy(), np.diff(first).astype(np.uint32)
            if self.n_par == self.n:
                self.par_of = None
        else:
            self.n_par = self.n
        if self.par_of is None:
            self.first = self.num = None
        self.alive, self.g = None, None


class _Txt:
    pass


class EmulatedLib:
    def __init__(self):
        self.err = b""
        self.handles = {}
        self.next = 1

    # ---- plumbing --------------------------------------------------------------------------------------------------------
    def _fail(self, code, msg):
        self.err = msg.encode()
        return code

    def _new(self, obj, out):
        h = self.next
        self.next += 1
        self.handles[h] = obj
        _deref(out).value = h
        return 0

    def _get(self, h):
        return self.handles[_v(h)]

    def nidx_last_error(self):
        return self.err

    def nidx_device_count(self):
        return 1

    def nidx_launch_count(self):
        return 0

    def nidx_use_hnsw(self, total, matching, k, rq, m):
        return int(O.use_hnsw(_v(total), _v(matching), _v(k), has_rabitq=bool(_v(rq)), M=_v(m)))

    def nidx_rank_fusion_rrf(self, device, sources, n_sources, nq, k, mem, out_keys, out_scores, out_refs, out_counts, stream):
        """ReciprocalRankFusion.fuse through the oracle's restatement (host buffers), in the C ABI's output layout."""
        from oracle.rank_fusion import rrf_fuse

        n_sources, nq, kk = _v(n_sources), _v(nq), float(_v(k))
        srcs = [sources[i] for i in range(n_sources)]
        cap = sum(s.k for s in srcs)
        ok, osc = _arr(out_keys, np.uint64, nq * cap).reshape(nq, cap), _arr(out_scores, np.float64, nq * cap).reshape(nq, cap)
        orf, ocn = _arr(out_refs, np.uint32, nq * cap).reshape(nq, cap), _arr(out_counts, np.int32, nq)
        for q in range(nq):
            lists = []
            for s in srcs:
                keys = _arr(C.c_void_p(s.keys), np.uint64, nq * s.k).reshape(nq, s.k)[q]
                scores = _arr(C.c_void_p(s.scores), np.float32, nq * s.k).reshape(nq, s.k)[q]
                n = int(_arr(C.c_void_p(s.counts), np.int32, nq)[q]) if s.counts else int(np.sum(keys != np.uint64(0xFFFFFFFFFFFFFFFF)))
                lists.append([(int(keys[j]), float(scores[j])) for j in range(n)])
            fused = rrf_fuse(lists, [s.weight for s in srcs], k=kk)
            ok[q], osc[q], orf[q], ocn[q] = np.uint64(0xFFFFFFFFFFFFFFFF), 0.0, NIL, len(fused)
            for j, (key, sc, first, pos, mask) in enumerate(fused):
                ok[q, j], osc[q, j], orf[q, j] = key, sc, (first << 28) | (mask << 24) | pos
        return 0

    def nidx_normalize_vectors(self, device, vectors, n, d, ld, mem, stream):
        n, d, ld = _v(n), _v(d), _v(ld)
        a = np.ctypeslib.as_array(C.cast(vectors, C.POINTER(C.c_float)), shape=(n, ld))
        for i in range(n):
            a[i, :d] = O.normalize(a[i, :d].copy())
        return 0

    # ---- vector segments -----------------------------------------------------------------------------------------------
    def nidx_vec_create(self, cfg, vectors, n, ld, mem, paragraph_of, out):
        cfg, n, ld = _deref(cfg), _v(n), _v(ld)
        if ld < cfg.dimension:
            return self._fail(-1, "ld < dimension (VectorErr::InconsistentDimensions)")
        v = _arr(vectors, np.float32, n * ld)
        v = np.zeros((0, cfg.dimension), np.float32) if v is None or n == 0 else v.reshape(n, ld)[:, : cfg.dimension].copy()
        par = _arr(paragraph_of, np.uint32, n)
        return self._new(_Vec(cfg, v, None if par is None else par.copy()), out)

    def nidx_vec_close(self, h):
        self.handles.pop(_v(h), None)

    def nidx_vec_len(self, h):
        return self._get(h).n

    def nidx_vec_set_alive(self, h, bits, mem):
        s = self._get(h)
        w = _arr(bits, np.uint64, (s.n_par + 63) // 64)
        s.alive = None if w is None else w.copy()
        return 0

    def nidx_vec_build_hnsw(self, h, seed, max_batch, stream):
        s = self._get(h)
        mb = _v(max_batch) if _v(max_batch) > 0 else 4096
        s.g = O.hnsw_build(s.v, sim=s.sim, M=s.m, M0=s.m0, efC=s.efc, seed=_v(seed), max_batch=mb, nthreads=4) if s.n else O.Graph(0, s.m, s.m0, np.zeros(0, np.uint8))
        return 0

    def nidx_vec_graph_dims(self, h, s0, su, rows, en, el):
        s = self._get(h)
        if s.g is None:
            return self._fail(-3, "segment has no HNSW graph")
        _deref(s0).value, _deref(su).value = s.g.adj0.shape[1], s.g.adjU.shape[1]
        _deref(rows).value = int(s.g.level.astype(np.int64).sum())
        _deref(en).value, _deref(el).value = s.g.entry_node, s.g.entry_layer
        return 0

    def nidx_vec_get_graph(self, h, level, adj0, w0, adjU, wU):
        s = self._get(h)
        if s.g is None:
            return self._fail(-3, "segment has no HNSW graph")
        g, rows = s.g, int(s.g.level.astype(np.int64).sum())
        for dst, src, dt in ((level, g.level, np.uint8), (adj0, g.adj0, np.uint32), (w0, g.w0, np.float32), (adjU, g.adjU[:rows], np.uint32), (wU, g.wU[:rows], np.float32)):
            out = _arr(dst, dt, src.size)
            if out is not None and src.size:
                out[:] = src.reshape(-1)
        return 0

    def nidx_vec_set_graph(self, h, level, adj0, w0, adjU, wU):
        s = self._get(h)
        lv = _arr(level, np.uint8, s.n).copy()
        g = O.Graph(s.n, s.m, s.m0, lv)
        rows = int(lv.astype(np.int64).sum())
        g.adj0[:] = _arr(adj0, np.uint32, g.adj0.size).reshape(g.adj0.shape)
        if _addr(w0):
            g.w0[:] = _arr(w0, np.float32, g.w0.size).reshape(g.w0.shape)
        if rows and _addr(adjU):
            g.adjU[:rows] = _arr(adjU, np.uint32, rows * g.adjU.shape[1]).reshape(rows, -1)
        if rows and _addr(wU):
            g.wU[:rows] = _arr(wU, np.float32, rows * g.wU.shape[1]).reshape(rows, -1)
        s.g = g
        return 0

    def nidx_vec_extend_hnsw(self, h, n_existing, level, adj0, w0, adjU, wU, entry_node, entry_layer, seed, max_batch, stream):
        s, n0 = self._get(h), _v(n_existing)
        lv = _arr(level, np.uint8, n0).copy()
        g0 = O.Graph(n0, s.m, s.m0, lv)
        rows = int(lv.astype(np.int64).sum())
        g0.adj0[:] = _arr(adj0, np.uint32, g0.adj0.size).reshape(g0.adj0.shape)
        g0.w0[:] = _arr(w0, np.float32, g0.w0.size).reshape(g0.w0.shape)
        if rows:
            g0.adjU[:rows] = _arr(adjU, np.uint32, rows * g0.adjU.shape[1]).reshape(rows, -1)
            g0.wU[:rows] = _arr(wU, np.float32, rows * g0.wU.shape[1]).reshape(rows, -1)
        g0.entry_node, g0.entry_layer = _v(entry_node), _v(entry_layer)
        mb = _v(max_batch) if _v(max_batch) > 0 else 4096
        s.g = O.hnsw_extend(s.v, g0, sim=s.sim, efC=s.efc, seed=_v(seed), max_batch=mb, nthreads=4)
        return 0

    # ---- filters on the "device" (api.cu filter_formula restated with numpy) --------------------------------------------
    def nidx_vec_set_inverted_index(self, h, which, n_keys, key_bytes, key_off, post_off, postings):
        s, which, n = self._get(h), _v(which), _v(n_keys)
        ko = _arr(key_off, np.uint64, n + 1) if n else np.zeros(1, np.uint64)
        po = _arr(post_off, np.uint64, n + 1) if n else np.zeros(1, np.uint64)
        kb = bytes(_arr(key_bytes, np.uint8, int(ko[n]))) if n and int(ko[n]) else b""
        ps = _arr(postings, np.uint32, int(po[n])).copy() if n and int(po[n]) else np.zeros(0, np.uint32)
        keys = [kb[int(ko[i]):int(ko[i + 1])] for i in range(n)]
        if any(keys[i] >= keys[i + 1] for i in range(n - 1)):
            return self._fail(-1, "inverted index keys must be strictly ascending")
        if not hasattr(s, "inv"):
            s.inv = {}
        s.inv[which] = (keys, [ps[int(po[i]):int(po[i + 1])] for i in range(n)])
        return 0

    def _formula_bits(self, s, nodes, n_nodes):
        """-> bool mask over paragraphs (before the alive intersection), or an error string."""
        nodes = C.cast(nodes, C.POINTER(_lib.FilterNode)) if not isinstance(nodes, C.Array) else nodes
        pos = [0]

        def ev():
            i = pos[0]
            if i >= n_nodes:
                raise ValueError("malformed filter formula")
            nd = nodes[i]
            pos[0] += 1
            out = np.zeros(s.n_par, dtype=bool)
            if nd.kind in (_lib.NIDX_F_LABEL, _lib.NIDX_F_KEYS):
                keys, posts = getattr(s, "inv", {}).get(_lib.NIDX_INV_LABELS if nd.kind == _lib.NIDX_F_LABEL else _lib.NIDX_INV_FIELDS, ([], []))
                for j in range(nd.n):
                    qk = C.string_at(nd.keys[j], nd.key_len[j]) if nd.key_len[j] else b""
                    for kk, pp in zip(keys, posts):
                        if (kk.startswith(qk) if nd.kind == _lib.NIDX_F_LABEL else kk == qk):
                            out[pp] = True
                return out
            if nd.n < 1:
                raise ValueError("a compound clause needs operands")
            acc = ev()
            for _ in range(nd.n - 1):
                b = ev()
                acc = (acc | b) if nd.kind == _lib.NIDX_F_OR else (acc & b)
            return ~acc if nd.kind == _lib.NIDX_F_NOT else acc

        mask = ev()
        if pos[0] != n_nodes:
            raise ValueError("malformed filter formula")
        return mask

    @staticmethod
    def _pack(mask):
        words = np.zeros((len(mask) + 63) // 64 * 8, dtype=np.uint8)
        pb = np.packbits(mask, bitorder="little")
        words[: len(pb)] = pb
        return words.view(np.uint64)

    def nidx_vec_filter(self, h, nodes, n_nodes, out_bits, mem, out_matching, stream):
        s = self._get(h)
        try:
            bits = self._pack(self._formula_bits(s, nodes, _v(n_nodes)))
        except ValueError as e:
            return self._fail(-1, str(e))
        if s.alive is not None:
            bits = bits & s.alive
        ob = _arr(out_bits, np.uint64, len(bits))
        if ob is not None:
            ob[:] = bits
        if out_matching is not None:
            _deref(out_matching).value = int(sum(bin(int(w)).count("1") for w in bits))
        return 0

    def nidx_vec_search_formula(self, h, queries, nq, ldq, mem, params, nodes, n_nodes, out_ids, out_scores, out_counts, stream):
        s = self._get(h)
        if _deref(params).filter_bits:
            return self._fail(-1, "give either filter_bits or a formula")
        try:
            bits = self._pack(self._formula_bits(s, nodes, _v(n_nodes)))
        except ValueError as e:
            return self._fail(-1, str(e))
        return self.nidx_vec_search(h, queries, nq, ldq, mem, params, out_ids, out_scores, out_counts, stream, formula_bits=bits)

    def nidx_vec_search(self, h, queries, nq, ldq, mem, params, out_ids, out_scores, out_counts, stream, formula_bits=None):
        s, nq, ldq, p = self._get(h), _v(nq), _v(ldq), _deref(params)
        if ldq < s.d:
            return self._fail(-1, f"query dimension {ldq} != index dimension {s.d} (VectorErr::InconsistentDimensions)")
        k = p.k
        q = _arr(queries, np.float32, nq * ldq).reshape(nq, ldq)[:, : s.d].copy()
        ids, sc, cnt = _arr(out_ids, np.uint32, nq * k).reshape(nq, k), _arr(out_scores, np.float32, nq * k).reshape(nq, k), _arr(out_counts, np.int32, nq)
        words = (s.n_par + 63) // 64
        bits = s.alive                                                      # api.cu: filter AND alive, matching as the caller states it
        matching = s.n_par if s.alive is None else int(sum(bin(int(w)).count("1") for w in s.alive))
        filtered = bool(p.filter_bits) or formula_bits is not None
        if filtered:
            f = formula_bits if formula_bits is not None else _arr(p.filter_bits, np.uint64, words)
            bits = f.copy() if s.alive is None else (f & s.alive)
            matching = (p.filter_matching if formula_bits is None else 0) or int(sum(bin(int(w)).count("1") for w in bits))
        if matching == 0:                                                   # segment.rs:532-534
            ids[:], sc[:], cnt[:] = NIL, 0, 0
            return 0
        method = p.method
        if method == _lib.NIDX_METHOD_AUTO:                                 # api.cu: choose_method
            if s.g is None:
                method = _lib.NIDX_METHOD_BRUTE
            else:
                method = _lib.NIDX_METHOD_HNSW if O.use_hnsw(s.n_par, matching, k, M=s.m) else _lib.NIDX_METHOD_BRUTE
        if s.n == 0:
            ids[:], sc[:], cnt[:] = NIL, 0, 0
            return 0
        if method == _lib.NIDX_METHOD_BRUTE:
            i, x, c = O.brute_force(s.v, q, k, sim=s.sim, min_score=p.min_score, alive_bits=bits, first_vec=s.first, num_vec=s.num, nthreads=2)
        elif method == _lib.NIDX_METHOD_HNSW:
            if s.g is None:
                return self._fail(-3, "HNSW search requested but the segment has no graph")
            i, x, c, _ = O.hnsw_search(s.v, s.g, q, k, p.ef or s.ef, sim=s.sim, min_score=p.min_score, with_duplicates=bool(p.with_duplicates),
                                       multi_vector=s.multi, filter_bits=bits, paragraph_of=s.par_of, nthreads=2)
        else:
            return self._fail(-1, "method not emulated")
        ids[:], sc[:], cnt[:] = i, x, c
        return 0

    def nidx_vec_save(self, h, directory):
        s, d = self._get(h), _v(directory).decode()
        par = s.par_of if s.par_of is not None else np.arange(s.n, dtype=np.uint32)
        open(os.path.join(d, "vectors.bin"), "wb").write(disk_v2.write_vectors_bin(s.v, par))
        if s.g is not None:
            layers = [{int(n): [(int(t), float(w)) for t, w in zip(s.g.edges(n, l), (s.g.w0[n] if l == 0 else s.g.wU[int(s.g.upper_off[n]) + l - 1]))]
                       for n in range(s.n) if s.g.level[n] >= l} for l in range(s.g.entry_layer + 1)] if s.n else []
            graph, edges = disk_v2.serialize_graph(layers, s.n, s.g.entry_node, s.g.entry_layer)
            open(os.path.join(d, "hnsw.graph"), "wb").write(graph)
            open(os.path.join(d, "hnsw.edges"), "wb").write(edges)
        return 0

    def nidx_vec_open(self, cfg, directory, out):
        cfg, d = _deref(cfg), _v(directory).decode()
        rec = np.dtype([("vector", np.float32, (cfg.dimension,)), ("paragraph", np.uint32)])
        stored = np.fromfile(os.path.join(d, "vectors.bin"), dtype=rec)
        s = _Vec(cfg, np.ascontiguousarray(stored["vector"]), stored["paragraph"].copy() if len(stored) else None)
        gp = os.path.join(d, "hnsw.graph")
        if os.path.exists(gp) and os.path.getsize(gp):
            graph, edges = open(gp, "rb").read(), np.frombuffer(open(os.path.join(d, "hnsw.edges"), "rb").read(), dtype=np.float32)
            entry_node, entry_layer = disk_v2.entrypoint(graph)
            level = np.zeros(s.n, np.uint8)
            rows = {}
            for n in range(s.n):                                            # a node is in layer l iff it links or is linked there (v2.rs:248-312)
                for l in range(entry_layer + 1):
                    e = disk_v2.get_out_edges(graph, n, l)
                    rows[(n, l)] = e
                    if e:
                        level[n] = max(level[n], l)
                        for t in e:
                            level[t] = max(level[t], l)
            level[entry_node] = max(level[entry_node], entry_layer)
            g, pos = O.Graph(s.n, s.m, s.m0, level), 0
            for n in range(s.n):                                            # hnsw.edges: one f32 per edge in file order (node, then layer)
                for l in range(entry_layer + 1):
                    e = rows[(n, l)]
                    if l <= level[n]:
                        r, w = (g.adj0[n], g.w0[n]) if l == 0 else (g.adjU[int(g.upper_off[n]) + l - 1], g.wU[int(g.upper_off[n]) + l - 1])
                        r[: len(e)], w[: len(e)] = e, edges[pos : pos + len(e)]
                    pos += len(e)
            g.entry_node, g.entry_layer = entry_node, entry_layer
            s.g = g
        return self._new(s, out)

    # ---- text segments ----------------------------------------------------------------------------------------------------
    def nidx_txt_create(self, device, n_docs, n_terms, term_off, post_doc, post_tf, fieldnorm_id, out):
        t = _Txt()
        t.n_docs, t.n_terms = _v(n_docs), _v(n_terms)
        t.term_off = _arr(term_off, np.uint64, t.n_terms + 1).copy()
        npost = int(t.term_off[-1])
        t.post_doc, t.post_tf = _arr(post_doc, np.uint32, npost).copy(), _arr(post_tf, np.uint32, npost).copy()
        t.fieldnorm_id = _arr(fieldnorm_id, np.uint8, t.n_docs).copy()
        t.doc_freq = np.diff(t.term_off.astype(np.int64)).astype(np.uint64)
        t.total_docs, t.total_tokens, t.alive = t.n_docs, 0, None
        return self._new(t, out)

    def nidx_txt_set_stats(self, h, total_docs, total_tokens, df):
        t = self._get(h)
        t.total_docs, t.total_tokens = _v(total_docs), _v(total_tokens)
        d = _arr(df, np.uint64, t.n_terms)
        if d is not None:
            t.doc_freq = d.copy()
        return 0

    def nidx_txt_set_alive(self, h, bits):
        t = self._get(h)
        w = _arr(bits, np.uint64, (t.n_docs + 63) // 64)
        t.alive = None if w is None else w.copy()
        return 0

    def nidx_txt_close(self, h):
        self.handles.pop(_v(h), None)

    def nidx_txt_search(self, h, query_terms, query_off, nq, mem, params, out_docs, out_scores, out_counts, out_total, stream):
        t, nq, p = self._get(h), _v(nq), _deref(params)
        k = p.k
        qo = _arr(query_off, np.uint32, nq + 1)
        qt = _arr(query_terms, np.uint32, int(qo[-1]))
        queries = [[] if qo[i] == qo[i + 1] else list(qt[qo[i] : qo[i + 1]]) for i in range(nq)]
        want = k if not p.after_mode else t.n_docs                          # search-after: rank everything, then cut (reader.rs:350-392)
        d, s, c, tot = O.bm25_search(t, queries, max(want, 1), mode=p.mode, use_tf=bool(p.use_tf), alive_bits=t.alive, total_docs=t.total_docs,
                                     total_tokens=t.total_tokens, doc_freq=t.doc_freq)
        docs, sc, cnt = _arr(out_docs, np.uint32, nq * k).reshape(nq, k), _arr(out_scores, np.float32, nq * k).reshape(nq, k), _arr(out_counts, np.int32, nq)
        total = _arr(out_total, np.uint64, nq)
        docs[:], sc[:] = NIL, 0
        for i in range(nq):
            keep = []
            for j in range(int(c[i])):
                score, doc = np.float32(s[i, j]), int(d[i, j])
                if p.after_mode:                                            # is_after(): strictly lower score, or an equal one the tie break keeps
                    a = np.float32(p.after_score)
                    if not (score < a or (score == a and (p.after_mode == 3 or (p.after_mode == 2 and p.docaddr_base + doc > p.after_docaddr)))):
                        continue
                if score < p.min_score:                                     # the min_score cut comes after the top-k (reader.rs:302-305)
                    continue
                keep.append((doc, score))
            keep = keep[:k]
            cnt[i] = len(keep)
            for j, (doc, score) in enumerate(keep):
                docs[i, j], sc[i, j] = doc, score
            if total is not None:
                total[i] = tot[i]
        return 0
