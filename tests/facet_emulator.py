"""TEST INFRASTRUCTURE: tests/abi_emulator.py's stand-in for libnidx_b200.so plus the facet entry points (nidx_txt_set_facets,
nidx_txt_facet_buckets, nidx_txt_search_faceted, nidx_txt_facet_count_all), answered by tests/facet_oracle.py, so the mirror's
facet flow (text.py, binding.py) runs on a machine without a GPU.  Tests monkeypatch `_lib._lib` with it, as with EmulatedLib."""
import ctypes as C

import numpy as np

import facet_oracle as FO
from abi_emulator import EmulatedLib, _arr, _deref, _v


def _request(req):
    r = _deref(req) if hasattr(req, "_obj") else req
    n = r.n
    if n == 0:
        return []
    off = _arr(C.c_void_p(r.key_off), np.uint64, n + 1)
    kb = bytes(_arr(C.c_void_p(r.key_bytes), np.uint8, int(off[n]))) if int(off[n]) else b""
    return [kb[int(off[i]):int(off[i + 1])] for i in range(n)]


class FacetEmulatedLib(EmulatedLib):
    def nidx_txt_set_facets(self, h, n_facets, key_bytes, key_off, doc_off, doc_ords):
        t, n = self._get(h), _v(n_facets)
        ko = _arr(key_off, np.uint64, n + 1) if n else np.zeros(1, np.uint64)
        kb = bytes(_arr(key_bytes, np.uint8, int(ko[n]))) if n and int(ko[n]) else b""
        keys = [kb[int(ko[i]):int(ko[i + 1])] for i in range(n)]
        if any(keys[i] >= keys[i + 1] for i in range(n - 1)):
            return self._fail(-1, "facet keys must be strictly ascending (facet order)")
        t.facet_keys = keys
        t.facet_off = _arr(doc_off, np.uint64, t.n_docs + 1).copy()
        t.facet_ords = _arr(doc_ords, np.uint32, int(t.facet_off[-1])).copy() if int(t.facet_off[-1]) else np.zeros(0, np.uint32)
        return 0

    def _plan(self, t, req):
        if not hasattr(t, "facet_keys"):
            raise RuntimeError("the segment has no facets")
        return FO.plan(t.facet_keys, _request(req))

    def nidx_txt_facet_buckets(self, h, req, out_req, out_ord, cap, out_n):
        try:
            _, b_req, b_ord = self._plan(self._get(h), req)
        except ValueError as e:
            return self._fail(-1, str(e))
        n = min(len(b_req), _v(cap))
        if n:
            _arr(out_req, np.uint32, n)[:] = b_req[:n]
            _arr(out_ord, np.uint32, n)[:] = b_ord[:n]
        _deref(out_n).value = len(b_req)
        return 0

    def _counts(self, t, req, mask):
        bucket, b_req, _ = self._plan(t, req)
        return FO.count(t.facet_off, t.facet_ords, bucket, len(b_req), mask)

    def nidx_txt_search_faceted(self, h, query_terms, query_off, nq, mem, params, req, out_docs, out_scores, out_counts, out_total, out_facets, stream):
        t, nq, p = self._get(h), _v(nq), _deref(params)
        try:
            bucket, b_req, _ = self._plan(t, req)
        except ValueError as e:
            return self._fail(-1, str(e))
        rc = self.nidx_txt_search(h, query_terms, query_off, nq, mem, params, out_docs, out_scores, out_counts, out_total, stream)
        if rc:
            return rc
        qo = _arr(query_off, np.uint32, nq + 1)
        qt = _arr(query_terms, np.uint32, int(qo[-1]))
        out = _arr(out_facets, np.uint32, nq * len(b_req))
        for i in range(nq):
            terms = [] if qo[i] == qo[i + 1] else list(qt[qo[i]:qo[i + 1]])
            mask = FO.matched(t.n_docs, t.term_off, t.post_doc, terms, p.mode == 1, t.alive)
            if len(b_req):
                out[i * len(b_req):(i + 1) * len(b_req)] = FO.count(t.facet_off, t.facet_ords, bucket, len(b_req), mask)
        return 0

    def nidx_txt_facet_count_all(self, h, req, mem, out_facets, stream):
        t = self._get(h)
        try:
            c = self._counts(t, req, FO.alive_mask(t.n_docs, t.alive))
        except ValueError as e:
            return self._fail(-1, str(e))
        if len(c):
            _arr(out_facets, np.uint32, len(c))[:] = c
        return 0
