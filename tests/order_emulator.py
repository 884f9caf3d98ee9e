"""TEST INFRASTRUCTURE: tests/facet_emulator.py's stand-in for libnidx_b200.so plus the order entry points (nidx_txt_set_dates,
nidx_txt_search_ordered, nidx_txt_list_ordered), answered by tests/order_oracle.py, so the mirror's order flow (text.py,
binding.py) runs on a machine without a GPU.  Tests monkeypatch `_lib._lib` with it, as with EmulatedLib."""
import numpy as np

import facet_oracle as FO
import order_oracle as OO
from abi_emulator import NIL, _arr, _deref, _v
from facet_emulator import FacetEmulatedLib


class OrderEmulatedLib(FacetEmulatedLib):
    def nidx_txt_set_dates(self, h, created, modified):
        t = self._get(h)
        t.dates = (_arr(created, np.int64, t.n_docs).copy() if t.n_docs else np.zeros(0, np.int64),
                   _arr(modified, np.int64, t.n_docs).copy() if t.n_docs else np.zeros(0, np.int64))
        return 0

    def _order(self, t, order):
        o = _deref(order) if hasattr(order, "_obj") else order
        if not hasattr(t, "dates"):
            return (None, None), self._fail(-1, "the segment has no dates (nidx_txt_set_dates)")
        return (t.dates[o.field], o.type), 0

    def nidx_txt_search_ordered(self, h, query_terms, query_off, nq, mem, params, order, facets, out_docs, out_dates, out_counts, out_total, out_facets, stream):
        t, nq, p = self._get(h), _v(nq), _deref(params)
        (secs, typ), rc = self._order(t, order)
        if rc:
            return rc
        k = p.k
        if facets is not None:
            try:
                bucket, b_req, _ = self._plan(t, facets)
            except ValueError as e:
                return self._fail(-1, str(e))
        qo = _arr(query_off, np.uint32, nq + 1)
        qt = _arr(query_terms, np.uint32, int(qo[-1]))
        docs, dates = _arr(out_docs, np.uint32, nq * k).reshape(nq, k), _arr(out_dates, np.int64, nq * k).reshape(nq, k)
        cnt, total = _arr(out_counts, np.int32, nq), _arr(out_total, np.uint64, nq)
        docs[:], dates[:] = NIL, OO.NONE
        for i in range(nq):
            terms = [] if qo[i] == qo[i + 1] else list(qt[qo[i]:qo[i + 1]])
            mask = FO.matched(t.n_docs, t.term_off, t.post_doc, terms, p.mode == 1, t.alive)
            d, s = OO.order_topk(mask, secs, k, typ)
            docs[i, :len(d)], dates[i, :len(d)], cnt[i] = d, s, len(d)
            if total is not None:
                total[i] = int(mask.sum())
            if facets is not None and len(b_req):
                _arr(out_facets, np.uint32, nq * len(b_req))[i * len(b_req):(i + 1) * len(b_req)] = FO.count(t.facet_off, t.facet_ords, bucket, len(b_req), mask)
        return 0

    def nidx_txt_list_ordered(self, h, order, k, mem, out_docs, out_dates, out_count, out_total, stream):
        t, k = self._get(h), _v(k)
        (secs, typ), rc = self._order(t, order)
        if rc:
            return rc
        d, s, tot = OO.list_all(t.n_docs, t.alive, secs, k, typ)
        docs, dates = _arr(out_docs, np.uint32, k), _arr(out_dates, np.int64, k)
        docs[:], dates[:] = NIL, OO.NONE
        docs[:len(d)], dates[:len(d)] = d, s
        _arr(out_count, np.int32, 1)[0] = len(d)
        tot_out = _arr(out_total, np.uint64, 1)
        if tot_out is not None:
            tot_out[0] = tot
        return 0
