"""Multi-GPU search: one process per GPU, segments sharded across ranks, per-rank partial top-k
exchanged with ``all_gather`` (NCCL over NVLink on the GPU box, gloo in the CPU tests) and merged on the device
-- the GPU-native form of the reference's gRPC scatter-gather + k-way merge (nidx/src/searcher/grpc.rs:253-431,
shard_merge.rs:332-348 / 177-231).  Vectors merge by ``kmerge_parts_kernel`` (merge_vector_responses' kmerge_by(score >=)),
text by ``parts_merge_kernel`` ((score desc, part asc, position asc): the parts are segments of one index).  Parts are
taken in rank order, which stands for the order of the reference's ``responses`` vector; the reference itself groups
responses by node (grpc.rs:253-285), so it fixes no order across nodes: what the merge pins is kmerge_by's output for a
given order.

The exchange is [nq, k] (u32 id, f32 score) per rank = 8*nq*k bytes (80 KB at nq=1024, k=10): latency
bound, so it is one collective per batch, not per query.
"""
from __future__ import annotations


def gather_partials(ids, scores, group=None):
    """All ranks contribute their [nq, k] partial results; every rank receives [world, nq, k] in rank order."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    ids_all = [torch.empty_like(ids) for _ in range(world)]
    sc_all = [torch.empty_like(scores) for _ in range(world)]
    dist.all_gather(ids_all, ids.contiguous(), group=group)
    dist.all_gather(sc_all, scores.contiguous(), group=group)
    return torch.stack(ids_all), torch.stack(sc_all)


def global_ids(local_ids, part, vectors_per_rank: int):
    """(segment rank, local vector address) -> global address; NIL (-1 as int32) stays NIL."""
    import torch

    g = local_ids.to(torch.int64) + part.to(torch.int64) * int(vectors_per_rank)
    return torch.where(local_ids.to(torch.int64) < 0, torch.full_like(g, -1), g)


class ShardedSearcher:
    """One rank's view of a segment-sharded index.  Buffers are allocated once: the local result is written
    straight into this rank's slot of the exchange buffer ([2, nq, k]: ids, score bits), ONE all_gather moves
    every rank's slot, and kmerge_parts_kernel merges the gathered buffer in place (part_stride = 2*nq*k).

    ``search`` does the three steps back to back.  ``submit`` / ``collect`` pipeline them over `depth` buffer sets:
    the all_gather of batch i runs on the process group's own stream while batch i+1 is being searched on the
    caller's stream, and batch i is merged once its exchange has landed -- the exchange latency leaves the
    critical path.  ``local_search`` / ``merge`` are injectable so that the CPU (gloo) tests drive the same
    submit/collect logic without a GPU; the defaults are the C-ABI calls."""

    def __init__(self, segment, nq, k, device, group=None, depth=2, local_search=None, merge=None):
        import torch
        import torch.distributed as dist

        self.segment, self.nq, self.k, self.device, self.group, self.depth = segment, nq, k, device, group, depth
        self.world = dist.get_world_size(group)
        dev = torch.device("cpu") if device == "cpu" else torch.device("cuda", device)
        self._local_search = local_search or self._search_segment
        self._merge = merge or self._merge_device
        self.slots = []
        for _ in range(depth):
            self.slots.append(dict(
                local=torch.empty((2, nq, k), dtype=torch.int32, device=dev), counts=torch.empty((nq,), dtype=torch.int32, device=dev),
                gathered=torch.empty((self.world, 2, nq, k), dtype=torch.int32, device=dev),
                out=(torch.empty((nq, k), dtype=torch.int32, device=dev), torch.empty((nq, k), dtype=torch.float32, device=dev),
                     torch.empty((nq, k), dtype=torch.int32, device=dev)), work=None))
        self._next, self._pending = 0, []          # slot of the next submit; slots in flight, oldest first

    # -- the two device steps (C ABI) -----------------------------------------------------------------------
    def _search_segment(self, queries, ef, slot, **kw):
        import torch

        from . import _lib

        self.segment.search(queries, self.k, ef=ef, method=_lib.NIDX_METHOD_HNSW,
                            out=(slot["local"][0], slot["local"][1].view(torch.float32), slot["counts"]), **kw)

    def _merge_device(self, slot):
        import torch

        from .segment import merge_vector_parts

        g = slot["gathered"]
        return merge_vector_parts(g[:, 0], g[:, 1].view(torch.float32), device=self.device, part_stride=2 * self.nq * self.k, out=slot["out"])

    # -- pipeline -----------------------------------------------------------------------------------------------
    def submit(self, queries, ef, **kw):
        """Search the local segment for this batch and start the exchange; at most `depth` batches in flight."""
        import torch.distributed as dist

        if len(self._pending) == self.depth:
            raise RuntimeError(f"{self.depth} batches already in flight: collect() first")
        slot = self.slots[self._next]
        self._local_search(queries, ef, slot, **kw)
        flat = slot["gathered"].view(self.world * 2, self.nq, self.k)       # concatenation along dim 0 (the form gloo accepts too)
        slot["work"] = dist.all_gather_into_tensor(flat, slot["local"], group=self.group, async_op=True)
        self._pending.append(self._next)
        self._next = (self._next + 1) % self.depth

    def collect(self):
        """-> (local ids, scores, part) of the oldest batch in flight, identical on every rank.  The tensors belong to
        the batch's buffer set and are overwritten `depth` submits later."""
        if not self._pending:
            raise RuntimeError("nothing in flight")
        slot = self.slots[self._pending.pop(0)]
        slot["work"].wait()                  # the caller's stream waits for the exchange; the host does not (NCCL)
        slot["work"] = None
        return self._merge(slot)

    def search(self, queries, ef, **kw):
        """-> (local ids, scores, part) of the merged top-k, identical on every rank."""
        self.submit(queries, ef, **kw)
        return self.collect()


def shard_record(segment, queries, k, rank=0, dedup=False, ef=0, min_score=-1.0, with_duplicates=True, method=None, filter_bits=None, out=None):
    """nidx_vec_shard_record: search `segment` into one exchange record -> a torch int32 tensor of 2*nq*k words ([ids][score
    bits]; 6*nq*k with dedup: + [par_key u64][vec_key u64]) on the segment's GPU, asynchronous on the current stream.  numpy
    queries / filter bits are host memory, torch CUDA tensors device memory."""
    import ctypes as C

    import numpy as np

    from . import _lib
    from .segment import _is_torch, _stage

    _, stream, alloc = _stage(segment.cfg.device, True)     # the record is device memory, whatever memory the queries are in
    if _is_torch(queries):
        mem = _lib.NIDX_MEM_DEVICE
    else:
        mem = _lib.NIDX_MEM_HOST
        queries = np.ascontiguousarray(np.atleast_2d(queries), dtype=np.float32)
        filter_bits = None if filter_bits is None else np.ascontiguousarray(filter_bits, dtype=np.uint64)
    p = _lib.VecSearchParams(k, ef, min_score, int(with_duplicates), _lib.NIDX_METHOD_AUTO if method is None else method, _lib.ptr(filter_bits), 0)
    nq, ldq = queries.shape
    out = out if out is not None else alloc(nq * k * (6 if dedup else 2), np.uint32)
    _lib.check(_lib.load().nidx_vec_shard_record(segment._h, _lib.ptr(queries), nq, ldq, mem, C.byref(p), rank, int(dedup), _lib.ptr(out), stream))
    return out


def shard_merge(records, n_parts, nq, k, dedup=False, with_duplicates=True, device=0, host=False):
    """nidx_shard_merge over n_parts records laid end to end in one torch CUDA tensor -> (ids local to their part, scores, part,
    counts): torch tensors on the device (asynchronous on the current stream), or numpy arrays with host=True."""
    import numpy as np

    from . import _lib
    from .segment import _stage, _torch_stream

    mem, _, alloc = _stage(device, not host)
    out = (alloc((nq, k), np.uint32), alloc((nq, k), np.float32), alloc((nq, k), np.int32), alloc(nq, np.int32))
    # the records are device memory: the merge runs on the current torch stream whatever memory the outputs are in
    _lib.check(_lib.load().nidx_shard_merge(device, _lib.ptr(records), n_parts, nq, k, int(dedup), int(with_duplicates), mem, *map(_lib.ptr, out),
                                            _torch_stream(device)))
    return out


def docaddr(local_docs, part):
    """nidx_paragraph reader.rs:310 / nidx_text reader.rs: docaddr = (segment_ord << 32) + doc; NIL stays -1."""
    import torch

    a = (part.to(torch.int64) << 32) + (local_docs.to(torch.int64) & 0xFFFFFFFF)
    return torch.where(part.to(torch.int64) < 0, torch.full_like(a, -1), a)


class ShardedTextSearcher(ShardedSearcher):
    """BM25 over a doc-partitioned index: every rank holds the postings of its own documents (one tantivy segment per rank in
    the reference's terms) scored with the statistics of the WHOLE index (`TextSegment.set_stats`; tantivy computes N, df and
    the average length over the union of segments, nidx_tantivy/src/index_reader.rs:39-77).  Per batch: local top-k + local
    `Count` -> one all_gather of the [2, nq, k] (doc, score bits) partials + one all_reduce of the [nq] counts -> the text
    merge (nidx_merge_topk), which ranks (score desc, part asc, position asc).  The parts are segments of one index, so part
    ascending is docaddr ascending (docaddr = segment << 32 | doc) and this is merge_document_responses' order within one
    shard (bm25 desc, lower docaddr first; shard_merge.rs:211-231) because every part arrives sorted (score desc, doc asc)."""

    def _merge_device(self, slot):
        import torch

        from .segment import merge_topk

        g = slot["gathered"]
        return merge_topk(g[:, 0], g[:, 1].view(torch.float32), device=self.device, part_stride=2 * self.nq * self.k, out=slot["out"])

    def __init__(self, segment, nq, k, device, group=None, depth=2, local_search=None, merge=None):
        import torch

        super().__init__(segment, nq, k, device, group, depth, local_search, merge)
        for slot in self.slots:
            slot["total"] = torch.zeros((nq,), dtype=torch.int64, device=slot["local"].device)
            slot["work_total"] = None

    def _search_segment(self, queries, ef, slot, **kw):
        import torch

        terms, offsets = queries
        self.segment.search(terms, offsets, self.k, out=(slot["local"][0], slot["local"][1].view(torch.float32), slot["counts"], slot["total"]), **kw)

    def submit(self, queries, ef=None, **kw):
        """queries = (query_terms, query_off) as for TextSegment.search; kw: mode, use_tf, min_score, after."""
        import torch.distributed as dist

        super().submit(queries, ef, **kw)
        slot = self.slots[self._pending[-1]]
        slot["work_total"] = dist.all_reduce(slot["total"], op=dist.ReduceOp.SUM, group=self.group, async_op=True)

    def collect(self):
        """-> (local docs, scores, part, total matching documents over all parts) of the oldest batch in flight."""
        slot = self.slots[self._pending[0]]
        merged = super().collect()
        slot["work_total"].wait()
        slot["work_total"] = None
        return (*merged, slot["total"])


class ShardComm:
    """nidx_shard_comm: the library's own NCCL communicator (include/nidx_b200.h "Segments sharded over the GPUs of one node").
    The 128-byte NCCL id is created by rank 0 inside the library and handed to the other ranks through `exchange`, any
    callable that returns rank 0's bytes on every rank -- by default a broadcast over the already initialised
    torch.distributed group (any backend: the id is host data)."""

    def __init__(self, rank: int, world: int, device: int, exchange=None):
        import ctypes as C

        from . import _lib

        L = _lib.require_device()
        buf = (C.c_uint8 * 128)()
        if rank == 0:
            _lib.check(L.nidx_shard_unique_id(buf))
        payload = bytes(buf)
        if exchange is None:
            import torch.distributed as dist

            box = [payload]
            dist.broadcast_object_list(box, src=0)
            payload = box[0]
        else:
            payload = exchange(payload)
        ident = (C.c_uint8 * 128).from_buffer_copy(payload)
        self._h = C.c_void_p()
        _lib.check(L.nidx_shard_init(ident, rank, world, device, C.byref(self._h)))
        self.rank, self.world, self.device = rank, world, device

    def close(self):
        from . import _lib

        if self._h is not None:
            _lib.load().nidx_shard_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def search_vectors(self, segment, queries, k, ef=0, min_score=-1.0, with_duplicates=True, method=None, dedup=False, out=None, stream=None):
        """nidx_vec_search_sharded: -> (ids local to their part, scores, part, counts), identical on every rank.  torch CUDA
        queries: device path, asynchronous on the current stream; numpy queries: host path (copies inside the call)."""
        import ctypes as C

        import numpy as np

        from . import _lib
        from .segment import _is_torch, _stage

        p = _lib.VecSearchParams(k, ef, min_score, int(with_duplicates), _lib.NIDX_METHOD_HNSW if method is None else method, None, 0)
        mem, stream, alloc = _stage(self.device, _is_torch(queries), stream)
        if mem == _lib.NIDX_MEM_HOST:
            queries = np.ascontiguousarray(np.atleast_2d(queries), dtype=np.float32)
        nq, ldq = queries.shape
        out = out or (alloc((nq, k), np.uint32), alloc((nq, k), np.float32), alloc((nq, k), np.int32), alloc(nq, np.int32))
        _lib.check(_lib.load().nidx_vec_search_sharded(self._h, segment._h, _lib.ptr(queries), nq, ldq, mem, C.byref(p), int(dedup), *map(_lib.ptr, out),
                                                       stream))
        return out

    def search_text(self, segment, query_terms, query_off, k, mode=0, use_tf=True, min_score=0.0, out=None):
        """nidx_txt_search_sharded: -> (docs local to their part, scores, part, counts, total over all parts)."""
        import ctypes as C

        import numpy as np

        from . import _lib

        p = _lib.TxtSearchParams(k, mode, int(use_tf), min_score, 0, 0.0, 0, 0)
        mem, stream, alloc, query_terms, query_off, nq = segment._queries(query_terms, query_off)
        out = out or (alloc((nq, k), np.uint32), alloc((nq, k), np.float32), alloc((nq, k), np.int32), alloc(nq, np.int32), alloc(nq, np.uint64))
        _lib.check(_lib.load().nidx_txt_search_sharded(self._h, segment._h, _lib.ptr(query_terms), _lib.ptr(query_off), nq, mem, C.byref(p), *map(_lib.ptr, out),
                                                       stream))
        return out
