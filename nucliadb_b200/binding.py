"""The outer boundary of the hot path: the ``nidx_binding.NidxBinding`` Python surface and the ``NidxSearcher.Search`` gRPC
service, over the GPU searchers of this package.

Reference:
  nidx/nidx_binding/nidx_binding.pyi:15-71, src/lib.rs:53-127    NidxBinding(settings), index(bytes) -> seq, wait_for_sync(),
                                                                   searcher_port, api_port
  nidx/nidx_protos/nidx.proto:9,20-21                             NidxApi.NewShard, NidxSearcher.Search
  nidx/src/searcher/shard_search.rs:60-241                        one SearchRequest -> prefilter -> vector / paragraph / document searches
  nidx/src/searcher/shard_merge.rs:177-348, 380-414               merge of the per-shard responses (merge_facets: facet counts)
  nidx/src/searcher/shard_merge.rs:235-249, 313-328, 416-436      ... under SearchRequest.order: by date (merge_order_key)
  nidx/nidx_vector/src/indexer.rs:96-146                          Resource -> vector Elems (key = sentence id, labels = paragraph labels)
  nidx/nidx_text/src/resource_indexer.rs:22-91                    Resource.texts -> one document per field
  nidx/nidx_paragraph/src/resource_indexer.rs:33-131              Resource.paragraphs -> one document per paragraph (text[start:end])
  nidx/nidx_text/src/resource_indexer.rs:49-62                    Resource.security -> the access groups of its documents
  nidx/nidx_json/src/resource_indexer.rs, lib.rs                  Resource.json_fields -> one JSON document per resource
  nidx/src/searcher/query_planner/prefilter.rs:24-72              SearchRequest.json_filter, combined with the text prefilter
  nidx/nidx_relation/src/resource_indexer.rs, reader.rs           Resource.field_relations -> one relation document each; GraphSearch
  nidx/src/searcher/shard_search.rs:290-362, shard_merge.rs:350-375   NidxSearcher.GraphSearch: prefilter, search, concatenation
  nidx/src/searcher/shard_suggest.rs:94-161, shard_merge.rs:101-151    NidxSearcher.Suggest: prefilter, paragraphs, entities, merge

What is kept of the reference's machinery is the INTERFACE: metadata lives in memory (no PostgreSQL), every index message
becomes one immutable segment per index (as in the reference), deletions are (key, seq) pairs applied to older segments, and
"sync" re-opens the searchers (index_cache.rs:180-200).  Scheduler, worker, merges-in-the-background, NATS, object stores other
than the local file store are outside the hot path (SURVEY 8); the RPCs served are Search, GraphSearch and Suggest.
"""
from __future__ import annotations

import itertools
import os
import threading
import uuid as _uuid
from concurrent import futures
from dataclasses import dataclass, field
from typing import Optional

import numpy as np

from . import graph as Gr
from . import json_index as J
from . import nidx_protos as P
from . import suggest as S
from . import text as T
from . import vector as V
from .shard_merge import bm25_order_key, kmerge_by


@dataclass
class _VectorIndex:
    config: V.VectorConfig
    segments: list = field(default_factory=list)     # [(OpenSegment, seq)]
    deletions: list = field(default_factory=list)    # [(key prefix, seq)]
    searcher: Optional[V.VectorSearcher] = None


@dataclass
class _Shard:
    kbid: str
    vectorsets: dict = field(default_factory=dict)   # name -> _VectorIndex
    text_segments: list = field(default_factory=list)        # [[TextDoc]] one list per index message
    paragraph_segments: list = field(default_factory=list)   # [[TextDoc]] (+ paragraph positions in .field / extra)
    deleted_resources: set = field(default_factory=set)
    json_docs: list = field(default_factory=list)            # [(resource id, [(path, kind, value)], seq)]
    resource_groups: dict = field(default_factory=dict)      # resource id -> access groups of its latest index message
    json_deletions: list = field(default_factory=list)       # [(deletion key, seq)]: json_fields_to_delete and resource deletions
    json_index: Optional[J.JsonIndex] = None
    graph_docs: list = field(default_factory=list)           # [([GraphDoc], seq)] one list per index message
    graph_index: Optional[Gr.GraphIndex] = None
    text_searcher: Optional[T.TextSearcher] = None
    paragraph_searcher: Optional[T.ParagraphSearcher] = None


def _expr_to_boolean(e) -> Optional[V.BooleanExpression]:
    """nodereader.FilterExpression (paragraph_filter) -> BooleanExpression over labels (query_io::map_expression's input)."""
    kind = e.WhichOneof("expr")
    if kind == "facet":
        return V.Literal(e.facet.facet)
    if kind == "bool_not":
        inner = _expr_to_boolean(e.bool_not)
        return V.Not(inner) if inner is not None else None
    if kind in ("bool_and", "bool_or"):
        ops = [x for x in (_expr_to_boolean(o) for o in getattr(e, kind).operands) if x is not None]
        return V.Operation("and" if kind == "bool_and" else "or", tuple(ops)) if ops else None
    return None


def _doc_matches(e, doc: T.TextDoc) -> bool:
    """nodereader.FilterExpression (field_filter) evaluated on one text document, for the facet / field / resource / and / or / not
    nodes (every other kind matches).  The search path runs TextSearcher.prefilter on the device instead; this per-document loop is
    what it replaced, kept for a stand-in library without the prefilter (the ABI emulator of the host-logic tests) and as the
    reference tests/test_prefilter_model.py compares the prefilter's model with on the nodes both evaluate."""
    kind = e.WhichOneof("expr")
    if kind == "facet":
        return any(l == e.facet.facet or l.startswith(e.facet.facet + "/") for l in doc.labels)
    if kind == "resource":
        return doc.uuid == e.resource.resource_id
    if kind == "field":
        ft, fid = e.field.field_type, e.field.field_id if e.field.HasField("field_id") else None
        return doc.field.startswith(f"/{ft}/") and (fid is None or doc.field == f"/{ft}/{fid}")
    if kind == "bool_not":
        return not _doc_matches(e.bool_not, doc)
    if kind == "bool_and":
        return all(_doc_matches(o, doc) for o in e.bool_and.operands)
    if kind == "bool_or":
        return any(_doc_matches(o, doc) for o in e.bool_or.operands)
    return True


def _json_deletes(key: str, rid: str) -> bool:
    """JsonDeletionQueryBuilder (nidx_json/src/lib.rs): a key's first 32 characters (the whole key when shorter) are a resource
    UUID, and every JSON document of that resource id goes; a key that does not parse as a UUID deletes nothing."""
    raw = key[:32] if len(key) > 32 else key
    try:
        _uuid.UUID(raw)
    except ValueError:
        return False
    return raw == rid


def _uuid_hex(rid: str) -> str:
    try:
        return _uuid.UUID(rid).hex
    except ValueError:
        return rid


def merge_graph(into, part):
    """shard_merge.rs:350-375: a shard's GraphSearchResponse appended to the merged one, its paths' node and relation indices offset
    by what is already there."""
    n_nodes, n_rels = len(into.nodes), len(into.relations)
    into.nodes.extend(part.nodes)
    into.relations.extend(part.relations)
    into.scores.extend(part.scores)
    for p in part.graph:
        q = into.graph.add()
        q.CopyFrom(p)
        q.source, q.relation, q.destination = p.source + n_nodes, p.relation + n_rels, p.destination + n_nodes


def merge_facets(shards_facets) -> dict:
    """shard_merge.rs:380-414: the counts of equal (group, tag) pairs of the shards' facet maps ({group: [(tag, total)]}) are
    summed; the merged lists are not cut again.  The reference lists them in a HashMap's order; here count descending, then tag
    in facet order."""
    counts: dict = {}
    for facets in shards_facets:
        for group, values in facets.items():
            for tag, total in values:
                counts[(group, tag)] = counts.get((group, tag), 0) + int(total)
    merged: dict = {}
    for (group, tag), total in counts.items():
        merged.setdefault(group, []).append((tag, total))
    return {g: sorted(v, key=lambda t: (-t[1], T.facet_key(t[0]) or b"")) for g, v in merged.items()}


def merge_order_key(seconds: Optional[int], order_type: int, shard_pos: int, rank: int):
    """Cross-shard order of date-ordered results (sort_documents_fn / sort_paragraphs_fn with SortExpr::Date, shard_merge.rs:235-249,
    313-328): the date in the requested direction, then the shard's position in the request, then the result's rank in its shard.
    The reference's kmerge_by leaves equal dates unpinned; this is the rule here.  Results without a date come last."""
    return T.date_sort_key(seconds, order_type) + (shard_pos, rank)


class NidxBinding:
    """nidx_binding.pyi:15-71.  ``settings`` mirrors the reference's environment schema; the keys read here are
    ``INDEXER__OBJECT_STORE`` (must be ``file``), ``INDEXER__FILE_PATH`` (where IndexMessage.storage_key points into) and
    ``NIDX_B200__DEVICE`` (CUDA ordinal, default 0)."""

    def __init__(self, settings: dict):
        import grpc

        settings = dict(settings)
        settings["INDEXER__NATS_SERVER"] = ""                      # lib.rs:73: always the in-process indexer
        self.settings = settings
        self.device = int(settings.get("NIDX_B200__DEVICE", "0"))
        self._lock = threading.RLock()
        self._shards: dict = {}
        self._seq = 1                                               # lib.rs:128-140: the sequence every index message consumes
        self._dirty = set()
        self._searcher = grpc.server(futures.ThreadPoolExecutor(max_workers=8))
        self._searcher.add_generic_rpc_handlers((grpc.method_handlers_generic_handler("nidx.NidxSearcher", {
            "Search": grpc.unary_unary_rpc_method_handler(self._grpc_search, request_deserializer=P.SearchRequest.FromString,
                                                          response_serializer=lambda m: m.SerializeToString()),
            "GraphSearch": grpc.unary_unary_rpc_method_handler(self._grpc_graph_search, request_deserializer=P.GraphSearchRequest.FromString,
                                                               response_serializer=lambda m: m.SerializeToString()),
            "Suggest": grpc.unary_unary_rpc_method_handler(self._grpc_suggest, request_deserializer=P.SuggestRequest.FromString,
                                                           response_serializer=lambda m: m.SerializeToString())}),))
        self.searcher_port = self._searcher.add_insecure_port("127.0.0.1:0")
        self._api = grpc.server(futures.ThreadPoolExecutor(max_workers=2))
        self._api.add_generic_rpc_handlers((grpc.method_handlers_generic_handler("nidx.NidxApi", {
            "NewShard": grpc.unary_unary_rpc_method_handler(self._grpc_new_shard, request_deserializer=P.NewShardRequest.FromString,
                                                            response_serializer=lambda m: m.SerializeToString())}),))
        self.api_port = self._api.add_insecure_port("127.0.0.1:0")
        self._searcher.start()
        self._api.start()

    # ---- NidxApi.NewShard (nidx.proto:9, grpc.rs) --------------------------------------------------------------------------
    def new_shard(self, kbid: str, vectorsets: dict) -> str:
        """vectorsets: name -> VectorConfig."""
        sid = str(_uuid.uuid4())
        with self._lock:
            self._shards[sid] = _Shard(kbid, {n: _VectorIndex(c) for n, c in vectorsets.items()})
        return sid

    def _grpc_new_shard(self, request, context):
        cfgs = {}
        for name, c in request.vectorsets_configs.items():
            if not c.HasField("vector_dimension"):
                import grpc

                context.abort(grpc.StatusCode.INVALID_ARGUMENT, f"vectorset {name}: vector_dimension is required")
            cfgs[name] = V.VectorConfig(dimension=int(c.vector_dimension), similarity=V.Similarity.Cosine if c.similarity == 0 else V.Similarity.Dot,
                                        normalize_vectors=bool(c.normalize_vectors), device=self.device)
        return P.ShardCreated(id=self.new_shard(request.kbid, cfgs))

    # ---- index (lib.rs:83-111 -> process_index_message) ---------------------------------------------------------------------
    def index(self, bytes: bytes) -> int:  # noqa: A002  (the reference names the parameter `bytes`: nidx_binding.pyi:45, callers may pass it by keyword)
        msg = P.IndexMessage.FromString(memoryview(bytes).tobytes())
        with self._lock:
            seq = self._seq
            self._seq += 1                                          # lib.rs:104-105: always incremented, even on failure
            try:
                self._process(msg, seq)
            except Exception as e:  # noqa: BLE001
                raise Exception(f"Error indexing {e}") from e
            self._dirty.add(msg.shard)
        return seq

    def _load_resource(self, storage_key: str):
        if self.settings.get("INDEXER__OBJECT_STORE", "file") != "file":
            raise ValueError("only the local file object store is supported (INDEXER__OBJECT_STORE=file)")
        path = os.path.join(self.settings.get("INDEXER__FILE_PATH", ""), storage_key)
        with open(path, "rb") as f:
            return P.Resource.FromString(f.read())

    def _process(self, msg, seq: int):
        shard = self._shards.get(msg.shard)
        if shard is None:
            raise KeyError(f"shard {msg.shard} not found")
        if msg.typemessage == 1:                                    # DELETION: every index drops the resource (indexer.rs delete_resource)
            for vi in shard.vectorsets.values():
                vi.deletions.append((msg.resource, seq))
            shard.deleted_resources.add((msg.resource, seq))
            shard.json_deletions.append((msg.resource, seq))
            return
        res = self._load_resource(msg.storage_key)
        rid = res.resource.uuid
        # the JSON document (nidx_json/src/resource_indexer.rs), flattened first: invalid JSON fails the message before any index
        # changes.  Its deletions are json_fields_to_delete only (JsonIndexer::deletions_for_resource), not the re-index itself
        json_entries = J.flatten({k: v.value for k, v in res.json_fields.items()}) if res.json_fields and not res.skip_json else None
        graph_docs = Gr.docs_from_resource(res) if res.field_relations else []   # a relation without source or target fails the message
        # a re-indexed resource replaces its older copies: prefixes to delete, applied to OLDER segments only (seq rule, lib.rs:188-199)
        for vi in shard.vectorsets.values():
            for key in list(res.vectors_to_delete_in_all_vectorsets) or [rid]:
                vi.deletions.append((key, seq))
        shard.deleted_resources.add((rid, seq))
        # vectors: one segment per vectorset (indexer.rs:96-146)
        for name, vi in shard.vectorsets.items():
            elems = []
            for _, paragraphs in res.paragraphs.items():
                for _, par in paragraphs.paragraphs.items():
                    sentences = par.vectorsets_sentences[name].sentences if name in par.vectorsets_sentences else par.sentences
                    for key, sentence in sentences.items():
                        if len(sentence.vector) == 0:
                            continue
                        meta = sentence.metadata.SerializeToString() if sentence.HasField("metadata") else None
                        elems.append(V.Elem(key, [np.asarray(sentence.vector, dtype=np.float32)], labels=list(par.labels), metadata=meta))
            if elems:
                vi.segments.append((V.VectorIndexer.index_elems(elems, vi.config), seq))
        # documents (nidx_text/src/resource_indexer.rs:22-91): one per field; paragraphs (nidx_paragraph): one per paragraph
        # dates (IndexMetadata, seconds: nidx_text/src/schema.rs:48-57); a resource without metadata is indexed without dates
        meta = res.metadata if res.HasField("metadata") else None
        created = meta.created.seconds if meta is not None and meta.HasField("created") else None
        modified = meta.modified.seconds if meta is not None and meta.HasField("modified") else None
        # access groups (nidx_text/src/resource_indexer.rs:49-62): every document of the resource carries them, its paragraphs too,
        # so that each keyword index evaluates SearchRequest.security over its own documents
        groups = tuple(res.security.access_groups) if res.HasField("security") else ()
        if not res.skip_texts:
            docs = [T.TextDoc(rid, "/" + fid if not fid.startswith("/") else fid, ti.text, tuple(list(res.labels) + list(ti.labels)), created, modified,
                              groups) for fid, ti in res.texts.items()]
            if docs:
                shard.text_segments.append((docs, seq))
        if not res.skip_paragraphs:
            pdocs = []
            for fid, paragraphs in res.paragraphs.items():
                text = res.texts[fid].text if fid in res.texts else ""
                for pid, par in paragraphs.paragraphs.items():
                    labels = tuple(list(res.labels) + list(res.texts[fid].labels if fid in res.texts else ()) + list(par.labels))
                    pdocs.append(T.TextDoc(rid, "/" + fid if not fid.startswith("/") else fid, text[par.start:par.end], labels, created, modified, groups,
                                           repeated=bool(par.repeated_in_field), paragraph=(pid, par)))
            if pdocs:
                shard.paragraph_segments.append((pdocs, seq))
        if graph_docs:
            shard.graph_docs.append((graph_docs, seq))
        shard.json_deletions.extend((key, seq) for key in res.json_fields_to_delete)
        if json_entries is not None:
            shard.json_docs.append((rid, json_entries, seq))
        shard.resource_groups[rid] = groups

    # ---- sync (lib.rs:113-126; searcher/sync.rs + index_cache.rs:180-200: searchers are re-opened, never mutated) --------------
    def wait_for_sync(self) -> None:
        with self._lock:
            for sid in list(self._dirty):
                self._reopen(self._shards[sid])
            self._dirty.clear()

    def _alive(self, docs_segments, deleted):
        out = []
        for docs, seq in docs_segments:
            keep = [d for d in docs if not any(d.uuid == rid and dseq > seq for rid, dseq in deleted)]
            if keep:
                out.append(keep)
        return out

    def _reopen(self, shard: _Shard):
        for vi in shard.vectorsets.values():
            vi.searcher = V.VectorSearcher.open(vi.config, vi.segments, vi.deletions) if vi.segments else None
        ts = self._alive(shard.text_segments, shard.deleted_resources)
        ps = self._alive(shard.paragraph_segments, shard.deleted_resources)
        shard.text_searcher = T.TextSearcher.open(ts, device=self.device) if ts else None
        shard.paragraph_searcher = T.ParagraphSearcher.open(ps, device=self.device) if ps else None
        # a JSON document carries its resource's groups of the latest message, which may have changed security without touching
        # the JSON document (skip_json, or no json_fields): the JSON pass must never see groups the text documents no longer have
        jd = [(rid, entries, shard.resource_groups.get(rid, ())) for rid, entries, seq in shard.json_docs
              if not any(dseq > seq and _json_deletes(key, rid) for key, dseq in shard.json_deletions)]
        if shard.json_index is not None:
            shard.json_index.close()
        shard.json_index = J.JsonIndex(jd, device=self.device) if jd else None
        # relations (nidx_relation): a newer message replaces a resource's relations, a deletion hides the older ones
        last_del: dict = {}   # resource -> its latest deletion (or replacement) seq
        for rid, dseq in shard.deleted_resources:
            r = _uuid_hex(rid)
            last_del[r] = max(last_del.get(r, 0), dseq)
        gd = [d for docs, seq in shard.graph_docs for d in docs if last_del.get(d.rid, 0) <= seq]
        if shard.graph_index is not None:
            shard.graph_index.close()
        shard.graph_index = Gr.GraphIndex(gd, device=self.device) if gd else None

    # ---- NidxSearcher.Search (shard_search.rs:60-241 + shard_merge.rs) ---------------------------------------------------------
    def search(self, request):
        """nodereader.SearchRequest -> nodereader.SearchResponse (in-process twin of the gRPC method)."""
        parts = []
        with self._lock:
            for sid in request.shard_ids:
                shard = self._shards.get(sid)
                if shard is None:
                    raise KeyError(f"shard {sid} not found")
                parts.append((sid, self._search_shard(shard, request)))
        return self._merge(request, parts)

    def _grpc_search(self, request, context):
        import grpc

        try:
            return self.search(request)
        except KeyError as e:
            context.abort(grpc.StatusCode.NOT_FOUND, str(e))
        except V.NidxError as e:
            context.abort(grpc.StatusCode.INTERNAL, str(e))
        except ValueError as e:
            context.abort(grpc.StatusCode.INVALID_ARGUMENT, str(e))

    # ---- NidxSearcher.GraphSearch (shard_search.rs:290-362, shard_merge.rs:350-375) ---------------------------------------------
    def graph_search(self, request):
        """nodereader.GraphSearchRequest -> nodereader.GraphSearchResponse: each shard's answer, concatenated in request order with its
        node and relation indices offset.  A VectorMatch leaf is NotImplementedError (semantic node / edge matches)."""
        resp = P.GraphSearchResponse()
        with self._lock:
            for sid in request.shard_ids:
                shard = self._shards.get(sid)
                if shard is None:
                    raise KeyError(f"shard {sid} not found")
                security = list(request.security.access_groups) if request.HasField("security") else None
                field_filter = request.field_filter if request.HasField("field_filter") else None
                merge_graph(resp, self._graph_shard(shard, request, field_filter, security))
        resp.shard_ids.extend(request.shard_ids)
        return resp

    def _graph_shard(self, shard: _Shard, request, field_filter, security):
        """Prefilter::parse_graph (field_filter and security only): no text index or a None result answers nothing."""
        if shard.graph_index is None:
            return P.GraphSearchResponse()
        prefilter = None
        if field_filter is not None or security is not None:
            if shard.text_searcher is None:
                return P.GraphSearchResponse()
            prefilter = shard.text_searcher.prefilter(field_filter, security=security)
        return Gr.GraphSearcher(shard.graph_index).search(request, prefilter)

    def _grpc_graph_search(self, request, context):
        import grpc

        try:
            return self.graph_search(request)
        except KeyError as e:
            context.abort(grpc.StatusCode.NOT_FOUND, str(e))
        except NotImplementedError as e:
            context.abort(grpc.StatusCode.UNIMPLEMENTED, str(e))
        except V.NidxError as e:
            context.abort(grpc.StatusCode.INTERNAL, str(e))
        except ValueError as e:
            context.abort(grpc.StatusCode.INVALID_ARGUMENT, str(e))

    # ---- NidxSearcher.Suggest (shard_suggest.rs:94-161, shard_merge.rs:101-151) --------------------------------------------------
    def suggest(self, request):
        """nodereader.SuggestRequest -> nodereader.SuggestResponse: each shard's paragraph and entity suggestions (nucliadb_b200/suggest.py),
        merged.  An unknown shard is a KeyError, a top_k above 1024 or a filter the device cannot run a ValueError."""
        parts = []
        with self._lock:
            for sid in request.shard_ids:
                shard = self._shards.get(sid)
                if shard is None:
                    raise KeyError(f"shard {sid} not found")
                parts.append((sid, self._suggest_shard(shard, request, sid)))
        return S.merge_suggest(parts, int(request.top_k))

    def _suggest_shard(self, shard: _Shard, req, sid: str):
        """SuggestPlan::build + blocking_suggest: nothing for top_k == 0 or without a feature; the prefilter of Prefilter::parse_suggest
        (field_filter and security on the text index, json_filter combined under filter_operator), whose None empties the answer; the
        paragraph pass under the suggest mask; the entity NODES search under the text part of the prefilter (json_filter does not apply
        to relations, DESIGN 9)."""
        resp = P.SuggestResponse(shard_ids=[sid])
        k = int(req.top_k)
        paragraphs, entities = P.SUGGEST_PARAGRAPHS in req.features, P.SUGGEST_ENTITIES in req.features
        if k == 0 or not (paragraphs or entities):
            return resp
        if k > S.MAX_TOP_K:
            raise ValueError(f"top_k must be at most {S.MAX_TOP_K}")
        security = list(req.security.access_groups) if req.HasField("security") else None
        field_filter = req.field_filter if req.HasField("field_filter") else None
        text_pf = None   # All
        if field_filter is not None or security is not None:
            text_pf = shard.text_searcher.prefilter(field_filter, security=security) if shard.text_searcher is not None else V.PrefilterResult.none()
        prefilter = text_pf
        if req.HasField("json_filter"):
            J.validate(req.json_filter)
            res_bits, found = None, 0
            if shard.json_index is not None:
                _, found, res_bits = shard.json_index.prefilter(req.json_filter, security)
            prefilter = (text_pf or V.PrefilterResult.all()).combine(shard.json_index, res_bits, found, req.filter_operator == P.FILTER_OR)
        if prefilter is not None and prefilter.kind == "none":
            return resp
        if paragraphs:
            resp.query = req.body
            ps = shard.paragraph_searcher
            if ps is None:
                resp.ematches.extend(S.ematches(T.paragraph_query_tokens(req.body)))
            else:
                pfilter = req.paragraph_filter if req.HasField("paragraph_filter") else None
                masks = ps.suggest_masks(security, pfilter, prefilter, req.filter_operator == P.FILTER_OR)
                r = ps.suggest(req.body, k, masks)
                resp.total = len(r.hits)
                resp.ematches.extend(r.ematches)
                for h in r.hits[: S.RESULTS_PER_PAGE]:
                    d = ps.segments[h.segment].docs[h.doc]
                    pid, par = d.paragraph
                    o = resp.results.add(uuid=d.uuid, field=d.field, start=par.start, end=par.end, paragraph=pid, split=par.split, index=par.index)
                    o.labels.extend(S.extract_labels(d.labels))
                    if par.HasField("metadata"):
                        o.metadata.CopyFrom(par.metadata)
                    o.score.bm25, o.score.docaddr = h.score, (h.segment << 32) + h.doc
                    o.matches.extend(h.matches)
        if entities:
            resp.entity_results.SetInParent()
            greq = S.entity_request(req.body, k)
            if greq is not None and shard.graph_index is not None:
                resp.entity_results.nodes.extend(Gr.GraphSearcher(shard.graph_index).search(greq, text_pf).nodes)
        return resp

    def _grpc_suggest(self, request, context):
        import grpc

        try:
            return self.suggest(request)
        except KeyError as e:
            context.abort(grpc.StatusCode.NOT_FOUND, str(e))
        except V.NidxError as e:
            context.abort(grpc.StatusCode.INTERNAL, str(e))
        except ValueError as e:
            context.abort(grpc.StatusCode.INVALID_ARGUMENT, str(e))

    def _search_shard(self, shard: _Shard, req):
        k = int(req.result_per_page)
        out = {}
        order = T.OrderBy(sort_by=int(req.order.sort_by), type=int(req.order.type)) if req.HasField("order") else None
        # prefilter (shard_search.rs:108-137, query_planner/prefilter.rs:106-160): field_filter and security evaluated on the device
        # over the documents -> the fields that may answer
        security = list(req.security.access_groups) if req.HasField("security") else None
        field_filter = req.field_filter if req.HasField("field_filter") else None
        prefilter = V.PrefilterResult.all()
        if security is not None and shard.text_searcher is None:   # no document to grant access through
            prefilter = V.PrefilterResult.none()
        elif (field_filter is not None or security is not None) and shard.text_searcher is not None:
            if security is not None or hasattr(V._lib.load(), "nidx_txt_prefilter"):
                prefilter = shard.text_searcher.prefilter(field_filter, security=security)
            else:   # a stand-in for libnidx_b200.so without the prefilter (the ABI emulator of the host-logic tests): the host loop
                fields = [V.FieldId(_uuid.UUID(d.uuid), d.field) for seg in shard.text_searcher.segments for d in seg.docs if _doc_matches(req.field_filter, d)]
                prefilter = V.PrefilterResult.some(fields) if fields else V.PrefilterResult.none()
        # SearchRequest.graph_search (query_planner.rs:291-300): a PATH search with top_k = max(result_per_page, 20), prefiltered as
        # GraphSearch is (_graph_shard: field_filter and security; json_filter does not apply to relations, DESIGN 9)
        if req.HasField("graph_search"):
            greq = P.GraphSearchRequest(query=req.graph_search.query, kind=Gr.PATH, top_k=max(k, 20))
            out["graph"] = self._graph_shard(shard, greq, field_filter, security)
        # the JSON prefilter (query_planner/prefilter.rs:24-72): the JSON resource set, ANDed on the device with security, combined
        # with the text result under filter_operator (PrefilterResult::combine).  Security is applied outside the combination:
        # AND(security, op(field_filter, json)), so a security filter is never widened (DESIGN 7)
        masks = None
        if req.HasField("json_filter"):
            J.validate(req.json_filter)
            res_bits, found = None, 0
            if shard.json_index is not None:
                _, found, res_bits = shard.json_index.prefilter(req.json_filter, security)
            prefilter = prefilter.combine(shard.json_index, res_bits, found, req.filter_operator == P.FILTER_OR)
            if prefilter.kind == "none":   # IndexQueries::apply_prefilter: the sections are absent
                return out
            if prefilter.on_device and req.paragraph and shard.paragraph_searcher is not None:
                masks = shard.paragraph_searcher.json_masks(security, prefilter)
        if len(req.vector):
            name = req.vectorset
            if name not in shard.vectorsets:
                raise ValueError(f"vectorset {name!r} not found")          # shard_search.rs:95-99 InvalidArgument
            vi = shard.vectorsets[name]
            formula = _expr_to_boolean(req.paragraph_filter) if req.HasField("paragraph_filter") else None
            vreq = V.VectorSearchRequest(vector=list(req.vector), result_per_page=k, with_duplicates=bool(req.with_duplicates), vector_set=name,
                                         min_score=float(req.min_score_semantic), filtering_formula=formula,
                                         filter_operator=V.FilterOperator.Or if req.filter_operator == P.FILTER_OR else V.FilterOperator.And)
            out["vector"] = vi.searcher.search(vreq, prefilter).documents if vi.searcher is not None else []
        if req.document and shard.text_searcher is not None:
            out["document"] = shard.text_searcher.search(T.DocumentSearchRequest(body=req.body, result_per_page=k, min_score=float(req.min_score_bm25),
                                                                                 faceted=list(req.faceted.labels), only_faceted=bool(req.only_faceted), order=order,
                                                                                 security=security))
        if req.paragraph and shard.paragraph_searcher is not None:
            after = None
            if req.HasField("search_after"):
                after = T.SearchAfter(score=req.search_after.score, tie_break="keep_after", docaddr=int(req.search_after.docaddr))
            out["paragraph"] = shard.paragraph_searcher.search(T.DocumentSearchRequest(body=req.body, result_per_page=k, min_score=float(req.min_score_bm25), search_after=after,
                                                                                       faceted=list(req.faceted.labels), only_faceted=bool(req.only_faceted), order=order,
                                                                                       security=security), masks=masks)
        return out

    def _merge(self, req, parts):
        k = int(req.result_per_page)
        resp = P.SearchResponse()
        resp.shard_ids.extend(sid for sid, _ in parts)
        if req.HasField("graph_search"):
            for _, p in parts:
                if "graph" in p:
                    merge_graph(resp.graph, p["graph"])
        # vectors: kmerge_by(score >=), take(k) (shard_merge.rs:332-348), shards in request order standing for the reference's
        # `responses` order; equal scores come out in the order itertools' heap gives them, not first shard first
        merged = kmerge_by([p.get("vector", []) for _, p in parts], lambda a, b: a.score >= b.score)
        vec = [d for _, d in itertools.islice(merged, max(k, 0))]
        for d in vec:
            ds = resp.vector.documents.add()
            ds.doc_id.id, ds.score = d.doc_id, d.score
            ds.labels.extend(d.labels)
            if d.metadata:
                ds.metadata.CopyFrom(P.SentenceMetadata.FromString(d.metadata))
        # documents / paragraphs: bm25 desc (total_cmp), then shard_id bytes descending, then lower docaddr (shard_merge.rs:211-231,
        # 289-309); the bytes are those written to `shard_id` below.  Under an order by date (merge_order_key), the sort value is the date
        ordered = req.HasField("order")
        for kind, target in (("document", resp.document), ("paragraph", resp.paragraph)):
            found = [(sid, p[kind]) for sid, p in parts if kind in p]
            if not found:
                continue
            if ordered:
                rows = sorted(((merge_order_key(r.date, int(req.order.type), i, j), i, 0, sid, r) for i, (sid, rs) in enumerate(found) for j, r in enumerate(rs.results)),
                              key=lambda t: t[0])
            else:
                rows = sorted(((bm25_order_key(r.score.bm25, sid.encode(), r.score.docaddr), i, 0, sid, r) for i, (sid, rs) in enumerate(found) for r in rs.results),
                              key=lambda t: t[0])
            target.total = sum(rs.total for _, rs in found)
            target.next_page = any(rs.next_page for _, rs in found) or len(rows) > k
            target.query = req.body
            for group, values in merge_facets([{g: [(f.tag, f.total) for f in v] for g, v in rs.facets.items()} for _, rs in found]).items():
                target.facets[group].facetresults.extend(P.FacetResult(tag=tag, total=total) for tag, total in values)
            for _, _, _, sid, r in rows[:k]:
                o = target.results.add()
                o.uuid, o.field = r.uuid, r.field
                if not ordered:
                    o.score.bm25, o.score.docaddr = r.score.bm25, r.score.docaddr
                elif r.date is not None:
                    o.date.seconds, o.date.nanos = r.date, 0   # second precision: {seconds, nanos: 0} (nidx_text/src/schema.rs:48-57)
                o.labels.extend(r.labels)
                o.shard_id = sid.encode()
        return resp

    def close(self):
        """Stop the servers and release every device-resident segment (the reference's Drop cancels its runtime)."""
        if getattr(self, "_closed", False):
            return
        self._closed = True
        self._searcher.stop(0)
        self._api.stop(0)
        with self._lock:
            for shard in self._shards.values():
                for vi in shard.vectorsets.values():
                    vi.searcher = None
                    for seg, _ in vi.segments:
                        seg.close()
                    vi.segments.clear()
                for searcher in (shard.text_searcher, shard.paragraph_searcher):
                    if searcher is not None:
                        for seg in searcher.segments:
                            if seg._gpu is not None:
                                seg._gpu.close()
                shard.text_searcher = shard.paragraph_searcher = None
                if shard.json_index is not None:
                    shard.json_index.close()
                    shard.json_index = None
                if shard.graph_index is not None:
                    shard.graph_index.close()
                    shard.graph_index = None
            self._shards.clear()

    def __del__(self):   # lib.rs Drop: the cancellation token
        try:
            self.close()
        except Exception:
            pass
