"""The wire schema of the nidx searcher / indexer that the hot path needs, built at import time from descriptors written by
hand (there is no protoc in this image): same packages, message names, field names, numbers and types as the reference's
``nidx/nidx_protos/{nidx,nodereader,noderesources,nodewriter}.proto`` for the SUBSET of fields the search path reads or writes
(cited per message below).  Fields that are not declared here are skipped by the protobuf runtime as unknown fields, so requests
serialised by the reference's clients (``nidx_protos`` / ``nucliadb_protos``) decode, and the responses decode on their side.

    SearchRequest / SearchResponse                         nodereader.proto:388-437, 476-488
    Faceted, FacetResult, FacetResults                     nodereader.proto:20-22, 40-46
    OrderBy                                                nodereader.proto:24-38
    DocumentSearchResponse / DocumentResult / ResultScore  nodereader.proto:48-81
    ParagraphSearchResponse / ParagraphResult              nodereader.proto:83-124
    VectorSearchResponse / DocumentScored                  nodereader.proto:126-142
    FilterExpression, FilterOperator, SearchAfter          nodereader.proto:287-336, 382-386
    IndexMessage, TypeMessage                              nodewriter.proto:26-43
    Resource, IndexParagraph(s), VectorSentence, ...       noderesources.proto:8-180
    IndexMetadata                                          noderesources.proto:17-20 (google.protobuf.Timestamp)
    Security (Resource.security, SearchRequest.security)   nucliadb_protos utils.proto: repeated string access_groups = 1
    JsonFieldValue, Resource.json_fields / skip_json       noderesources.proto:13-15, 169-176
    JsonFilterExpression, JsonFieldPathFilter              nodereader.proto:338-380 (SearchRequest.json_filter = 32)
    GraphQuery, GraphSearchRequest / Response              nodereader.proto:148-290 (SearchRequest.graph_search = 29, SearchResponse.graph = 5)
    Relation, RelationNode, RelationMetadata, IndexRelation(s), Resource.field_relations   utils.proto, noderesources.proto
    SuggestFeatures, SuggestRequest / Response, RelationPrefixSearchResponse   nodereader.proto (NidxSearcher.Suggest)
"""
from __future__ import annotations

from google.protobuf import descriptor_pb2, descriptor_pool, message_factory, timestamp_pb2

_F = descriptor_pb2.FieldDescriptorProto
_T = {"string": _F.TYPE_STRING, "bytes": _F.TYPE_BYTES, "int32": _F.TYPE_INT32, "int64": _F.TYPE_INT64, "uint32": _F.TYPE_UINT32, "uint64": _F.TYPE_UINT64,
      "float": _F.TYPE_FLOAT, "double": _F.TYPE_DOUBLE, "bool": _F.TYPE_BOOL}


def _field(msg, name, number, typ, repeated=False, oneof=None, optional=False):
    f = msg.field.add()
    f.name, f.number = name, number
    f.label = _F.LABEL_REPEATED if repeated else _F.LABEL_OPTIONAL
    if typ in _T:
        f.type = _T[typ]
    elif typ.startswith("enum:"):
        f.type, f.type_name = _F.TYPE_ENUM, typ[5:]
    else:
        f.type, f.type_name = _F.TYPE_MESSAGE, typ
    if oneof is not None:
        f.oneof_index = oneof
    if optional:  # proto3 `optional`: a synthetic one-field oneof
        msg.oneof_decl.add().name = "_" + name
        f.oneof_index = len(msg.oneof_decl) - 1
        f.proto3_optional = True
    return f


def _map(msg, pkg_path, name, number, key_type, value_type):
    """map<key, value> name = number  ==  repeated NameEntry (map_entry) with key = 1, value = 2."""
    entry = msg.nested_type.add()
    entry.name = "".join(p.capitalize() for p in name.split("_")) + "Entry"
    entry.options.map_entry = True
    _field(entry, "key", 1, key_type)
    _field(entry, "value", 2, value_type)
    _field(msg, name, number, f"{pkg_path}.{entry.name}", repeated=True)


def _build():
    pool = descriptor_pool.DescriptorPool()
    ts = descriptor_pb2.FileDescriptorProto()   # google/protobuf/timestamp.proto, as the protobuf runtime ships it
    timestamp_pb2.DESCRIPTOR.CopyToProto(ts)
    pool.Add(ts)

    # ---- utils.proto (nucliadb_protos) ---------------------------------------------------------------------------------------
    fd = descriptor_pb2.FileDescriptorProto(name="nucliadb_protos/utils.proto", package="utils", syntax="proto3")
    m = fd.message_type.add(name="Security")
    _field(m, "access_groups", 1, "string", repeated=True)
    m = fd.message_type.add(name="RelationNode")                   # utils.proto: RelationNode
    e = m.enum_type.add(name="NodeType")
    for i, n in enumerate(("ENTITY", "LABEL", "RESOURCE", "USER")):
        e.value.add(name=n, number=i)
    _field(m, "value", 4, "string"); _field(m, "ntype", 5, "enum:.utils.RelationNode.NodeType"); _field(m, "subtype", 6, "string")
    m = fd.message_type.add(name="RelationMetadata")
    _field(m, "paragraph_id", 1, "string", optional=True); _field(m, "source_start", 2, "int32", optional=True)
    _field(m, "source_end", 3, "int32", optional=True); _field(m, "to_start", 4, "int32", optional=True); _field(m, "to_end", 5, "int32", optional=True)
    _field(m, "data_augmentation_task_id", 6, "string", optional=True)
    m = fd.message_type.add(name="Relation")
    e = m.enum_type.add(name="RelationType")
    for i, n in enumerate(("CHILD", "ABOUT", "ENTITY", "COLAB", "SYNONYM", "OTHER")):
        e.value.add(name=n, number=i)
    _field(m, "relation", 5, "enum:.utils.Relation.RelationType"); _field(m, "source", 6, ".utils.RelationNode"); _field(m, "to", 7, ".utils.RelationNode")
    _field(m, "relation_label", 8, "string"); _field(m, "metadata", 9, ".utils.RelationMetadata")
    pool.Add(fd)

    # ---- noderesources.proto ---------------------------------------------------------------------------------------------
    fd = descriptor_pb2.FileDescriptorProto(name="nidx_protos/noderesources.proto", package="noderesources", syntax="proto3",
                                            dependency=["google/protobuf/timestamp.proto", "nucliadb_protos/utils.proto"])
    m = fd.message_type.add(name="TextInformation")           # :8-11
    _field(m, "text", 1, "string"); _field(m, "labels", 2, "string", repeated=True)
    m = fd.message_type.add(name="JsonFieldValue")            # :13-15: a JSON-encoded value
    _field(m, "value", 1, "string")
    m = fd.message_type.add(name="ResourceID")                # :36-39
    _field(m, "shard_id", 1, "string"); _field(m, "uuid", 2, "string")
    m = fd.message_type.add(name="IndexMetadata")             # :17-20
    _field(m, "modified", 1, ".google.protobuf.Timestamp"); _field(m, "created", 2, ".google.protobuf.Timestamp")
    m = fd.message_type.add(name="Position")                  # :53-67
    _field(m, "index", 1, "uint64"); _field(m, "start", 2, "uint64"); _field(m, "end", 3, "uint64"); _field(m, "page_number", 4, "uint64")
    _field(m, "start_seconds", 5, "uint32", repeated=True); _field(m, "end_seconds", 6, "uint32", repeated=True); _field(m, "in_page", 7, "bool")
    m = fd.message_type.add(name="Representation")            # :69-72
    _field(m, "is_a_table", 1, "bool"); _field(m, "file", 2, "string")
    for name in ("SentenceMetadata", "ParagraphMetadata"):    # :74-78, 89-93
        m = fd.message_type.add(name=name)
        _field(m, "position", 1, ".noderesources.Position"); _field(m, "page_with_visual", 2, "bool"); _field(m, "representation", 3, ".noderesources.Representation")
    m = fd.message_type.add(name="VectorSentence")            # :80-83
    _field(m, "vector", 1, "float", repeated=True); _field(m, "metadata", 9, ".noderesources.SentenceMetadata")
    m = fd.message_type.add(name="VectorsetSentences")        # :85-87
    _map(m, ".noderesources.VectorsetSentences", "sentences", 1, "string", ".noderesources.VectorSentence")
    m = fd.message_type.add(name="IndexParagraph")            # :95-106
    _field(m, "start", 1, "int32"); _field(m, "end", 2, "int32"); _field(m, "labels", 3, "string", repeated=True)
    _map(m, ".noderesources.IndexParagraph", "sentences", 4, "string", ".noderesources.VectorSentence")
    _field(m, "field", 5, "string"); _field(m, "split", 6, "string"); _field(m, "index", 7, "uint64"); _field(m, "repeated_in_field", 8, "bool")
    _field(m, "metadata", 9, ".noderesources.ParagraphMetadata")
    _map(m, ".noderesources.IndexParagraph", "vectorsets_sentences", 10, "string", ".noderesources.VectorsetSentences")
    m = fd.message_type.add(name="IndexParagraphs")           # :118-121
    _map(m, ".noderesources.IndexParagraphs", "paragraphs", 1, "string", ".noderesources.IndexParagraph")
    m = fd.message_type.add(name="IndexRelation")             # IndexRelation / IndexRelations
    _field(m, "relation", 1, ".utils.Relation"); _field(m, "resource_field_id", 2, "string"); _field(m, "facets", 3, "string", repeated=True)
    m = fd.message_type.add(name="IndexRelations")
    _field(m, "relations", 1, ".noderesources.IndexRelation", repeated=True)
    m = fd.message_type.add(name="Resource")                  # :123-180
    _field(m, "resource", 1, ".noderesources.ResourceID"); _field(m, "metadata", 2, ".noderesources.IndexMetadata")
    _map(m, ".noderesources.Resource", "texts", 3, "string", ".noderesources.TextInformation")
    _field(m, "labels", 4, "string", repeated=True)
    _map(m, ".noderesources.Resource", "paragraphs", 6, "string", ".noderesources.IndexParagraphs")
    _field(m, "paragraphs_to_delete", 7, "string", repeated=True)
    _field(m, "vectors_to_delete_in_all_vectorsets", 8, "string", repeated=True)
    _field(m, "shard_id", 11, "string"); _field(m, "security", 14, ".utils.Security", optional=True)
    _field(m, "texts_to_delete", 17, "string", repeated=True)
    _field(m, "skip_texts", 18, "bool"); _field(m, "skip_paragraphs", 19, "bool")
    _map(m, ".noderesources.Resource", "json_fields", 22, "string", ".noderesources.JsonFieldValue")
    _field(m, "json_fields_to_delete", 23, "string", repeated=True); _field(m, "skip_json", 24, "bool")
    _map(m, ".noderesources.Resource", "field_relations", 10, "string", ".noderesources.IndexRelations")
    pool.Add(fd)

    # ---- nodereader.proto ------------------------------------------------------------------------------------------------
    fd = descriptor_pb2.FileDescriptorProto(name="nidx_protos/nodereader.proto", package="nodereader", syntax="proto3",
                                            dependency=["nidx_protos/noderesources.proto", "google/protobuf/timestamp.proto", "nucliadb_protos/utils.proto"])
    e = fd.enum_type.add(name="FilterOperator")               # :333-336
    e.value.add(name="AND", number=0); e.value.add(name="OR", number=1)
    m = fd.message_type.add(name="Faceted")                   # :20-22
    _field(m, "labels", 1, "string", repeated=True)
    m = fd.message_type.add(name="FacetResult")               # :40-43
    _field(m, "tag", 1, "string"); _field(m, "total", 2, "int32")
    m = fd.message_type.add(name="FacetResults")              # :44-46
    _field(m, "facetresults", 1, ".nodereader.FacetResult", repeated=True)
    m = fd.message_type.add(name="OrderBy")                   # :24-38
    e = m.enum_type.add(name="OrderType"); e.value.add(name="DESC", number=0); e.value.add(name="ASC", number=1)
    e = m.enum_type.add(name="OrderField"); e.value.add(name="CREATED", number=0); e.value.add(name="MODIFIED", number=1)
    _field(m, "type", 2, "enum:.nodereader.OrderBy.OrderType"); _field(m, "sort_by", 3, "enum:.nodereader.OrderBy.OrderField")
    m = fd.message_type.add(name="ResultScore")               # :48-53
    _field(m, "bm25", 1, "float"); _field(m, "docaddr", 3, "uint64")
    m = fd.message_type.add(name="DocumentResult")            # :55-64
    m.oneof_decl.add().name = "sort_value"
    _field(m, "uuid", 1, "string"); _field(m, "score", 3, ".nodereader.ResultScore", oneof=0); _field(m, "field", 4, "string")
    _field(m, "labels", 5, "string", repeated=True); _field(m, "shard_id", 7, "bytes"); _field(m, "date", 6, ".google.protobuf.Timestamp", oneof=0)
    m = fd.message_type.add(name="DocumentSearchResponse")    # :66-81
    _field(m, "total", 1, "int32"); _field(m, "results", 2, ".nodereader.DocumentResult", repeated=True); _field(m, "query", 6, "string")
    _field(m, "next_page", 7, "bool"); _map(m, ".nodereader.DocumentSearchResponse", "facets", 3, "string", ".nodereader.FacetResults")
    m = fd.message_type.add(name="ParagraphResult")           # :83-104
    m.oneof_decl.add().name = "sort_value"
    _field(m, "uuid", 1, "string"); _field(m, "field", 3, "string"); _field(m, "start", 4, "uint64"); _field(m, "end", 5, "uint64")
    _field(m, "paragraph", 6, "string"); _field(m, "split", 7, "string"); _field(m, "index", 8, "uint64")
    _field(m, "score", 9, ".nodereader.ResultScore", oneof=0); _field(m, "matches", 10, "string", repeated=True)
    _field(m, "metadata", 11, ".noderesources.ParagraphMetadata"); _field(m, "labels", 12, "string", repeated=True); _field(m, "shard_id", 14, "bytes")
    _field(m, "date", 13, ".google.protobuf.Timestamp", oneof=0)
    m = fd.message_type.add(name="ParagraphSearchResponse")   # :106-124
    _field(m, "total", 1, "int32"); _field(m, "results", 2, ".nodereader.ParagraphResult", repeated=True); _field(m, "query", 6, "string")
    _field(m, "next_page", 7, "bool"); _field(m, "ematches", 9, "string", repeated=True)
    _map(m, ".nodereader.ParagraphSearchResponse", "facets", 3, "string", ".nodereader.FacetResults")
    m = fd.message_type.add(name="DocumentVectorIdentifier")  # :126-128
    _field(m, "id", 1, "string")
    m = fd.message_type.add(name="DocumentScored")            # :130-135
    _field(m, "doc_id", 1, ".nodereader.DocumentVectorIdentifier"); _field(m, "score", 2, "float")
    _field(m, "metadata", 3, ".noderesources.SentenceMetadata"); _field(m, "labels", 4, "string", repeated=True)
    m = fd.message_type.add(name="VectorSearchResponse")      # :137-142
    _field(m, "documents", 1, ".nodereader.DocumentScored", repeated=True)
    m = fd.message_type.add(name="FilterExpression")          # :287-331
    lst = m.nested_type.add(name="FilterExpressionList"); _field(lst, "operands", 1, ".nodereader.FilterExpression", repeated=True)
    r = m.nested_type.add(name="ResourceFilter"); _field(r, "resource_id", 1, "string")
    ff = m.nested_type.add(name="FieldFilter"); _field(ff, "field_type", 1, "string"); _field(ff, "field_id", 2, "string", optional=True)
    kw = m.nested_type.add(name="KeywordFilter"); _field(kw, "keyword", 1, "string")
    fc = m.nested_type.add(name="FacetFilter"); _field(fc, "facet", 1, "string")
    dr = m.nested_type.add(name="DateRangeFilter")
    e = dr.enum_type.add(name="DateField"); e.value.add(name="CREATED", number=0); e.value.add(name="MODIFIED", number=1)
    _field(dr, "field", 1, "enum:.nodereader.FilterExpression.DateRangeFilter.DateField")
    _field(dr, "since", 2, ".google.protobuf.Timestamp", optional=True); _field(dr, "until", 3, ".google.protobuf.Timestamp", optional=True)
    rfp = m.nested_type.add(name="ResourceFieldPrefixFilter")
    _field(rfp, "resource_id", 1, "string"); _field(rfp, "field_type", 2, "string"); _field(rfp, "field_id_prefix", 3, "string")
    m.oneof_decl.add().name = "expr"
    _field(m, "bool_and", 1, ".nodereader.FilterExpression.FilterExpressionList", oneof=0)
    _field(m, "bool_or", 2, ".nodereader.FilterExpression.FilterExpressionList", oneof=0)
    _field(m, "bool_not", 3, ".nodereader.FilterExpression", oneof=0)
    _field(m, "resource", 4, ".nodereader.FilterExpression.ResourceFilter", oneof=0)
    _field(m, "field", 5, ".nodereader.FilterExpression.FieldFilter", oneof=0)
    _field(m, "keyword", 6, ".nodereader.FilterExpression.KeywordFilter", oneof=0)
    _field(m, "date", 7, ".nodereader.FilterExpression.DateRangeFilter", oneof=0)
    _field(m, "facet", 8, ".nodereader.FilterExpression.FacetFilter", oneof=0)
    _field(m, "resource_field_prefix", 9, ".nodereader.FilterExpression.ResourceFieldPrefixFilter", oneof=0)
    m = fd.message_type.add(name="JsonFieldPathFilter")       # :338-367
    _field(m, "field_id", 1, "string"); _field(m, "json_path", 2, "string")
    ir = m.nested_type.add(name="IntegerRangePredicate"); _field(ir, "lower", 1, "int64", optional=True); _field(ir, "upper", 2, "int64", optional=True)
    fr = m.nested_type.add(name="FloatRangePredicate"); _field(fr, "lower", 1, "double", optional=True); _field(fr, "upper", 2, "double", optional=True)
    dr = m.nested_type.add(name="DateRangePredicate")
    _field(dr, "lower", 1, ".google.protobuf.Timestamp", optional=True); _field(dr, "upper", 2, ".google.protobuf.Timestamp", optional=True)
    m.oneof_decl.add().name = "predicate"
    _field(m, "text", 3, "string", oneof=0); _field(m, "boolean", 6, "bool", oneof=0); _field(m, "int", 8, "int64", oneof=0)
    _field(m, "float", 9, "double", oneof=0); _field(m, "date", 10, ".google.protobuf.Timestamp", oneof=0)
    _field(m, "int_range", 4, ".nodereader.JsonFieldPathFilter.IntegerRangePredicate", oneof=0)
    _field(m, "float_range", 5, ".nodereader.JsonFieldPathFilter.FloatRangePredicate", oneof=0)
    _field(m, "date_range", 7, ".nodereader.JsonFieldPathFilter.DateRangePredicate", oneof=0)
    m = fd.message_type.add(name="JsonFilterExpression")      # :369-380
    lst = m.nested_type.add(name="List"); _field(lst, "operands", 1, ".nodereader.JsonFilterExpression", repeated=True)
    m.oneof_decl.add().name = "expr"
    _field(m, "bool_and", 1, ".nodereader.JsonFilterExpression.List", oneof=0)
    _field(m, "bool_or", 2, ".nodereader.JsonFilterExpression.List", oneof=0)
    _field(m, "bool_not", 3, ".nodereader.JsonFilterExpression", oneof=0)
    _field(m, "path", 4, ".nodereader.JsonFieldPathFilter", oneof=0)
    m = fd.message_type.add(name="SearchAfter")               # :382-386
    _field(m, "score", 1, "float"); _field(m, "shard_id", 2, "bytes"); _field(m, "docaddr", 3, "uint64")
    m = fd.message_type.add(name="GraphQuery")                # :148-231
    nd = m.nested_type.add(name="Node")
    e = nd.enum_type.add(name="MatchLocation")
    for i, n in enumerate(("FULL", "PREFIX", "WORDS", "PREFIX_WORDS")):
        e.value.add(name=n, number=i)
    em = nd.nested_type.add(name="ExactMatch"); _field(em, "kind", 1, "enum:.nodereader.GraphQuery.Node.MatchLocation")
    fm = nd.nested_type.add(name="FuzzyMatch"); _field(fm, "kind", 1, "enum:.nodereader.GraphQuery.Node.MatchLocation"); _field(fm, "distance", 2, "uint32")
    vm = nd.nested_type.add(name="VectorMatch"); _field(vm, "vector", 1, "float", repeated=True)
    nd.oneof_decl.add().name = "match_kind"
    _field(nd, "exact", 5, ".nodereader.GraphQuery.Node.ExactMatch", oneof=0); _field(nd, "fuzzy", 6, ".nodereader.GraphQuery.Node.FuzzyMatch", oneof=0)
    _field(nd, "vector", 7, ".nodereader.GraphQuery.Node.VectorMatch", oneof=0)
    _field(nd, "value", 1, "string", optional=True); _field(nd, "node_type", 2, "enum:.utils.RelationNode.NodeType", optional=True)
    _field(nd, "node_subtype", 3, "string", optional=True)
    rl = m.nested_type.add(name="Relation")
    rl.nested_type.add(name="ExactMatch")
    vm = rl.nested_type.add(name="VectorMatch"); _field(vm, "vector", 1, "float", repeated=True)
    rl.oneof_decl.add().name = "match_kind"
    _field(rl, "exact", 3, ".nodereader.GraphQuery.Relation.ExactMatch", oneof=0); _field(rl, "vector", 4, ".nodereader.GraphQuery.Relation.VectorMatch", oneof=0)
    _field(rl, "value", 1, "string", optional=True); _field(rl, "relation_type", 2, "enum:.utils.Relation.RelationType", optional=True)
    pa = m.nested_type.add(name="Path")
    _field(pa, "source", 1, ".nodereader.GraphQuery.Node"); _field(pa, "relation", 2, ".nodereader.GraphQuery.Relation")
    _field(pa, "destination", 3, ".nodereader.GraphQuery.Node"); _field(pa, "undirected", 4, "bool")
    bq = m.nested_type.add(name="BoolQuery"); _field(bq, "operands", 1, ".nodereader.GraphQuery.PathQuery", repeated=True)
    ff = m.nested_type.add(name="FacetFilter"); _field(ff, "facet", 1, "string")
    pq = m.nested_type.add(name="PathQuery")
    pq.oneof_decl.add().name = "query"
    _field(pq, "path", 1, ".nodereader.GraphQuery.Path", oneof=0); _field(pq, "bool_not", 2, ".nodereader.GraphQuery.PathQuery", oneof=0)
    _field(pq, "bool_and", 3, ".nodereader.GraphQuery.BoolQuery", oneof=0); _field(pq, "bool_or", 4, ".nodereader.GraphQuery.BoolQuery", oneof=0)
    _field(pq, "facet", 5, ".nodereader.GraphQuery.FacetFilter", oneof=0)
    _field(m, "path", 1, ".nodereader.GraphQuery.PathQuery")
    m = fd.message_type.add(name="GraphSearchRequest")        # :233-262
    e = m.enum_type.add(name="QueryKind"); e.value.add(name="PATH", number=0); e.value.add(name="NODES", number=1); e.value.add(name="RELATIONS", number=2)
    _field(m, "shard_ids", 1, "string", repeated=True); _field(m, "query", 2, ".nodereader.GraphQuery")
    _field(m, "kind", 3, "enum:.nodereader.GraphSearchRequest.QueryKind"); _field(m, "top_k", 4, "uint32")
    _field(m, "security", 5, ".utils.Security", optional=True); _field(m, "field_filter", 6, ".nodereader.FilterExpression", optional=True)
    _field(m, "graph_node_vectorset", 7, "string"); _field(m, "graph_edge_vectorset", 8, "string")
    _field(m, "min_score_node_semantic", 9, "float"); _field(m, "min_score_edge_semantic", 10, "float")
    m = fd.message_type.add(name="GraphSearchResponse")       # :264-290
    rl = m.nested_type.add(name="Relation"); _field(rl, "relation_type", 1, "enum:.utils.Relation.RelationType"); _field(rl, "label", 2, "string")
    pa = m.nested_type.add(name="Path")
    _field(pa, "source", 1, "uint32"); _field(pa, "relation", 2, "uint32"); _field(pa, "destination", 3, "uint32")
    _field(pa, "metadata", 4, ".utils.RelationMetadata", optional=True); _field(pa, "resource_field_id", 5, "string", optional=True)
    _field(pa, "facets", 6, "string", repeated=True)
    _field(m, "nodes", 1, ".utils.RelationNode", repeated=True); _field(m, "relations", 2, ".nodereader.GraphSearchResponse.Relation", repeated=True)
    _field(m, "graph", 3, ".nodereader.GraphSearchResponse.Path", repeated=True); _field(m, "scores", 4, "float", repeated=True)
    _field(m, "shard_ids", 5, "string", repeated=True)
    m = fd.message_type.add(name="SearchRequest")             # :388-437
    _field(m, "shard_ids", 1, "string", repeated=True); _field(m, "body", 3, "string"); _field(m, "order", 5, ".nodereader.OrderBy")
    _field(m, "faceted", 6, ".nodereader.Faceted")
    _field(m, "result_per_page", 8, "int32")
    _field(m, "vector", 10, "float", repeated=True); _field(m, "paragraph", 12, "bool"); _field(m, "document", 13, "bool")
    _field(m, "with_duplicates", 14, "bool"); _field(m, "vectorset", 15, "string"); _field(m, "only_faceted", 16, "bool")
    _field(m, "min_score_semantic", 23, "float"); _field(m, "security", 24, ".utils.Security", optional=True); _field(m, "min_score_bm25", 25, "float")
    _field(m, "field_filter", 26, ".nodereader.FilterExpression", optional=True); _field(m, "paragraph_filter", 27, ".nodereader.FilterExpression", optional=True)
    _field(m, "filter_operator", 28, "enum:.nodereader.FilterOperator"); _field(m, "search_after", 35, ".nodereader.SearchAfter", optional=True)
    _field(m, "json_filter", 32, ".nodereader.JsonFilterExpression", optional=True)
    gs = m.nested_type.add(name="GraphSearch"); _field(gs, "query", 1, ".nodereader.GraphQuery")
    _field(m, "graph_search", 29, ".nodereader.SearchRequest.GraphSearch", optional=True)
    m = fd.message_type.add(name="SearchResponse")            # :476-488
    _field(m, "document", 1, ".nodereader.DocumentSearchResponse"); _field(m, "paragraph", 2, ".nodereader.ParagraphSearchResponse")
    _field(m, "vector", 3, ".nodereader.VectorSearchResponse"); _field(m, "shard_ids", 6, "string", repeated=True)
    _field(m, "graph", 5, ".nodereader.GraphSearchResponse")
    e = fd.enum_type.add(name="SuggestFeatures")              # :439-442
    e.value.add(name="ENTITIES", number=0); e.value.add(name="PARAGRAPHS", number=1)
    m = fd.message_type.add(name="SuggestRequest")            # :444-457
    _field(m, "shard_ids", 1, "string", repeated=True); _field(m, "body", 2, "string")
    _field(m, "features", 6, "enum:.nodereader.SuggestFeatures", repeated=True)
    _field(m, "field_filter", 7, ".nodereader.FilterExpression", optional=True); _field(m, "paragraph_filter", 8, ".nodereader.FilterExpression", optional=True)
    _field(m, "filter_operator", 9, "enum:.nodereader.FilterOperator"); _field(m, "security", 10, ".utils.Security", optional=True)
    _field(m, "top_k", 11, "uint32"); _field(m, "json_filter", 12, ".nodereader.JsonFilterExpression", optional=True)
    m = fd.message_type.add(name="RelationPrefixSearchResponse")   # :144-146
    _field(m, "nodes", 1, ".utils.RelationNode", repeated=True)
    m = fd.message_type.add(name="SuggestResponse")           # :468-474
    _field(m, "total", 1, "int32"); _field(m, "results", 2, ".nodereader.ParagraphResult", repeated=True); _field(m, "query", 3, "string")
    _field(m, "ematches", 4, "string", repeated=True)
    _field(m, "entity_results", 6, ".nodereader.RelationPrefixSearchResponse"); _field(m, "shard_ids", 7, "string", repeated=True)
    pool.Add(fd)

    # ---- nodewriter.proto ------------------------------------------------------------------------------------------------
    fd = descriptor_pb2.FileDescriptorProto(name="nidx_protos/nodewriter.proto", package="nodewriter", syntax="proto3")
    e = fd.enum_type.add(name="TypeMessage")                  # :26-29
    e.value.add(name="CREATION", number=0); e.value.add(name="DELETION", number=1)
    m = fd.message_type.add(name="IndexMessage")              # :32-43
    _field(m, "node", 1, "string"); _field(m, "shard", 2, "string"); _field(m, "txid", 3, "uint64"); _field(m, "resource", 4, "string")
    _field(m, "typemessage", 5, "enum:.nodewriter.TypeMessage"); _field(m, "reindex_id", 6, "string"); _field(m, "storage_key", 8, "string")
    _field(m, "kbid", 9, "string")
    m = fd.message_type.add(name="OpStatus")
    _field(m, "detail", 2, "string")
    m = fd.message_type.add(name="VectorIndexConfig")         # :49-54 (similarity: utils.VectorSimilarity COSINE = 0, DOT = 1, utils.proto:96-99)
    _field(m, "similarity", 1, "int32"); _field(m, "normalize_vectors", 2, "bool"); _field(m, "vector_type", 3, "int32")
    _field(m, "vector_dimension", 4, "uint32", optional=True)
    m = fd.message_type.add(name="NewShardRequest")           # :56-71
    _field(m, "kbid", 2, "string")
    _map(m, ".nodewriter.NewShardRequest", "vectorsets_configs", 6, "string", ".nodewriter.VectorIndexConfig")
    pool.Add(fd)
    # noderesources.ShardCreated / ShardId live in noderesources.proto; declared in a side file of the same package
    fd = descriptor_pb2.FileDescriptorProto(name="nidx_protos/noderesources_shards.proto", package="noderesources", syntax="proto3")
    m = fd.message_type.add(name="ShardCreated")              # noderesources.proto:30-34
    _field(m, "id", 1, "string")
    m = fd.message_type.add(name="ShardId")                   # :22-24
    _field(m, "id", 1, "string")
    pool.Add(fd)
    return pool


POOL = _build()


def _cls(name):
    return message_factory.GetMessageClass(POOL.FindMessageTypeByName(name))


SearchRequest = _cls("nodereader.SearchRequest")
SearchResponse = _cls("nodereader.SearchResponse")
FilterExpression = _cls("nodereader.FilterExpression")
Faceted = _cls("nodereader.Faceted")
OrderBy = _cls("nodereader.OrderBy")
IndexMetadata = _cls("noderesources.IndexMetadata")
FacetResult = _cls("nodereader.FacetResult")
FacetResults = _cls("nodereader.FacetResults")
DocumentSearchResponse = _cls("nodereader.DocumentSearchResponse")
ParagraphSearchResponse = _cls("nodereader.ParagraphSearchResponse")
VectorSearchResponse = _cls("nodereader.VectorSearchResponse")
SentenceMetadata = _cls("noderesources.SentenceMetadata")
Resource = _cls("noderesources.Resource")
Security = _cls("utils.Security")
JsonFieldValue = _cls("noderesources.JsonFieldValue")
JsonFilterExpression = _cls("nodereader.JsonFilterExpression")
JsonFieldPathFilter = _cls("nodereader.JsonFieldPathFilter")
GraphQuery = _cls("nodereader.GraphQuery")
GraphSearchRequest = _cls("nodereader.GraphSearchRequest")
GraphSearchResponse = _cls("nodereader.GraphSearchResponse")
SuggestRequest = _cls("nodereader.SuggestRequest")
SuggestResponse = _cls("nodereader.SuggestResponse")
RelationPrefixSearchResponse = _cls("nodereader.RelationPrefixSearchResponse")
SUGGEST_ENTITIES, SUGGEST_PARAGRAPHS = 0, 1   # SuggestFeatures
Relation = _cls("utils.Relation")
RelationNode = _cls("utils.RelationNode")
RelationMetadata = _cls("utils.RelationMetadata")
IndexRelation = _cls("noderesources.IndexRelation")
IndexRelations = _cls("noderesources.IndexRelations")
IndexMessage = _cls("nodewriter.IndexMessage")
NewShardRequest = _cls("nodewriter.NewShardRequest")
ShardCreated = _cls("noderesources.ShardCreated")
NEW_SHARD_METHOD = "/nidx.NidxApi/NewShard"           # nidx.proto:9
FILTER_AND, FILTER_OR = 0, 1
GRAPH_SEARCH_METHOD = "/nidx.NidxSearcher/GraphSearch"   # nidx.proto: rpc GraphSearch
SUGGEST_METHOD = "/nidx.NidxSearcher/Suggest"            # nidx.proto: rpc Suggest
SEARCH_METHOD = "/nidx.NidxSearcher/Search"   # nidx.proto:20-21: package nidx, service NidxSearcher, rpc Search
