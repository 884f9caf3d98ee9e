"""``NidxSearcher.Suggest``: the plan of a request, the answer of one shard and the merge of several.

Reference:
  src/searcher/query_planner/suggest.rs            SuggestPlan::build, split_suggest_query (MAX_SUGGEST_COMPOUND_WORDS = 3)
  src/searcher/shard_suggest.rs:94-161             one shard: prefilter, paragraphs, entities
  src/searcher/query_planner/prefilter.rs:105-133  Prefilter::parse_suggest
  nidx_paragraph/src/reader.rs:58-90               keyword pass, then the fuzzy pass when it found nothing; results_per_page = 10
  nidx_paragraph/src/search_query.rs:87-183        Must(query) AND Must(repeated_in_field == 0) AND Must(op(paragraph_filter, prefilter))
  nidx_paragraph/src/query_parser/fuzzy_parser.rs  clause kinds: MIN_FUZZY_LEN = 3, MIN_FUZZY_PREFIX_LEN = 4 bytes, distance 1
  nidx_paragraph/src/search_response.rs:218-310    ParagraphResult (labels under /l, matches = sorted expanded terms)
  nidx_relation/src/lib.rs:216-261                 entities: the groups as fuzzy prefix ENTITY nodes, one NODES search
  src/searcher/shard_merge.rs:101-151              merge across shards

Chosen here (DESIGN 10 lists them with the reasons):
  * filters and repeated_in_field only filter; the keyword pass scores the body's BM25 as the paragraph search does, the fuzzy pass
    0.5 * (1.0 per fuzzy clause + BM25 per exact term at tf = 1 + BM25 per phrase at its frequency);
  * security is never widened: the mask is AND(security, op(paragraph_filter, prefilter));
  * json_filter does not apply to entities; stop words are not removed; excluded words are searched as exact terms;
  * a body without a clause answers no paragraph; top_k above 1024, a fuzzy pass of more than 64 clauses and fuzzy literals of more
    than 4096 code points in all are ValueErrors (INVALID_ARGUMENT);
  * ties: score descending, then segment, then document; ematches in first-occurrence order; entity nodes by score, then node key.
"""
from __future__ import annotations

from dataclasses import dataclass, field

from . import nidx_protos as P

MAX_SUGGEST_COMPOUND_WORDS = 3   # suggest.rs
MIN_SUGGEST_PREFIX_LENGTH = 2    # nidx_relation/src/lib.rs: groups of fewer bytes are dropped
MIN_FUZZY_LEN = 3                # fuzzy_parser.rs: literals of fewer bytes are exact terms
MIN_FUZZY_PREFIX_LEN = 4         # the last literal of at least this many bytes is a fuzzy prefix term
FUZZY_DISTANCE = 1
RESULTS_PER_PAGE = 10            # nidx_paragraph/src/reader.rs:78-89
MAX_TOP_K = 1024
MAX_CLAUSES = 64                 # clauses of one fuzzy pass (NIDX_SG_MAX_CLAUSES)
MAX_FUZZY_CODE_POINTS = 4096     # code points of the fuzzy literals of one body (graph_dict_match_kernel's shared memory)

FUZZY, FUZZY_PREFIX, TERM, PHRASE = "fuzzy", "fuzzy_prefix", "term", "phrase"


def split_suggest_query(query: str, max_group: int = MAX_SUGGEST_COMPOUND_WORDS) -> list:
    """suggest.rs split_suggest_query: the last max_group words (split on ' ' exactly), longest group first; always max_group
    entries (empty strings when the body has fewer words)."""
    words = query.split(" ")[::-1][:max_group][::-1]
    prefixes = [""] * max_group
    for index, word in enumerate(words):
        for i in range(index + 1):
            prefixes[i] = (prefixes[i] + " " + word) if prefixes[i] else word
    return prefixes


def entity_groups(body: str) -> list:
    """The groups that become entity nodes: split_suggest_query's, those shorter than MIN_SUGGEST_PREFIX_LENGTH bytes dropped."""
    return [g for g in split_suggest_query(body) if len(g.encode("utf-8")) >= MIN_SUGGEST_PREFIX_LENGTH]


def fuzzy_clauses(tokens: list) -> list:
    """paragraph_query_tokens' tokens -> the fuzzy pass's clauses [(kind, value)] in token order (fuzzy_parser.rs): a literal of fewer
    than MIN_FUZZY_LEN bytes is a TERM, the last literal of at least MIN_FUZZY_PREFIX_LEN bytes a FUZZY_PREFIX, any other literal a
    FUZZY; a quoted group of two or more words a PHRASE (its words), of one word a TERM; an excluded word a TERM."""
    last = max((i for i, (k, _) in enumerate(tokens) if k == "L"), default=None)
    out = []
    for i, (kind, text) in enumerate(tokens):
        n = len(text.encode("utf-8"))
        if kind == "L":
            if n < MIN_FUZZY_LEN:
                out.append((TERM, text))
            elif i == last and n >= MIN_FUZZY_PREFIX_LEN:
                out.append((FUZZY_PREFIX, text))
            else:
                out.append((FUZZY, text))
        elif kind == "Q":
            words = text.split(" ")
            out.append((PHRASE, words) if len(words) >= 2 else (TERM, words[0]))
        else:
            out.append((TERM, text))
    return out


def ematches(tokens: list) -> list:
    """The literal and quoted token values, distinct, in first-occurrence order (the reference collects them in a HashSet)."""
    out = []
    for kind, text in tokens:
        if kind in ("L", "Q") and text not in out:
            out.append(text)
    return out


def extract_labels(labels) -> list:
    """search_response.rs extract_labels: the facets under /l."""
    return [label for label in labels if label == "/l" or label.startswith("/l/")]


@dataclass
class ParagraphHit:
    """One result of ParagraphSearcher.suggest."""
    score: float
    segment: int
    doc: int
    matches: list = field(default_factory=list)


@dataclass
class ParagraphSuggest:
    hits: list          # [ParagraphHit] best first, at most top_k
    fuzzy: bool         # the hits come from the fuzzy pass
    ematches: list


def entity_request(body: str, top_k: int):
    """nidx_relation suggest: OR of one undirected fuzzy-prefix ENTITY source node per group, as a NODES GraphSearchRequest; None
    without a group."""
    groups = entity_groups(body)
    if not groups:
        return None
    req = P.GraphSearchRequest(kind=P.GraphSearchRequest.NODES, top_k=top_k)
    ops = req.query.path.bool_or.operands
    for g in groups:
        p = ops.add().path
        p.source.value = g
        p.source.node_type = P.RelationNode.ENTITY
        p.source.fuzzy.kind = 1   # MatchLocation.PREFIX (nodereader.proto GraphQuery.Node.MatchLocation)
        p.source.fuzzy.distance = FUZZY_DISTANCE
        p.undirected = True
    return req


def merge_suggest(parts: list, top_k: int):
    """shard_merge.rs:101-151 over [(shard id, SuggestResponse)] in request order: shard ids concatenated, query from the last shard,
    totals summed, ematches united (first occurrence first), results merged by (bm25 desc, shard id bytes desc, docaddr asc) and cut to
    top_k, entity nodes united (first occurrence first) and absent when no shard found one.  One shard's answer is returned as it is
    (SuggestOp::merge, grpc.rs:514-520): its entity_results stay present when empty."""
    from .shard_merge import bm25_order_key

    if len(parts) == 1:
        return parts[0][1]
    out = P.SuggestResponse()
    rows, nodes, seen = [], [], set()
    for sid, r in parts:
        out.shard_ids.extend(r.shard_ids or [sid])
        out.query = r.query
        out.total += r.total
        for e in r.ematches:
            if e not in out.ematches:
                out.ematches.append(e)
        rows += [(bm25_order_key(x.score.bm25, sid.encode(), x.score.docaddr), sid, x) for x in r.results]
        if r.HasField("entity_results"):
            for n in r.entity_results.nodes:
                key = (n.value, n.ntype, n.subtype)
                if key not in seen:
                    seen.add(key)
                    nodes.append(n)
    rows.sort(key=lambda t: t[0])
    for _, sid, x in rows[:top_k]:
        o = out.results.add()
        o.CopyFrom(x)
        o.shard_id = sid.encode()
    if nodes:
        out.entity_results.nodes.extend(nodes)
    return out
