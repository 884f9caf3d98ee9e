"""tests/security_model.py against the reference's rules for SearchRequest.security (each case cites them), and the host side of the
device path against the model: the group dictionary and security_nodes' ranges (nucliadb_b200/text.py), the indexing of
Resource.security and the sequence rule in NidxBinding.  No GPU."""
import random
import types

import security_model as M
from nucliadb_b200 import nidx_protos as P
from nucliadb_b200 import text as T


def _doc(groups=(), labels=(), field="/a/title", uuid="r1"):
    return T.TextDoc(uuid, field, "alpha beta", tuple(labels), None, None, tuple(groups))


def test_leading_slash_on_both_sides():
    # resource_indexer.rs:53-57 and search_query.rs:76-80 both put a '/' in front of a group id that lacks one
    assert M.granted(["a"], ["/a"]) and M.granted(["/a"], ["a"]) and M.granted(["a"], ["a"])
    assert T.group_key("a") == T.group_key("/a") == b"a"
    assert T.group_key("a/b") == T.group_key("/a/b") == b"a\0b"


def test_ancestor_grants_at_path_boundaries_only():
    # a facet term matches the facet and its descendants (search_query.rs:81-83 over groups_with_access)
    assert M.granted(["/a/b"], ["/a"]) and M.granted(["/a/b/c"], ["a/b"])
    assert not M.granted(["/ab"], ["/a"]) and not M.granted(["/a"], ["/a/b"])


def test_resource_without_groups_is_public():
    # resource_indexer.rs:60-61: groups_public = 1; search_query.rs:67-71: always in the union
    assert M.granted([], ["/x"]) and M.granted([], [])
    assert M.matches(_doc(), ["/x"])


def test_empty_access_groups_match_public_resources_only():
    # security_query with no groups is the union of groups_public = 1 alone
    assert M.granted([], []) and not M.granted(["/a"], [])


def test_security_and_field_filter_intersect():
    # reader.rs:147-160: BooleanQuery::intersection of the security query and filter_to_query
    f = P.FilterExpression()
    f.facet.facet = "/l/x"
    docs = [_doc(["/g"], ["/l/x"]), _doc(["/g"], ["/l/y"]), _doc(["/h"], ["/l/x"]), _doc([], ["/l/x"])]
    assert [M.matches(d, ["/g"], f) for d in docs] == [True, False, False, True]
    assert [M.matches(d, ["/g"]) for d in docs] == [True, True, False, True]
    assert [M.matches(d, None, f) for d in docs] == [True, False, True, True]


def test_reindex_replaces_groups_under_the_sequence_rule():
    # a re-indexed resource replaces its copies in OLDER segments (deletions apply to lower seqs): the newest groups count
    msgs = [("index", "r1", ["/a"]), ("index", "r2", []), ("index", "r1", ["/b"]), ("delete", "r2")]
    assert M.visible(msgs) == {"r1": ("/b",)}
    # NidxBinding applies the same rule to the documents it keeps (the binding's _alive is the one the searchers open)
    from nucliadb_b200.binding import NidxBinding

    segs = [([_doc(["/a"], uuid="r1")], 1), ([_doc([], uuid="r2")], 2), ([_doc(["/b"], uuid="r1")], 3)]
    deleted = {("r1", 1), ("r2", 2), ("r1", 3), ("r2", 4)}
    kept = NidxBinding._alive(None, segs, deleted)
    assert [(d.uuid, d.groups) for s in kept for d in s] == [("r1", ("/b",))]
    assert not M.granted(kept[0][0].groups, ["/a"]) and M.granted(kept[0][0].groups, ["/b"])


def _nested_groups(rng, n):
    out = set()
    while len(out) < n:
        depth = rng.randint(1, 4)
        out.add("/".join(rng.choice(["a", "ab", "b", "c", "a_", "x"]) + str(rng.randint(0, 3)) for _ in range(depth)))
    return sorted(out)


def test_security_nodes_equal_the_model():
    """TextSearcher.security_nodes compiles OR(PUBLIC, GROUP ranges) over the sorted dictionary; evaluated on each document's ords
    it must equal the model on the document's strings, for random nested groups with and without the leading '/'."""
    rng = random.Random(5)
    groups = _nested_groups(rng, 300)
    docs = []
    for _ in range(2000):
        g = rng.sample(groups, rng.choice([0, 0, 1, 2, 3, 5]))
        docs.append([x if rng.random() < 0.5 else "/" + x for x in g])
    keys = sorted({T.group_key(g) for d in docs for g in d})
    ord_of = {k: i for i, k in enumerate(keys)}
    fake = types.SimpleNamespace(group_keys=keys, _ensure_groups=lambda: None)
    requests = [[], ["/a0"], ["a0"], ["a0/b1"], ["/x3/a1", "c2"], ["/nothere"], ["/a"], [rng.choice(groups) for _ in range(4)]]
    requests += [[g.split("/")[0]] for g in rng.sample(groups, 20)]
    for req in requests:
        flat = T.TextSearcher.security_nodes(fake, req)
        for d in docs:
            ords = sorted({ord_of[T.group_key(g)] for g in d})
            assert M.eval_nodes(flat, ords) == M.granted(d, req), (req, d)


def test_binding_indexes_resource_security():
    """NidxBinding._process puts Resource.security.access_groups on every text and paragraph document of the resource."""
    from nucliadb_b200.binding import NidxBinding, _Shard

    res = P.Resource()
    res.resource.uuid = "r1"
    res.texts["a/title"].text = "alpha beta gamma"
    res.paragraphs["a/title"].paragraphs["r1/a/title/0-5"].end = 5
    res.security.access_groups.extend(["g1", "/g2/x"])
    b = types.SimpleNamespace(_shards={"s": _Shard("kb")}, _load_resource=lambda key: res)
    NidxBinding._process(b, P.IndexMessage(shard="s", storage_key="k"), 1)
    shard = b._shards["s"]
    assert [d.groups for d, _ in [(d, s) for docs, s in shard.text_segments for d in docs]] == [("g1", "/g2/x")]
    assert [d.groups for docs, _ in shard.paragraph_segments for d in docs] == [("g1", "/g2/x")]
    res.ClearField("security")
    NidxBinding._process(b, P.IndexMessage(shard="s", storage_key="k"), 2)
    assert shard.text_segments[-1][0][0].groups == ()
