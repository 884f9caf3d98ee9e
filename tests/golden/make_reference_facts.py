"""Extracts the facts the CPU tests compare against from a checkout of the reference (nucliadb) and stores them as
tests/golden/reference_facts.json (committed), so that the tests need no copy of the reference:
  * nidx_vector constants: HNSW parameters, prune_m, the RaBitQ constants, the constants of segment.rs's use_hnsw,
    the v2 segment file names (test_constants_vs_reference.py);
  * every message / enum field of nidx_protos/*.proto (number, type, cardinality) and the rpc signatures of nidx.proto
    (test_protos_vs_reference.py);
  * the parameter names of nidx_binding.pyi's NidxBinding methods and its attributes (test_host_logic.py).

    python tests/golden/make_reference_facts.py <path of a nucliadb checkout>
"""
import ast
import json
import os
import re
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def rust_const(path, name):
    m = re.search(rf"const\s+{name}\s*:\s*\w+\s*=\s*([0-9.]+)\s*;", open(path).read())
    assert m, (path, name)
    return float(m.group(1))


def rust_str_const(path, name):
    m = re.search(rf'const\s+{name}\s*:\s*&str\s*=\s*"([^"]+)"', open(path).read())
    assert m, (path, name)
    return m.group(1)


def parse_proto(path):
    """-> ({full message name: {field: (number, type, repeated)}}, {full enum name: {value name: number}}); handles nesting, oneof, map<>."""
    text = re.sub(r"//[^\n]*", "", open(path).read())
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    pkg = re.search(r"\bpackage\s+([\w.]+)\s*;", text).group(1)
    tokens = re.findall(r"[{};=<>,]|[\w.]+|\"[^\"]*\"|\[[^\]]*\]", text)
    msgs, enums = {}, {}
    stack = []          # [(kind, name)]
    i = 0
    while i < len(tokens):
        t = tokens[i]
        if t in ("message", "enum", "oneof", "service") and tokens[i + 2] == "{":
            name = tokens[i + 1]
            if t == "oneof":
                stack.append(("oneof", None))
            else:
                scope = ".".join([pkg] + [n for k, n in stack if k == "message"] + [name])
                stack.append((t, name))
                if t == "message":
                    msgs[scope] = {}
                elif t == "enum":
                    enums[scope] = {}
            i += 3
            continue
        if t == ";":
            i += 1
            continue
        if t == "{":                 # any other block (rpc bodies, option blocks)
            stack.append(("block", None))
            i += 1
            continue
        if t == "}":
            stack.pop()
            i += 1
            continue
        kinds = [k for k, _ in stack]
        if kinds and kinds[-1] == "enum" and i + 2 < len(tokens) and tokens[i + 1] == "=":
            scope = ".".join([pkg] + [n for k, n in stack if k in ("message", "enum")])
            enums[scope][t] = int(tokens[i + 2])
            i += 3
            continue
        if kinds and kinds[-1] in ("message", "oneof") and t not in ("option", "reserved", "extensions"):
            scope = ".".join([pkg] + [n for k, n in stack if k == "message"])
            rep = False
            j = i
            if tokens[j] in ("repeated", "optional"):
                rep = tokens[j] == "repeated"
                j += 1
            if tokens[j] == "map" and tokens[j + 1] == "<":
                ktype, vtype, name, num = tokens[j + 2], tokens[j + 4], tokens[j + 6], int(tokens[j + 8])
                msgs[scope][name] = (num, f"map<{ktype},{vtype}>", True)
                i = j + 9
            elif j + 3 < len(tokens) and tokens[j + 2] == "=":
                msgs[scope][tokens[j + 1]] = (int(tokens[j + 3]), tokens[j], rep)
                i = j + 4
            else:
                i += 1
                continue
            while i < len(tokens) and tokens[i] != ";" and tokens[i] not in ("}", "{"):
                i += 1
            continue
        i += 1
    return msgs, enums


def vector_facts(src):
    params = os.path.join(src, "hnsw", "params.rs")
    rabitq = os.path.join(src, "vector_types", "rabitq.rs")
    facts = {name: rust_const(params, name) for name in ("M", "M_MAX", "M_MAX_0", "EF_CONSTRUCTION", "EF_SEARCH")}
    m = re.search(r"fn prune_m\(m: usize\) -> usize \{\s*m \* (\d+) / (\d+)", open(params).read())
    facts["prune_m"] = [int(m.group(1)), int(m.group(2))]
    facts.update({name: rust_const(rabitq, name) for name in ("EPSILON", "RERANKING_FACTOR", "RERANKING_LIMIT")})
    seg = open(os.path.join(src, "segment.rs")).read()
    body = seg[seg.index("fn use_hnsw("):]
    body = body[: body.index("\n}\n")]
    full = re.search(r"if has_rabitq \{\s*full_cost = (\d+);\s*search_mult = rabitq::RERANKING_FACTOR \* (\d+) / (\d+);\s*"
                     r"rerank_mult = rabitq::RERANKING_FACTOR / (\d+);", body)
    ln = re.search(r"\(total_nodes as f32\)\.ln\(\) - ([0-9.]+)\)\.powi\((\d+)\)", body)
    facts["use_hnsw"] = {"full_cost": int(full.group(1)), "search_mult": [int(full.group(2)), int(full.group(3))], "rerank_div": int(full.group(4)),
                         "ln_offset": float(ln.group(1)), "power": int(ln.group(2))}
    names = {"GRAPH_FILENAME": "hnsw/disk/v2.rs", "EDGES_FILENAME": "hnsw/disk/v2.rs", "FILENAME": "data_store/v2/vector_store.rs",
             "FILENAME_QUANT": ("data_store/v2/quant_vector_store.rs", "FILENAME"), "FILENAME_DATA": "data_store/v2/paragraph_store.rs",
             "FILENAME_POS": "data_store/v2/paragraph_store.rs"}
    files = {}
    for key, where in names.items():
        path, const = (where if isinstance(where, tuple) else (where, key))
        files[f"{path}:{const}"] = rust_str_const(os.path.join(src, path), const)
    facts["file_names"] = files
    return facts


def proto_facts(src):
    msgs, enums = {}, {}
    for f in sorted(os.listdir(src)):
        if f.endswith(".proto"):
            m, e = parse_proto(os.path.join(src, f))
            msgs.update(m)
            enums.update(e)
    nidx = open(os.path.join(src, "nidx.proto")).read()
    rpcs = {}
    parts = re.split(r"\bservice\s+(\w+)\s*\{", nidx)   # [before, name, body..., name, body...]
    for service, body in zip(parts[1::2], parts[2::2]):
        for name, req, resp in re.findall(r"rpc\s+(\w+)\s*\(\s*([\w.]+)\s*\)\s*returns\s*\(\s*(?:stream\s+)?([\w.]+)\s*\)", body):
            rpcs[f"{service}.{name}"] = [req, resp]
    return {"messages": msgs, "enums": enums, "rpcs": rpcs}


def binding_facts(pyi):
    cls = next(n for n in ast.parse(open(pyi).read()).body if isinstance(n, ast.ClassDef) and n.name == "NidxBinding")
    methods = {n.name: [a.arg for a in n.args.args] for n in cls.body if isinstance(n, ast.FunctionDef)}
    attrs = [n.target.id for n in cls.body if isinstance(n, ast.AnnAssign)]
    return {"methods": methods, "attributes": attrs}


def main():
    ref = sys.argv[1]
    nidx = os.path.join(ref, "nidx")
    facts = {"nidx_vector": vector_facts(os.path.join(nidx, "nidx_vector", "src")),
             "nidx_protos": proto_facts(os.path.join(nidx, "nidx_protos")),
             "nidx_binding": binding_facts(os.path.join(nidx, "nidx_binding", "nidx_binding.pyi"))}
    with open(os.path.join(HERE, "reference_facts.json"), "w") as f:
        json.dump(facts, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main()
