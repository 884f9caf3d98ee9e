"""Writes graph_knowledge.json: the knowledge graph of the reference's nidx_tests/src/graph.rs (knowledge_graph_as_relations), as
data: entities (value -> subtype), relation labels (label -> RelationType number) and the (source, label, target) triples.
Usage: python make_graph_knowledge.py <reference checkout>"""
import json
import os
import re
import sys

TYPES = {"Child": 0, "About": 1, "Entity": 2, "Colab": 3, "Synonym": 4, "Other": 5}


def main(ref: str):
    src = open(os.path.join(ref, "nidx/nidx_tests/src/graph.rs")).read()
    body = src[src.index("fn knowledge_graph_as_relations"):]
    ent_block = body[body.index("let entities"):body.index("let relations")]
    rel_block = body[body.index("let relations"):body.index("let graph")]
    graph_block = body[body.index("let graph"):body.index("let mut pb_relations")]
    entities = dict(re.findall(r'\("([^"]+)",\s*"([^"]+)"\)', ent_block))
    labels = {k: TYPES[v] for k, v in re.findall(r'\("([^"]+)",\s*RelationType::(\w+)\)', rel_block)}
    triples = re.findall(r'\("([^"]+)",\s*"([^"]+)",\s*"([^"]+)"\)', graph_block)
    out = {"entities": entities, "labels": labels, "triples": [list(t) for t in triples]}
    with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "graph_knowledge.json"), "w") as f:
        json.dump(out, f, indent=1, sort_keys=True)
        f.write("\n")


if __name__ == "__main__":
    main(sys.argv[1] if len(sys.argv) > 1 else "/path/to/reference")
