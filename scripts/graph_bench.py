"""Graph search on one GPU: CUDA-event medians and spread of the dictionary pass, the scored pass, the collection (unique max +
top-k) and the whole call (nidx_graph_last_times), for the graph RAG strategy's NODES query (fuzzy WORDS, distance 1, undirected)
and a 3-leaf PATH query, over a seeded synthetic relation index with skewed node popularity.  Prints one JSON line per size and
query, with the bytes per document the scored pass reads and the card's name and power limit.

    python scripts/graph_bench.py --relations 1000000 --reps 20
"""
import argparse
import json
import os
import random
import subprocess
import sys
import threading
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power = [x.strip() for x in out.splitlines()[0].split(",")]
        return name, power
    except Exception:   # noqa: BLE001
        return "unknown", "unknown"


def synthetic(n, seed=11):
    from nucliadb_b200.graph import GraphDoc

    rng = random.Random(seed)
    words = [f"w{i:04d}" for i in range(5000)] + ["anna", "annabel", "climbing", "computer", "science", "new", "york"]
    n_nodes = max(n // 4, 10)
    nodes = [(" ".join(rng.choice(words) for _ in range(rng.randrange(1, 4))), rng.randrange(4), rng.choice(["PERSON", "PLACE", "ORG", ""]))
             for _ in range(n_nodes)]
    ranks = np.minimum((np.random.default_rng(seed).zipf(1.3, size=2 * n) - 1), n_nodes - 1)   # skewed node popularity
    labels = ["IS", "LOVE", "WORK_IN", "BORN_IN", "FOLLOW", "LIVE_IN"]
    return [GraphDoc(f"{i % 100000:032x}", "a/metadata", nodes[ranks[2 * i]], nodes[ranks[2 * i + 1]], rng.randrange(6), rng.choice(labels))
            for i in range(n)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--relations", type=int, nargs="+", default=[1_000_000])
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--k", type=int, default=20)
    a = ap.parse_args()

    def heartbeat():   # building a large synthetic index on the host takes minutes: say it is alive
        while True:
            time.sleep(60)
            print("# building ...", file=sys.stderr, flush=True)

    threading.Thread(target=heartbeat, daemon=True).start()
    from nucliadb_b200 import graph as G
    from nucliadb_b200 import nidx_protos as P

    name, power = card()
    for n in a.relations:
        t0 = time.time()
        ix = G.GraphIndex(synthetic(n))
        print(f"# {n} relations indexed in {time.time() - t0:.0f} s", file=sys.stderr, flush=True)
        nodes_q = P.GraphQuery.PathQuery()
        nodes_q.path.source.value, nodes_q.path.source.fuzzy.kind, nodes_q.path.source.fuzzy.distance = "Anna", 2, 1
        nodes_q.path.undirected = True
        path_q = P.GraphQuery.PathQuery()
        path_q.path.source.value = ix.docs[0].source[0]
        path_q.path.relation.value = "LOVE"
        path_q.path.destination.node_type = 0
        avg_tok = float(np.mean([len(G.tokenize(d.source[0])) + len(G.tokenize(d.target[0])) for d in ix.docs[:10000]]))
        queries = {
            # two programs (source side, destination side), each: the token CSR offset (4 B) and that side's token ords (4 B each),
            # alive 1/8, score 4 and bits 1/8 written; the automaton bitset is small enough to stay in L2
            "nodes_fuzzy_words": ([G.node_query(nodes_q, "src"), G.node_query(nodes_q, "dst")], G.NODES, 2 * (8.25 + 4 * avg_tok / 2)),
            # three ord columns (4 B each) + alive + score + bits
            "path_3_leaves": ([G.path_query(path_q)], G.PATH, 3 * 4 + 4.25),
        }
        for qname, (trees, kind, bytes_per_doc) in queries.items():
            ix.search(trees, kind, a.k)   # warm-up
            times = []
            for _ in range(a.reps):
                hits = ix.search(trees, kind, a.k)
                times.append(ix.last_times())
            t = np.asarray(times)
            med = np.median(t, axis=0)
            row = {"relations": n, "query": qname, "hits": len(hits), "card": name, "power_limit": power,
                   "dict_ms": float(med[0]), "scored_ms": float(med[1]), "collect_ms": float(med[2]), "call_ms": float(med[3]),
                   "call_ms_min": float(t[:, 3].min()), "call_ms_max": float(t[:, 3].max()),
                   "scored_bytes_per_doc": round(bytes_per_doc, 2),
                   "scored_GBps": round(bytes_per_doc * n / (med[1] * 1e-3) / 1e9, 1) if med[1] > 0 else None}
            print(json.dumps(row), flush=True)
        ix.close()


if __name__ == "__main__":
    main()
