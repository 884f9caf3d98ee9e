"""The constants the hot path takes from the reference, as read from the reference's own Rust sources (nidx/nidx_vector/src) into
tests/golden/reference_facts.json by tests/golden/make_reference_facts.py, compared with what the mirror, the oracle and the CUDA
sources use."""
import json
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FACTS = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_facts.json")))["nidx_vector"]


def test_hnsw_parameters():
    """hnsw/params.rs:34-46: M, M_MAX, M_MAX_0, EF_CONSTRUCTION, EF_SEARCH and prune_m = m * 95 / 100 = the mirror's and the library's defaults."""
    from nucliadb_b200 import vector as V

    cfg = V.VectorConfig(dimension=8)
    assert cfg.m == FACTS["M"] == FACTS["M_MAX"]
    assert cfg.m0 == FACTS["M_MAX_0"]
    assert cfg.ef_construction == FACTS["EF_CONSTRUCTION"]
    assert cfg.ef_search == FACTS["EF_SEARCH"]
    num, den = FACTS["prune_m"]
    assert f"mmax * {num} / {den}" in open(os.path.join(ROOT, "nucliadb_b200", "csrc", "hnsw_build.cuh")).read()
    header = open(os.path.join(ROOT, "include", "nidx_b200.h")).read()
    for field, want in (("m;", 30), ("m0;", 60), ("ef_construction;", 100), ("ef_search;", 30)):
        assert re.search(rf"int32_t {re.escape(field)}[^\n]*0 => {want} \*/", header), field


def test_rabitq_constants():
    """vector_types/rabitq.rs:30-36: EPSILON, RERANKING_FACTOR, RERANKING_LIMIT in the kernels, the host code and the oracle."""
    eps, fac, lim = FACTS["EPSILON"], FACTS["RERANKING_FACTOR"], FACTS["RERANKING_LIMIT"]
    cu = open(os.path.join(ROOT, "nucliadb_b200", "csrc", "rabitq.cuh")).read()
    assert float(re.search(r"RABITQ_EPSILON = ([0-9.]+)f", cu).group(1)) == eps
    assert float(re.search(r"RABITQ_EPSILON = ([0-9.]+)f", open(os.path.join(ROOT, "oracle", "rabitq.hpp")).read()).group(1)) == eps
    api = open(os.path.join(ROOT, "nucliadb_b200", "csrc", "api.cu")).read()
    m = re.search(r"last_k = \(int\)std::min<size_t>\(\(size_t\)k \* (\d+), (\d+)\)", api)
    assert (float(m.group(1)), float(m.group(2))) == (fac, lim)
    assert float(re.search(r"const size_t RERANKING_FACTOR = (\d+);", api).group(1)) == fac


def test_cost_model_matches_the_reference_source():
    """segment.rs:626-660 use_hnsw: the constants of the reference's function body (16, * 3 / 4, / 2, ln - 2.0) appear in api.cu's
    use_hnsw_cost, and the function agrees with a literal Python transcription of the Rust on a grid."""
    import math

    import oracle as O

    uh = FACTS["use_hnsw"]
    assert uh == {"full_cost": 16, "search_mult": [3, 4], "rerank_div": 2, "ln_offset": 2.0, "power": 2}

    def f32(x):
        import numpy as np

        return np.float32(x)

    def ref(total, matching, k, rq, M=30):
        full, smul, rmul = (16, 100 * 3 // 4, 100 // 2) if rq else (1, 1, 0)
        import numpy as np

        hnsw_rq = (np.log(f32(total)) - f32(2.0)) ** 2 * np.log(f32(k)) * f32(smul)
        hnsw_full = k * rmul + k * M * total // matching
        hnsw_cost = (int(hnsw_rq) if hnsw_rq > 0 else 0) + hnsw_full * full
        return hnsw_cost < matching + k * rmul * full

    for total in (100, 10_000, 200_000, 10_000_000):
        for frac in (1.0, 0.3, 0.01, 0.0001):
            matching = max(1, int(total * frac))
            for k in (1, 10, 100):
                for rq in (False, True):
                    assert bool(O.use_hnsw(total, matching, k, has_rabitq=rq, M=30)) == bool(ref(total, matching, k, rq)), (total, matching, k, rq)
    assert math.isfinite(1.0)


def test_segment_file_names():
    """The v2 segment directory's file names (hnsw/disk/v2.rs:64-65, data_store/v2/*.rs): what the library and the mirror read and write."""
    want = {"hnsw.graph": ("hnsw/disk/v2.rs", "GRAPH_FILENAME"), "hnsw.edges": ("hnsw/disk/v2.rs", "EDGES_FILENAME"),
            "vectors.bin": ("data_store/v2/vector_store.rs", "FILENAME"), "vectors.quant": ("data_store/v2/quant_vector_store.rs", "FILENAME"),
            "paragraphs.bin": ("data_store/v2/paragraph_store.rs", "FILENAME_DATA"), "paragraphs.pos": ("data_store/v2/paragraph_store.rs", "FILENAME_POS")}
    ours = open(os.path.join(ROOT, "nucliadb_b200", "csrc", "segment_io.hpp")).read() + open(os.path.join(ROOT, "nucliadb_b200", "csrc", "api.cu")).read() + \
        open(os.path.join(ROOT, "nucliadb_b200", "paragraph_store.py")).read() + open(os.path.join(ROOT, "nucliadb_b200", "vector.py")).read()
    for name, (path, const) in want.items():
        assert FACTS["file_names"][f"{path}:{const}"] == name, (path, const)
        assert f'"/{name}"' in ours or f'"{name}"' in ours, name
