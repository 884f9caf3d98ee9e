import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100: run with -m gpu)")


def make_vectors(n, d, seed=1234567890, latent=24, noise=0.15):
    """Synthetic embeddings with low intrinsic dimension (like real sentence embeddings): a random
    `latent`-dimensional gaussian pushed through a fixed random linear map plus isotropic noise,
    L2-normalised (the reference's test generator normalises too, segment.rs:682-695)."""
    rng = np.random.default_rng(seed)
    z = rng.standard_normal((n, latent)).astype(np.float32)
    w = np.random.default_rng(99).standard_normal((latent, d)).astype(np.float32)
    v = z @ w + noise * np.sqrt(latent) * rng.standard_normal((n, d)).astype(np.float32)
    v /= np.linalg.norm(v, axis=1, keepdims=True)
    return v.astype(np.float32)


def make_queries(vecs, nq, seed=123, distance=0.05):
    """Queries near data points (segment.rs:880-883: random_nearby_vector(base, 0.05))."""
    rng = np.random.default_rng(seed)
    base = vecs[rng.integers(0, len(vecs), nq)]
    fuzz = rng.uniform(-1, 1, base.shape).astype(np.float32)
    fuzz /= np.linalg.norm(fuzz, axis=1, keepdims=True)
    q = base + distance * fuzz
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return q.astype(np.float32)


@pytest.fixture(scope="session")
def small_data():
    v = make_vectors(20000, 128)
    q = make_queries(v, 64)
    return v, q
