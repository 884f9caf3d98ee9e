"""nucliadb_b200 — H100-native (sm_90a) implementation of NucliaDB's nidx search hot path.

Only what the hot path needs lives here (SURVEY.md §8): the CUDA kernels + C ABI (``csrc/``,
``libnidx_b200.so``) and a host-side mirror of the reference's plug-in interface
(``vector.VectorSearcher`` / ``text.TextSearcher``).  There is no CPU fallback: importing works
anywhere, but every operation needs the built library and a CUDA device and fails loudly otherwise.
"""
from . import _lib  # noqa: F401
from ._lib import NidxError  # noqa: F401

__all__ = ["NidxError"]
