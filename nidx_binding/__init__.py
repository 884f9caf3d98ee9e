"""``nidx_binding``: the module name and class the reference's Python side imports (nucliadb/src/nucliadb/common/nidx.py:106-146
``from nidx_binding import NidxBinding``), served by the GPU searchers of ``nucliadb_b200`` (see nucliadb_b200/binding.py)."""
from nucliadb_b200.binding import NidxBinding  # noqa: F401

__all__ = ["NidxBinding"]
