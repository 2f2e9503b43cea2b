"""Drop the H100 search path into an existing ``torchpq.index.IVFPQIndex`` *object*.

``patch(index)`` rebinds ``search`` / ``search_cells`` (and adds ``layout`` / ``set_shard``) on an instance of the
reference class -- trained and populated by the reference, or restored with ``load_state_dict`` -- so that
``index.search(x, k)`` (reference signature, torchpq/index/IVFPQIndex.py:469) runs the sm_90a library instead of
the CuPy kernels.  Only attributes the reference object already has are read: ``_storage``, ``_is_empty``,
``_cell_start``, ``_cell_size``, ``_address2id``, ``vq_codec`` / ``pq_codec`` (``.codebook``, ``.is_trained``),
``d_vector``, ``n_subvectors``, ``n_cells``, ``distance``, ``n_probe``, ``use_smart_probing``,
``smart_probing_temperature``, ``pq_use_residual``, ``device``.  ``unpatch(index)`` restores the class methods.
"""
from __future__ import annotations

import types

from .index import IVFPQIndex as _Mine

_METHODS = ("layout", "set_shard", "_check_query", "_search", "search", "search_cells")


def patch(index):
    for name in ("d_vector", "n_subvectors", "n_cells", "distance", "_storage", "_is_empty", "_cell_start",
                 "_cell_size", "_address2id", "vq_codec", "pq_codec"):
        assert hasattr(index, name), f"not an IVFPQIndex-shaped object: missing {name!r}"
    assert index.distance in ("euclidean", "cosine"), "only euclidean and cosine indexes can be searched"
    if hasattr(index, "n_subvectors_rerank"):
        raise NotImplementedError("patch() takes IVFPQIndex objects; an IVFPQRIndex needs its re-rank pass: "
                                  "load its state_dict into torchpq_b200.IVFPQRIndex instead")
    d = index.__dict__
    d["_layout"] = None
    d["_shard"] = (0, 1)
    if not hasattr(index, "pq_use_residual"):
        d["pq_use_residual"] = False
    for name in _METHODS:
        d[name] = types.MethodType(getattr(_Mine, name), index)     # instance attribute shadows the class method
    return index


def unpatch(index):
    for name in _METHODS + ("_layout", "_shard"):
        index.__dict__.pop(name, None)
    return index
