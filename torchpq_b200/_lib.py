"""ctypes binding of ``libtpq_b200.so`` (the C ABI declared in ``include/tpq_b200.h``).

The reference launches its kernels with bare ``tensor.data_ptr()`` integers through
CuPy (torchpq/kernels/CustomKernel.py:13-42); this is the same calling style against
an ahead-of-time compiled sm_90a library.  There is no fallback: if the library is
missing or was not built, importing this module raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# TPQ_B200_LIB: load another build of the same ABI (scripts/ use it for the -DTPQ_DEBUG_KNOBS experiment build)
LIB_PATH = os.environ.get("TPQ_B200_LIB") or os.path.join(_HERE, "libtpq_b200.so")

TPQ_OK = 0
TPQ_ERR_BAD_ARG = -1
TPQ_ERR_UNSUPPORTED = -2
TPQ_ERR_WORKSPACE = -3
TPQ_ERR_CUDA = -4

METRIC = {"euclidean": 0, "cosine": 1, "manhattan": 2, "inner": 3}   # manhattan: k-means assignment only; inner: flat search only


class TpqIndex(C.Structure):
    """struct tpq_index (include/tpq_b200.h)."""
    _fields_ = [
        ("d_vector", C.c_int32), ("n_subvectors", C.c_int32), ("n_cells", C.c_int32), ("metric", C.c_int32),
        ("capacity", C.c_int64),
        ("vq_codebook", C.c_void_p), ("pq_codebook", C.c_void_p), ("storage", C.c_void_p),
        ("is_empty", C.c_void_p), ("cell_start", C.c_void_p), ("cell_size", C.c_void_p),
        ("address2id", C.c_void_p),
        ("m_pad", C.c_int32), ("shard_rank", C.c_int32), ("shard_world", C.c_int32), ("mean_cell_live", C.c_int32),
        ("n_blocks", C.c_int64),
        ("codes_scan", C.c_void_p), ("block_valid", C.c_void_p), ("cell_block_start", C.c_void_p),
        ("pq_codebook_t", C.c_void_p), ("pq_norm_t", C.c_void_p),
        ("part2_scan", C.c_void_p), ("residual", C.c_int32), ("code_size", C.c_int32),
    ]


# name -> (restype, argtypes); every symbol include/tpq_b200.h declares
_P, _I, _I64, _F, _SZ = C.c_void_p, C.c_int, C.c_int64, C.c_float, C.c_size_t
_IX = C.POINTER(TpqIndex)
SIGNATURES = {
    "tpq_version": (_I, []),
    "tpq_last_error": (C.c_char_p, []),
    "tpq_device_supported": (_I, [_I]),
    "tpq_normalize_columns": (_I, [_P, _I, _I, _P, _P]),
    "tpq_coarse_workspace_bytes": (_SZ, [_I, _I, _I]),
    "tpq_coarse_probe": (_I, [_P, _P, _I, _I, _I, _I, _I, _F, _P, _P, _P, _P, _SZ, _P]),
    "tpq_build_lut": (_I, [_P, _P, _I, _I, _I, _I, _P, _P]),
    "tpq_ivfpq_topk_workspace_bytes": (_SZ, [_I, _I]),
    "tpq_ivfpq_topk": (_I, [_P, _P, _P, _P, _P, _P, _I64, _I, _I, _I, _I, _P, _P, _P, _SZ, _P]),
    "tpq_relayout_plan": (_I, [_P, _I, _I, _I, _P, _P]),
    "tpq_codes_scan_bytes": (_SZ, [_I, _I64]),
    "tpq_relayout_codes": (_I, [_IX, _P, _P, _P]),
    "tpq_relayout_codebook": (_I, [_P, _I, _I, _I, _P, _P, _P]),
    "tpq_search_workspace_bytes": (_SZ, [_IX, _I, _I, _I]),
    "tpq_ivfpq_search": (_I, [_IX, _P, _I, _I, _I, _I, _F, _P, _P, _P, _P, _P, _SZ, _P]),
    "tpq_ivfpq_search_cells": (_I, [_IX, _P, _P, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "tpq_part2_scan_bytes": (_SZ, [_I, _I]),
    "tpq_relayout_part2": (_I, [_P, _P, _I, _I, _I, _P, _P]),
    "tpq_max_sim": (_I, [_P, _P, _I, _I, _I64, _I, _I, _I, _P, _P, _P]),
    "tpq_kmeans_assign_workspace_bytes": (_SZ, [_I, _I, _I]),
    "tpq_kmeans_assign": (_I, [_P, _P, _I, _I, _I64, _I, _I, _I, _P, _P, _P, _SZ, _P]),
    "tpq_compute_centroids_workspace_bytes": (_SZ, [_I, _I]),
    "tpq_compute_centroids": (_I, [_P, _P, _I, _I, _I64, _I, _P, _P, _SZ, _P]),
    "tpq_pq_decode": (_I, [_P, _P, _I, _I, _I64, _P, _P]),
    "tpq_profile_enable": (_I, [_I]),
    "tpq_profile_scan_ms": (_I, [C.POINTER(C.c_float), C.POINTER(C.c_int)]),
    "tpq_merge_topk": (_I, [_P, _I, _I, _I, _P, _I64, _P, _P, _P, _P]),
    "tpq_ivfpq_scan_push": (_I, [_IX, _P, _P, _P, _P, _I, _I, _I, _I, _F, _P, _I, _I, _P, _SZ, _P]),
    "tpq_ioa_workspace_bytes": (_SZ, [_I64, _I]),
    "tpq_get_ioa": (_I, [_P, _I64, _I, _P, _P, _P, _SZ, _P]),
    "tpq_empty_prefix_workspace_bytes": (_SZ, [_I64]),
    "tpq_empty_prefix": (_I, [_P, _I64, _P, _P, _SZ, _P]),
    "tpq_get_write_address": (_I, [_P, _P, _I64, _P, _P, _P, _I, _P, _P, _P]),
    "tpq_store_codes": (_I, [_P, _P, _P, _P, _I64, _IX, _P, _P, _P, _P, _P, _P, _P]),
    "tpq_expand_move": (_I, [_P, _P, _P, _P, _P, _I, _I, _I64, _I64, _P, _P, _P, _P]),
    "tpq_flat_norms": (_I, [_P, _I64, _I, _I64, _I, _P, _P]),
    "tpq_flat_workspace_bytes": (_SZ, [_I, _I, _I64, _I]),
    "tpq_flat_search": (_I, [_P, _I, _I, _P, _I64, _I64, _P, _I, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "tpq_rerank_workspace_bytes": (_SZ, [_I, _I, _I]),
    "tpq_rerank": (_I, [_P, _I, _I, _P, _I, _P, _I64, _I, _I, _P, _P, _I, _I, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "tpq_refine_flat_workspace_bytes": (_SZ, [_I, _I, _I]),
    "tpq_refine_flat": (_I, [_P, _I, _I, _P, _I, _P, _I64, _I, _I, _P, _P, _P, _P, _P, _SZ, _P]),
    "tpq_topk_workspace_bytes": (_SZ, [_I64, _I64, _I, _I]),
    "tpq_topk": (_I, [_P, _I64, _I64, _I, _I, _P, _P, _P, _SZ, _P]),
    "tpq_ivfflat_workspace_bytes": (_SZ, [_I, _I, _I, _I, _I]),
    "tpq_ivfflat_search": (_I, [_P, _I, _I, _P, _I, _P, _I64, _P, _P, _P, _P, _I, _P, _P, _I, _I, _F, _I, _P, _P, _P,
                                _P, _P, _SZ, _P]),
    "tpq_sq_encode": (_I, [_P, _I, _I64, _I, _P, _P, _P, _P]),
    "tpq_sq_decode": (_I, [_P, _I, _I64, _I, _P, _P, _P, _P]),
    "tpq_ivfsq_search": (_I, [_P, _I, _I, _P, _I, _P, _I, _P, _P, _I64, _P, _P, _P, _P, _I, _P, _P, _I, _I, _F, _I,
                              _P, _P, _P, _P, _P, _SZ, _P]),
    "tpq_flat_range_workspace_bytes": (_SZ, [_I, _I, _I64]),
    "tpq_flat_range_search": (_I, [_P, _I, _I, _P, _I64, _I64, _P, _I, _F, _P, _P, _I64, _P, _P, _SZ, _P]),
    "tpq_ivfflat_range_workspace_bytes": (_SZ, [_I, _I, _I, _I]),
    "tpq_ivfflat_range_search": (_I, [_P, _I, _I, _P, _I, _P, _I64, _P, _P, _P, _P, _I, _P, _P, _I, _I, _F, _F, _P,
                                      _P, _I64, _P, _P, _SZ, _P]),
    "tpq_ivfsq_range_search": (_I, [_P, _I, _I, _P, _I, _P, _I, _P, _P, _I64, _P, _P, _P, _P, _I, _P, _P, _I, _I, _F,
                                    _F, _P, _P, _I64, _P, _P, _SZ, _P]),
    "tpq_ivfpq4_workspace_bytes": (_SZ, [_I, _I, _I, _I, _I]),
    "tpq_ivfpq4_search": (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _I64, _I, _P, _P, _P, _P, _P, _P, _I, _I, _F,
                               _I, _P, _P, _P, _P, _SZ, _P]),
    "tpq_ivfpq_range_workspace_bytes": (_SZ, [_IX, _I, _I]),
    "tpq_ivfpq_range_search": (_I, [_IX, _P, _P, _P, _P, _I, _I, _I, _F, _F, _P, _P, _I64, _P, _P, _SZ, _P]),
}

DTYPE_F32, DTYPE_F16 = 0, 1     # TPQ_DTYPE_* (include/tpq_b200.h)


def _load():
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} not found: the CUDA extension has not been built "
            "(run `python -c 'import __graft_entry__ as g; g.build()'` or `make -C torchpq_b200/csrc`). "
            "torchpq_b200 has no CPU or PyTorch fallback.")
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)           # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    return lib


lib = _load()


def last_error() -> str:
    return lib.tpq_last_error().decode("utf-8", "replace")


def check(rc: int) -> None:
    """0 -> ok; bad arguments re-raise as AssertionError (the reference's preconditions are Python
    asserts, e.g. IVFPQTopkCuda.py:98-114, IVFPQIndex.py:471-473); everything else RuntimeError."""
    if rc == TPQ_OK:
        return
    msg = last_error()
    if rc == TPQ_ERR_BAD_ARG:
        raise AssertionError(msg)
    if rc == TPQ_ERR_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise RuntimeError(f"tpq_b200 error {rc}: {msg}")


def ptr(t) -> C.c_void_p:
    """Device pointer of a tensor (None -> NULL)."""
    return C.c_void_p(0 if t is None else t.data_ptr())


def current_stream(device) -> C.c_void_p:
    import torch
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)
