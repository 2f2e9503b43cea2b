"""Operator-level mirrors of the reference's fused ops (same names, argument meaning and checks).

    IVFPQTopk.topk       torchpq/fn/IVFPQTopk.py:54-104 -> kernels/IVFPQTopkCuda.py:81-142
    precompute_adc       torchpq/codec/PQCodec.py:62-75
    coarse_probe         torchpq/metric.py:74-94 + fn/Topk.py:43-67 + index/IVFPQIndex.py:499-512
    normalize            torchpq/util.py:38-43
    Topk                 torchpq/fn/Topk.py:43-67 -> kernels/cuda/top1_select.cu, top32_select.cu, topk_select.cu
Each is one call into the sm_90a library; tensors are passed as raw device pointers.
"""
from __future__ import annotations

import torch

from . import _lib
from ._lib import lib, check, ptr
from .modules import on_data_device, on_device


def _cuda_f32(t, name):
    assert t.device.type == "cuda", f"{name} must be a CUDA tensor (torchpq_b200 has no CPU path)"
    assert t.dtype == torch.float32, f"{name} must be float32"
    return t.contiguous()


@on_data_device
def normalize(x, dim=0):
    """util.normalize for a [d, n] matrix along dim 0: x / (||x|| + 1e-9)."""
    assert dim == 0 and x.dim() == 2
    x = _cuda_f32(x, "x")
    out = torch.empty_like(x)
    check(lib.tpq_normalize_columns(ptr(x), x.shape[0], x.shape[1], ptr(out), _lib.current_stream(x.device)))
    return out


@on_data_device
def coarse_probe(x, vq_codebook, n_probe, use_smart_probing=True, smart_probing_temperature=30.0):
    """x [d, nq], vq_codebook [d, n_cells] -> (topk_sims [nq, n_probe] desc, cells [nq, n_probe] i64,
    n_probe_list [nq] i64)."""
    x, cb = _cuda_f32(x, "x"), _cuda_f32(vq_codebook, "vq_codebook")
    d, nq = x.shape
    assert cb.shape[0] == d
    n_cells = cb.shape[1]
    dev = x.device
    sims = torch.empty(nq, n_probe, dtype=torch.float32, device=dev)
    cells = torch.empty(nq, n_probe, dtype=torch.long, device=dev)
    npl = torch.empty(nq, dtype=torch.long, device=dev)
    ws_bytes = lib.tpq_coarse_workspace_bytes(d, nq, n_cells)
    ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
    check(lib.tpq_coarse_probe(ptr(x), ptr(cb), d, nq, n_cells, int(n_probe), int(bool(use_smart_probing)),
                               float(smart_probing_temperature), ptr(sims), ptr(cells), ptr(npl),
                               ptr(ws), ws_bytes, _lib.current_stream(dev)))
    return sims, cells, npl


@on_data_device
def precompute_adc(query, pq_codebook, distance="euclidean"):
    """PQCodec.precompute_adc: query [d, nq], pq_codebook [M, dsub, 256] -> [M, nq, 256] fp32."""
    q, cb = _cuda_f32(query, "query"), _cuda_f32(pq_codebook, "pq_codebook")
    M, dsub, K = cb.shape
    assert K == 256 and q.shape[0] == M * dsub                           # PQCodec.py:71
    nq = q.shape[1]
    out = torch.empty(M, nq, 256, dtype=torch.float32, device=q.device)
    check(lib.tpq_build_lut(ptr(q), ptr(cb), M * dsub, M, nq, _lib.METRIC[distance], ptr(out),
                            _lib.current_stream(q.device)))
    return out


class IVFPQTopk:
    """fn.IVFPQTopk (fn/IVFPQTopk.py:8-52): fused ADC scan + top-k over the reference storage layout."""

    def __init__(self, n_subvectors, contiguous_size=4, sm_size=None):
        assert contiguous_size == 4
        self.n_subvectors = n_subvectors

    @on_device(lambda self, data, *a, **k: data.device)
    def topk(self, data, precomputed, cell_start, cell_size, is_empty, n_probe_list, k=256):
        assert 0 < k <= 1024                                             # fn/IVFPQTopk.py:64
        n_data = data.shape[1]
        n_query, n_probe = cell_start.shape
        # IVFPQTopkCuda.py:98-110
        assert precomputed.shape == (self.n_subvectors, n_query, 256)
        assert data.shape[0] == self.n_subvectors // 4 and data.shape[2] == 4
        assert is_empty.shape[0] == n_data
        assert cell_size.shape[1] == n_probe
        assert data.dtype == torch.uint8 and precomputed.dtype == torch.float32
        assert cell_start.dtype == cell_size.dtype == torch.int64
        assert is_empty.dtype == torch.uint8
        assert n_probe_list.shape == (n_query,) and n_probe_list.dtype == torch.int64
        dev = data.device
        assert dev.type == "cuda"
        data, precomputed, is_empty = data.contiguous(), precomputed.contiguous(), is_empty.contiguous()
        cell_start, cell_size, n_probe_list = cell_start.contiguous(), cell_size.contiguous(), n_probe_list.contiguous()
        values = torch.empty(n_query, k, dtype=torch.float32, device=dev)
        address = torch.empty(n_query, k, dtype=torch.int64, device=dev)
        check(lib.tpq_ivfpq_topk(ptr(data), ptr(precomputed), ptr(is_empty), ptr(cell_start), ptr(cell_size),
                                 ptr(n_probe_list), n_data, self.n_subvectors, n_query, n_probe, k,
                                 ptr(values), ptr(address), None, 0, _lib.current_stream(dev)))
        return values, address


@on_data_device
def max_sim(data, centroids, distance="euclidean", exact=True, exact_values=True):
    """MultiKMeans.get_labels / MaxSimCuda(dim=2): data [l, d, n], centroids [l, d, k] ->
    (maxsims [l, n] f32, labels [l, n] i64); distance "euclidean", "cosine" (inner product) or "manhattan".  exact=False lets the TF32 tensor-core kernel run where it applies;
    exact_values then selects exact fp32 maxsims for the chosen centroid (True) or TF32-derived ones (False, faster)."""
    a, b = _cuda_f32(data, "data"), _cuda_f32(centroids, "centroids")
    assert a.dim() == 3 and b.dim() == 3 and a.shape[:2] == b.shape[:2]
    l, d, n = a.shape
    k = b.shape[2]
    sims = torch.empty(l, n, dtype=torch.float32, device=a.device)
    labels = torch.empty(l, n, dtype=torch.long, device=a.device)
    check(lib.tpq_max_sim(ptr(a), ptr(b), l, d, n, k, _lib.METRIC[distance], 1 if exact else (2 if exact_values else 0), ptr(sims), ptr(labels),
                          _lib.current_stream(a.device)))
    return sims, labels


@on_data_device
def kmeans_assign(data, centroids, distance="euclidean", exact_values=True):
    """The assignment step of KMeans / MultiKMeans: data [l, d, n], centroids [l, d, k] -> (maxsims [l, n] f32,
    labels [l, n] i64), on the TF32 tensor-core kernels wherever one takes the shape (tpq_kmeans_assign in
    include/tpq_b200.h lists the ranges), else on the exact kernel.  distance "cosine" scores inner products: pass
    normalised columns.  exact_values: exact fp32 maxsims for the chosen centroid (True) or TF32-derived ones."""
    a, b = _cuda_f32(data, "data"), _cuda_f32(centroids, "centroids")
    assert a.dim() == 3 and b.dim() == 3 and a.shape[:2] == b.shape[:2]
    l, d, n = a.shape
    k = b.shape[2]
    sims = torch.empty(l, n, dtype=torch.float32, device=a.device)
    labels = torch.empty(l, n, dtype=torch.long, device=a.device)
    ws_bytes = lib.tpq_kmeans_assign_workspace_bytes(l, d, k)
    ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=a.device)
    check(lib.tpq_kmeans_assign(ptr(a), ptr(b), l, d, n, k, _lib.METRIC[distance], int(bool(exact_values)),
                                ptr(sims), ptr(labels), ptr(ws), ws_bytes, _lib.current_stream(a.device)))
    return sims, labels


@on_data_device
def compute_centroids(data, labels, k):
    """ComputeCentroidsCuda.__call__: data [l, d, n], labels [l, n] i64 -> centroids [l, d, k]."""
    a = _cuda_f32(data, "data")
    assert labels.dtype == torch.int64 and labels.shape == (a.shape[0], a.shape[2])
    labels = labels.contiguous()
    l, d, n = a.shape
    cent = torch.empty(l, d, k, dtype=torch.float32, device=a.device)
    ws_bytes = lib.tpq_compute_centroids_workspace_bytes(l, k)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=a.device)
    check(lib.tpq_compute_centroids(ptr(a), ptr(labels), l, d, n, k, ptr(cent), ptr(ws), ws_bytes,
                                    _lib.current_stream(a.device)))
    return cent


@on_data_device
def pq_decode(codebook, code):
    """PQDecodeCuda.__call__: codebook [M, dsub, 256], code [M, n] u8 -> [M*dsub, n] f32."""
    cb = _cuda_f32(codebook, "codebook")
    assert code.dtype == torch.uint8 and code.dim() == 2 and code.shape[0] == cb.shape[0] and cb.shape[2] == 256
    code = code.contiguous()
    M, dsub, _ = cb.shape
    n = code.shape[1]
    out = torch.empty(M * dsub, n, dtype=torch.float32, device=cb.device)
    check(lib.tpq_pq_decode(ptr(cb), ptr(code), M, dsub, n, ptr(out), _lib.current_stream(cb.device)))
    return out


@on_data_device
def merge_topk(keys, address2id):
    """keys [n_parts, nq, k] int64-viewed packed candidates (each part sorted) -> (values, ids, address)."""
    assert keys.dim() == 3 and keys.dtype == torch.int64 and keys.is_contiguous()
    n_parts, nq, k = keys.shape
    dev = keys.device
    values = torch.empty(nq, k, dtype=torch.float32, device=dev)
    ids = torch.empty(nq, k, dtype=torch.long, device=dev)
    address = torch.empty(nq, k, dtype=torch.long, device=dev)
    check(lib.tpq_merge_topk(ptr(keys), nq, n_parts, k, ptr(address2id), address2id.shape[0],
                             ptr(values), ptr(ids), ptr(address), _lib.current_stream(dev)))
    return values, ids, address


class Topk:
    """fn.Topk (fn/Topk.py:43-67): row-wise top-k of a 2-D CUDA tensor, fp32 or fp16, on one sm_90a select kernel.

    ``__call__(x, k=1, dim=1)`` -> (values [m, k] in x.dtype, indices [m, k] int64).  Order: value descending, then
    column ascending; +0 ranks above -0 and every NaN, of either sign, above +inf.  Rows shorter than k are padded with
    (-inf, -1).  k > 1024 raises NotImplementedError (the reference falls back to torch.topk; this package has no
    torch fallback)."""

    @on_device(lambda self, x, *a, **k: x.device)
    def __call__(self, x, k=1, dim=1):
        if dim == -1:
            dim = 1
        assert dim == 1, "only support last dimention"
        assert len(x.shape) == 2, "only support 2d tensors"
        assert x.is_contiguous(), "x is not contiguous"
        assert k >= 1
        assert x.device.type == "cuda"
        assert x.dtype in (torch.float32, torch.float16), f"x must be float32 or float16, got {x.dtype}"
        k = int(k)
        if k > 1024:
            raise NotImplementedError(f"Topk: k={k} > 1024 is not supported")
        m, n = x.shape
        dtype = _lib.DTYPE_F32 if x.dtype == torch.float32 else _lib.DTYPE_F16
        dev = x.device
        values = torch.empty(m, k, dtype=torch.float32, device=dev)
        indices = torch.empty(m, k, dtype=torch.int64, device=dev)
        ws_bytes = lib.tpq_topk_workspace_bytes(m, n, k, dtype)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev) if ws_bytes else None
        check(lib.tpq_topk(ptr(x), m, n, dtype, k, ptr(values), ptr(indices), ptr(ws), ws_bytes, _lib.current_stream(dev)))
        return values.to(x.dtype), indices


# ------------------------------------------------------------------ build side (CellContainer.add, CellContainer.py:313-367)
@on_data_device
def get_ioa(cells, n_cells):
    """get_ioa (kernels/cuda/get_ioa.cu:8-47): cells [n] i64 -> (ioa [n] i64, counts [n_cells] i64)."""
    assert cells.dtype == torch.int64 and cells.dim() == 1 and cells.device.type == "cuda"
    cells = cells.contiguous()
    n, dev = cells.shape[0], cells.device
    ioa = torch.empty(n, dtype=torch.long, device=dev)
    counts = torch.empty(n_cells, dtype=torch.long, device=dev)
    ws_bytes = lib.tpq_ioa_workspace_bytes(n, n_cells)
    ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
    check(lib.tpq_get_ioa(ptr(cells), n, n_cells, ptr(ioa), ptr(counts), ptr(ws), ws_bytes, _lib.current_stream(dev)))
    return ioa, counts


@on_data_device
def empty_prefix(is_empty):
    """prefix[a] = number of empty slots in [0, a), a = 0..capacity  (int32-viewed uint32)."""
    assert is_empty.dtype == torch.uint8 and is_empty.device.type == "cuda"
    is_empty = is_empty.contiguous()
    cap, dev = is_empty.shape[0], is_empty.device
    prefix = torch.empty(cap + 1, dtype=torch.int32, device=dev)
    ws_bytes = lib.tpq_empty_prefix_workspace_bytes(cap)
    ws = torch.empty(max(1, ws_bytes), dtype=torch.uint8, device=dev)
    check(lib.tpq_empty_prefix(ptr(is_empty), cap, ptr(prefix), ptr(ws), ws_bytes, _lib.current_stream(dev)))
    return prefix


@on_data_device
def get_write_address(cells, ioa, cell_start, cell_size, cell_capacity, prefix=None):
    """get_write_address (kernels/cuda/get_write_address_v2.cu:9-41): the ioa-th empty slot of each item's cell."""
    n, dev = cells.shape[0], cells.device
    out = torch.empty(n, dtype=torch.long, device=dev)
    check(lib.tpq_get_write_address(ptr(cells), ptr(ioa), n, ptr(cell_start), ptr(cell_size), ptr(cell_capacity),
                                    cell_start.shape[0], ptr(prefix), ptr(out), _lib.current_stream(dev)))
    return out
