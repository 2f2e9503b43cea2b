"""CPU restatement of ``torchpq.index.IVFPQIndex.search`` (non-residual branch).

TEST INFRASTRUCTURE -- see ``oracle/__init__.py``.  Every function cites the
reference lines (relative to /root/reference) whose behaviour it restates.  The
code is written from the reference's *semantics* (SURVEY.md Appendix A), with
numpy for the integer/byte work and torch-CPU fp32 for the floating point so that
the transcendental functions are the same ones the reference calls.

Tie rule.  The reference's order among equal scores is whatever its bitonic
network yields (unspecified).  The oracle and the product both use the total
order (score descending, address ascending); parity tests are tie-free at the
k-th boundary where they demand identical ids.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Optional, Tuple

import numpy as np
import torch

INT64_MIN = np.iinfo(np.int64).min


# ----------------------------------------------------------------------------------
# index state (what search reads):  torchpq/container/CellContainer.py:46-81,
# torchpq/container/BaseContainer.py:32-38, codec/VQCodec.py:15-17, codec/PQCodec.py:36-46
# ----------------------------------------------------------------------------------
@dataclass
class IndexState:
    d_vector: int
    n_subvectors: int
    n_cells: int
    distance: str                      # "euclidean" | "cosine"
    vq_codebook: np.ndarray            # [d, C] f32
    pq_codebook: np.ndarray            # [M, dsub, 256] f32
    storage: np.ndarray                # [M/4, cap, 4] u8  (storage[g, a, j] = code[4g+j] of address a)
    is_empty: np.ndarray               # [cap] u8
    cell_start: np.ndarray             # [C] i64
    cell_size: np.ndarray              # [C] i64
    cell_capacity: np.ndarray          # [C] i64
    address2id: np.ndarray             # [cap] i64
    max_id: int = -1
    n_probe: int = 1
    use_smart_probing: bool = True
    smart_probing_temperature: float = 30.0

    @property
    def capacity(self) -> int:
        return int(self.address2id.shape[0])

    @property
    def d_subvector(self) -> int:
        return self.d_vector // self.n_subvectors


# ----------------------------------------------------------------------------------
# container write side (used to BUILD states the way the reference would place them)
# ----------------------------------------------------------------------------------
def empty_state(d_vector, n_subvectors, n_cells, initial_size, distance="euclidean",
                vq_codebook=None, pq_codebook=None) -> IndexState:
    """Freshly constructed container: CellContainer.__init__ (CellContainer.py:46-81),
    BaseContainer.__init__ (BaseContainer.py:32-37); contiguous_size=4 (IVFPQIndex.py:41)."""
    assert d_vector % n_subvectors == 0 and n_subvectors % 4 == 0
    cap = n_cells * initial_size
    M = n_subvectors
    if vq_codebook is None:
        vq_codebook = np.zeros((d_vector, n_cells), np.float32)
    if pq_codebook is None:
        pq_codebook = np.zeros((M, d_vector // M, 256), np.float32)
    return IndexState(
        d_vector=d_vector, n_subvectors=M, n_cells=n_cells, distance=distance,
        vq_codebook=np.ascontiguousarray(vq_codebook, np.float32),
        pq_codebook=np.ascontiguousarray(pq_codebook, np.float32),
        storage=np.zeros((M // 4, cap, 4), np.uint8),
        is_empty=np.ones(cap, np.uint8),
        cell_start=np.arange(n_cells, dtype=np.int64) * initial_size,
        cell_size=np.zeros(n_cells, np.int64),
        cell_capacity=np.zeros(n_cells, np.int64) + initial_size,
        address2id=-np.ones(cap, np.int64),
    )


def get_ioa(cells: np.ndarray) -> np.ndarray:
    """Index of appearance of each label among equal labels, in input order
    (kernels/cuda/get_ioa.cu:8-47; CPU form CellContainer.py:117-125)."""
    n = cells.shape[0]
    order = np.argsort(cells, kind="stable")
    sorted_cells = cells[order]
    first = np.ones(n, bool)
    first[1:] = sorted_cells[1:] != sorted_cells[:-1]
    run_start = np.maximum.accumulate(np.where(first, np.arange(n), 0))
    ioa = np.empty(n, np.int64)
    ioa[order] = np.arange(n) - run_start
    return ioa


def _expand(st: IndexState, cells: np.ndarray, expand_mode="double", expand_step_size=128):
    """CellContainer.expand (CellContainer.py:249-311): insert a block of fresh slots
    right after each listed cell and shift every later cell.  A cell of capacity 0 grows
    by expand_step_size in "double" mode too (the reference doubles it to 0, forever)."""
    for c in cells:
        c = int(c)
        start, cap = int(st.cell_start[c]), int(st.cell_capacity[c])
        end = start + cap
        n_new = (cap or expand_step_size) if expand_mode == "double" else expand_step_size
        st.storage = np.concatenate(
            [st.storage[:, :end], np.zeros((st.storage.shape[0], n_new, 4), np.uint8), st.storage[:, end:]], axis=1)
        st.address2id = np.concatenate([st.address2id[:end], -np.ones(n_new, np.int64), st.address2id[end:]])
        st.is_empty = np.concatenate([st.is_empty[:end], np.ones(n_new, np.uint8), st.is_empty[end:]])
        st.cell_capacity[c] += n_new
        st.cell_start[c + 1:] += n_new


def container_add(st: IndexState, codes: np.ndarray, cells: np.ndarray,
                  ids: Optional[np.ndarray] = None, expand_mode="double", expand_step_size=128):
    """CellContainer.add (CellContainer.py:313-367): place code[:, i] at the ioa[i]-th
    empty slot of cell cells[i] (get_write_address_v2.cu:9-41), expanding cells that
    are too small (CellContainer.py:338-344), and update the bookkeeping buffers
    (CellContainer.py:355-360).  Returns (ids, write_address)."""
    M, n = codes.shape
    assert M == st.n_subvectors and cells.shape == (n,)
    codes = np.ascontiguousarray(codes, np.uint8)
    cells = cells.astype(np.int64)
    if ids is None:
        ids = np.arange(n, dtype=np.int64) + st.max_id + 1
    ioa = get_ioa(cells)
    while True:
        free = st.cell_capacity[cells] - st.cell_size[cells] - (ioa + 1)
        need = np.unique(cells[free < 0])
        if need.shape[0] == 0:
            break
        _expand(st, need, expand_mode, expand_step_size)
    # ioa-th empty slot of [start, start+capacity) per item (get_write_address_v2.cu:25-39)
    write = np.empty(n, np.int64)
    order = np.argsort(cells, kind="stable")
    sc = cells[order]
    bounds = np.flatnonzero(np.r_[True, sc[1:] != sc[:-1], True])
    for b0, b1 in zip(bounds[:-1], bounds[1:]):
        c = int(sc[b0])
        s, cap = int(st.cell_start[c]), int(st.cell_capacity[c])
        empties = s + np.flatnonzero(st.is_empty[s:s + cap] == 1)
        idx = order[b0:b1]
        write[idx] = empties[ioa[idx]]
    # set_data_by_address (CellContainer.py:213-239): [M, n] -> [M/4, n, 4]
    st.storage[:, write, :] = codes.reshape(M // 4, 4, n).transpose(0, 2, 1)
    st.address2id[write] = ids
    st.max_id = max(st.max_id, int(ids.max())) if n else st.max_id
    st.is_empty[write] = 0
    uc, cnt = np.unique(cells, return_counts=True)
    st.cell_size[uc] += cnt
    return ids, write


def codes_at(st: IndexState, address: np.ndarray) -> np.ndarray:
    """get_data_by_address (CellContainer.py:175-211): [M, n] codes of the given addresses."""
    d = st.storage[:, address, :]                     # [M/4, n, 4]
    return d.transpose(0, 2, 1).reshape(st.n_subvectors, -1)


# ----------------------------------------------------------------------------------
# search path
# ----------------------------------------------------------------------------------
def normalize(x: torch.Tensor, dim: int = 0) -> torch.Tensor:
    """util.normalize (util.py:38-43): x / (||x||_2 + 1e-9)."""
    return x / (x.norm(dim=dim, keepdim=True) + 1e-9)


def negative_squared_l2(a: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    """metric.negative_squared_l2_distance fp32 branch (metric.py:74-94) and
    MultiKMeans.euc_sim (MultiKMeans.py:183-209): ((a^T b) * 2 - sum a^2) - sum b^2,
    in that order, fp32.  a: [..., d, m], b: [..., d, n] -> [..., m, n]."""
    y = a.transpose(-2, -1).contiguous() @ b
    y = y * 2
    a2 = (a ** 2).sum(dim=-2)[..., :, None]
    y = y - a2
    b2 = (b ** 2).sum(dim=-2)[..., None, :]
    y = y - b2
    return y


def topk_desc(sims: torch.Tensor, k: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """fn.Topk.__call__ (fn/Topk.py:43-67) -> top32_select / topk_select write-out
    (top32_select.cu:629-635): per row the k largest, sorted DESCENDING, int64 indices.
    Ties: lower column index first (oracle's tie rule)."""
    s = sims.numpy()
    n = s.shape[1]
    # stable sort on (-value) keeps lower index first among equals
    order = np.argsort(-s, axis=1, kind="stable")[:, :k]
    vals = np.take_along_axis(s, order, axis=1)
    return torch.from_numpy(vals.copy()), torch.from_numpy(order.astype(np.int64))


def smart_probing(topk_sims: torch.Tensor, n_probe: int, temperature: float) -> torch.Tensor:
    """IVFPQIndex.search smart-probing block (IVFPQIndex.py:499-510):
    p = softmax(-sqrt|s| / T); H = -sum p log2 p / log2(n_probe); ceil(H * n_probe).long().
    A NaN entropy (some p == 0) converts to INT64_MIN, as CUDA's float->int64 cast does."""
    p = -topk_sims.abs().sqrt()
    p = torch.softmax(p / temperature, dim=-1)
    max_n_probe = torch.tensor(n_probe)
    h = -torch.sum(p * torch.log2(p) / torch.log2(max_n_probe), dim=-1)
    v = torch.ceil(h * max_n_probe)
    out = np.empty(v.shape[0], np.int64)
    vn = v.numpy()
    nan = np.isnan(vn)
    out[~nan] = vn[~nan].astype(np.int64)
    out[nan] = INT64_MIN
    return torch.from_numpy(out)


def precompute_adc(x: torch.Tensor, pq_codebook: torch.Tensor, distance: str) -> torch.Tensor:
    """PQCodec.precompute_adc (PQCodec.py:62-75) -> MultiKMeans.sim (MultiKMeans.py:211-223):
    euclidean -> euc_sim; cosine -> cos_sim(normalize=False) = plain inner product.
    x [d, nq] -> LUT [M, nq, 256] fp32."""
    M, dsub, K = pq_codebook.shape
    q = x.reshape(M, dsub, x.shape[1])
    if distance == "euclidean":
        return negative_squared_l2(q, pq_codebook)
    elif distance == "cosine":
        return q.transpose(-2, -1) @ pq_codebook
    raise ValueError(f"unsupported distance {distance!r} (reference supports euclidean, cosine)")


def effective_probes(n_probe_list: np.ndarray, n_probe: int) -> np.ndarray:
    """ivfpq_topk.cu:837 reads nProbeList as a 32-bit int; cell 0 is entered
    unconditionally (:850-856) and the nProbe test happens only when advancing (:858-860).
    Values above n_probe would read past the row in the reference; we clamp (SURVEY App. C #3)."""
    as_int = n_probe_list.astype(np.int64).astype(np.int32)   # (int) truncation of the int64
    return np.maximum(1, np.minimum(as_int.astype(np.int64), n_probe))


def probed_addresses(cell_start_g: np.ndarray, cell_size_g: np.ndarray, P: int) -> np.ndarray:
    """Addresses visited for one query: first P probe entries in order, entry j skipped when its
    start equals the previous entry's start (ivfpq_topk.cu:857-870), range [start, start+size)."""
    chunks = []
    prev_start = None
    for j in range(P):
        s, n = int(cell_start_g[j]), int(cell_size_g[j])
        if j > 0 and s == prev_start:
            continue
        prev_start = s
        if n > 0:
            chunks.append(np.arange(s, s + n, dtype=np.int64))
    return np.concatenate(chunks) if chunks else np.zeros(0, np.int64)


def adc_scores(storage: np.ndarray, lut_q: np.ndarray, addr: np.ndarray) -> np.ndarray:
    """consume_data (ivfpq_topk.cu:662-679): fp32 sum of LUT[m][code_m] for m ascending, from 0.f.
    storage [M/4, cap, 4]; lut_q [M, 256] fp32; returns fp32 [len(addr)]."""
    M = lut_q.shape[0]
    codes = storage[:, addr, :]                             # [M/4, n, 4]
    acc = np.zeros(addr.shape[0], np.float32)
    for m in range(M):
        acc = acc + lut_q[m][codes[m // 4, :, m % 4]]       # fp32 add, m ascending
    return acc


def select_topk(scores: np.ndarray, addr: np.ndarray, k: int):
    """Keep the k best (score desc, address asc); pad with (-inf, -1)
    (ivfpq_topk.cu:966-970; IVFPQTopkCuda.py:118-120,142)."""
    vals = np.full(k, -np.inf, np.float32)
    out = np.full(k, -1, np.int64)
    if scores.shape[0]:
        order = np.lexsort((addr, -scores.astype(np.float64)))[:k]
        vals[:order.shape[0]] = scores[order]
        out[:order.shape[0]] = addr[order]
    return vals, out


def ivfpq_topk(storage, precomputed, is_empty, cell_start_g, cell_size_g, n_probe_list, k):
    """fn.IVFPQTopk.topk (fn/IVFPQTopk.py:54-104) -> IVFPQTopkCuda.topk (IVFPQTopkCuda.py:81-142)
    -> ivfpq_topk kernel (ivfpq_topk.cu:822-971).  precomputed [M, nq, 256]; cell_start_g/size_g
    [nq, n_probe]; returns (values [nq,k] f32 desc, address [nq,k] i64)."""
    pre = np.asarray(precomputed, np.float32)
    nq, n_probe = cell_start_g.shape
    P = effective_probes(np.asarray(n_probe_list), n_probe)
    vals = np.empty((nq, k), np.float32)
    adr = np.empty((nq, k), np.int64)
    for q in range(nq):
        a = probed_addresses(cell_start_g[q], cell_size_g[q], int(P[q]))
        a = a[is_empty[a] == 0]                              # ivfpq_topk.cu:878,883-884
        s = adc_scores(storage, np.ascontiguousarray(pre[:, q, :]), a)
        vals[q], adr[q] = select_topk(s, a, k)
    return vals, adr


def get_id_by_address(address2id: np.ndarray, address: np.ndarray) -> np.ndarray:
    """BaseContainer.get_id_by_address (BaseContainer.py:58-65)."""
    ok = (address >= 0) & (address < address2id.shape[0])
    ids = -np.ones_like(address)
    ids[ok] = address2id[address[ok]]
    return ids


def coarse_probe(st: IndexState, x: torch.Tensor):
    """IVFPQIndex.search lines 474-512: optional cosine normalisation, coarse scores against
    the VQ codebook (always L2, IVFPQIndex.py:63-71), top-n_probe, smart probing.
    Returns (x_used, topk_sims [nq,np] f32, cells [nq,np] i64, n_probe_list [nq] i64)."""
    if st.distance == "cosine":
        x = normalize(x, dim=0)
    sims = negative_squared_l2(x, torch.from_numpy(st.vq_codebook)).contiguous()
    topk_sims, cells = topk_desc(sims, st.n_probe)
    if st.use_smart_probing and st.n_probe > 1:
        npl = smart_probing(topk_sims, st.n_probe, st.smart_probing_temperature)
    else:
        npl = torch.zeros(x.shape[1], dtype=torch.long) + st.n_probe
    return x, topk_sims, cells, npl


def search(st: IndexState, x, k: int = 1, return_address: bool = False):
    """IVFPQIndex.search (IVFPQIndex.py:469-524) + search_cells non-residual branch (:407-467).
    x [d, nq] fp32 -> (values [nq,k] f32 desc, ids [nq,k] i64[, address])."""
    x = torch.as_tensor(x, dtype=torch.float32)
    assert x.dim() == 2 and x.shape[0] == st.d_vector and 0 < k <= 1024
    x, topk_sims, cells, npl = coarse_probe(st, x)
    cells_np = cells.numpy()
    cell_start_g = st.cell_start[cells_np]                   # IVFPQIndex.py:420-421
    cell_size_g = st.cell_size[cells_np]
    lut = precompute_adc(x, torch.from_numpy(st.pq_codebook), st.distance).numpy()
    vals, adr = ivfpq_topk(st.storage, lut, st.is_empty, cell_start_g, cell_size_g, npl.numpy(), k)
    ids = get_id_by_address(st.address2id, adr)
    if return_address:
        return vals, ids, adr
    return vals, ids


# ----------------------------------------------------------------------------------
# exact brute force (ground truth for recall; not a reference function)
# ----------------------------------------------------------------------------------
def exact_topk(base: torch.Tensor, x: torch.Tensor, k: int, distance: str):
    """Ground truth neighbours of x [d,nq] in base [d,N] by exact L2 / cosine (fp32)."""
    if distance == "cosine":
        s = normalize(x, 0).T @ normalize(base, 0)
    else:
        s = negative_squared_l2(x, base)
    return torch.topk(s, k, dim=1).indices


def recall_at_k(found_ids: np.ndarray, truth_ids: np.ndarray) -> float:
    nq, k = truth_ids.shape
    hit = 0
    for q in range(nq):
        hit += np.intersect1d(found_ids[q], truth_ids[q]).shape[0]
    return hit / float(nq * k)


# ----------------------------------------------------------------------------------
# residual IVFPQ (pq_use_residual=True, precomputed part-2 tables)  --  SURVEY.md section 8(f) rank 3
# ----------------------------------------------------------------------------------
def precompute_part2(vq_codebook: torch.Tensor, pq_codebook: torch.Tensor) -> torch.Tensor:
    """IVFPQIndex.precompute_part2 (IVFPQIndex.py:160-170): [M, n_cells, 256] =
    bmm(vq^T, pq) * -2 - ||p||^2, with ||p||^2 computed as norm(dim=1).pow(2) exactly as the reference does."""
    M, dsub, K = pq_codebook.shape
    n_cells = vq_codebook.shape[1]
    vq = vq_codebook.reshape(M, dsub, n_cells)
    return torch.bmm(vq.transpose(-1, -2), pq_codebook) * -2 - pq_codebook.norm(dim=1).pow(2)[:, None]


def residual_parts(x: torch.Tensor, vq_codebook: torch.Tensor, pq_codebook: torch.Tensor):
    """precomputed_adc_residual_precomputed (IVFPQIndex.py:366-380):
    part1 [nq, M, 256] = 2 * (x_m^T p_m), part2 [n_cells, M, 256] = precompute_part2^T(0,1)."""
    M, dsub, K = pq_codebook.shape
    nq = x.shape[1]
    xm = x.reshape(M, dsub, nq).transpose(-1, -2)
    part1 = 2 * (xm @ pq_codebook).permute(1, 0, 2)
    part2 = precompute_part2(vq_codebook, pq_codebook).transpose(0, 1)
    return part1.contiguous(), part2.contiguous()


def ivfpq_topk_residual_precomputed(storage, part1, part2, cells, base_sims, is_empty, cell_start_g, cell_size_g,
                                    n_probe_list, k):
    """ivfpq_topk_residual_precomputed (ivfpq_topk.cu:1039-1207) as launched by
    IVFPQTopkCuda.topk_residual_precomputed (IVFPQTopkCuda.py:212-283).
    score = base_sims[q, j] + sum_m (part1[q, m, code] + part2[cell, m, code]), the smem entry being the fp32 sum
    part1 + part2 (store_precomputed_to_smem :609-628), accumulated m ascending starting from the base similarity.
    The loop runs over cCell < nProbe only (no unconditional first cell, unlike the non-residual kernel); an entry
    whose start equals the previous entry's start is skipped (:1088-1104)."""
    p1 = np.asarray(part1, np.float32); p2 = np.asarray(part2, np.float32)
    base = np.asarray(base_sims, np.float32)
    nq, n_probe = cell_start_g.shape
    M = p1.shape[1]
    as_int = np.asarray(n_probe_list).astype(np.int64).astype(np.int32).astype(np.int64)
    P = np.clip(as_int, 0, n_probe)
    vals = np.empty((nq, k), np.float32); adr = np.empty((nq, k), np.int64)
    for q in range(nq):
        sc, ad = [], []
        prev = None
        for j in range(int(P[q])):
            s, n = int(cell_start_g[q, j]), int(cell_size_g[q, j])
            if j > 0 and s == prev:
                continue
            prev = s
            if n <= 0:
                continue
            a = np.arange(s, s + n, dtype=np.int64)
            a = a[is_empty[a] == 0]
            lut = (p1[q] + p2[int(cells[q, j])]).astype(np.float32)          # [M, 256]
            codes = storage[:, a, :]
            acc = np.full(a.shape[0], base[q, j], np.float32)
            for m in range(M):
                acc = acc + lut[m][codes[m // 4, :, m % 4]]
            sc.append(acc); ad.append(a)
        if sc:
            vals[q], adr[q] = select_topk(np.concatenate(sc), np.concatenate(ad), k)
        else:
            vals[q], adr[q] = select_topk(np.zeros(0, np.float32), np.zeros(0, np.int64), k)
    return vals, adr


def search_residual(st: IndexState, x, k: int = 1, return_address: bool = False):
    """IVFPQIndex.search with pq_use_residual=True and use_precomputed=True (IVFPQIndex.py:469-524, 407-438)."""
    x = torch.as_tensor(x, dtype=torch.float32)
    x, topk_sims, cells, npl = coarse_probe(st, x)
    cn = cells.numpy()
    part1, part2 = residual_parts(x, torch.from_numpy(st.vq_codebook), torch.from_numpy(st.pq_codebook))
    vals, adr = ivfpq_topk_residual_precomputed(st.storage, part1.numpy(), part2.numpy(), cn, topk_sims.numpy(),
                                                st.is_empty, st.cell_start[cn], st.cell_size[cn], npl.numpy(), k)
    ids = get_id_by_address(st.address2id, adr)
    return (vals, ids, adr) if return_address else (vals, ids)
