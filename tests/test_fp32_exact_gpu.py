"""GPU: the search kernels equal their fp32 restatements (oracle/fp32_exact.py) bit for bit on real-valued data -- the
coarse GEMM, probe select and cosine normalisation, the LUT builders, and the scan's summation order on every path
(in-CTA and staged LUTs, wide codes, sliced batches, the cell-major scan, cosine, residual) -- and smart probing lies
within a derived fp32 error margin of float64.  Every comparison is exact; a tolerance here would hide the subtle
kernel changes these tests exist to catch."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import build_state as B, fp32_exact as X, ivfpq_oracle as O
from helpers import make_index
from test_cell_scan_gpu import NQ as CELL_NQ, cell_major_index

pytestmark = pytest.mark.gpu

F32 = np.float32


def g(a):
    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def assert_bits(got, want):
    got, want = np.asarray(got, F32), np.asarray(want, F32)
    assert got.shape == want.shape
    bad = got.view(np.uint32) != want.view(np.uint32)
    assert not bad.any(), f"{int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0]}: " \
                          f"{got[bad][0]!r} != {want[bad][0]!r}"


def gpu_coarse(x, cb, n_probe, smart=False, temperature=30.0):
    import torchpq_b200 as T
    s, c, n = T.fn.coarse_probe(g(x), g(cb), n_probe, smart, temperature)
    return s.cpu().numpy(), c.cpu().numpy(), n.cpu().numpy()


def check_coarse(x, cb, n_probe):
    s, c, n = gpu_coarse(x, cb, n_probe)
    ws, wc = X.coarse_probe(x, cb, n_probe)
    assert_bits(s, ws)
    assert np.array_equal(c, wc)
    assert (n == n_probe).all()
    return wc


# ----------------------------------------------------------------------------------------- coarse stage
def _randn(shape, seed, scale=1.0):
    return (np.random.default_rng(seed).standard_normal(shape) * scale).astype(F32)


@pytest.mark.parametrize("d", [1, 2, 15, 16, 17, 33, 128, 960])
def test_coarse_d(cuda_device, d):
    """K = d: a partial first K slab, exactly one, one and a bit, many (coarse_gemm_kernel's GK = 16)."""
    check_coarse(_randn((d, 129), d), _randn((d, 131), d + 1), 131)


@pytest.mark.parametrize("C", [1, 3, 4, 127, 128, 129, 131, 1000, 1027])
def test_coarse_cells(cuda_device, C):
    """C % 4 != 0 (the scalar-store epilogue), partial column tiles, several tiles on both grid axes (129 queries)."""
    check_coarse(_randn((33, 129), C), _randn((33, C), C + 1), min(C, 1024))


@pytest.mark.parametrize("nq", [1, 127, 128, 129, 300])
def test_coarse_queries(cuda_device, nq):
    check_coarse(_randn((17, nq), nq), _randn((17, 131), nq + 1), 131)


@pytest.mark.parametrize("n_probe", [1, 31, 32, 33, 64, 65, 255, 256, 257, 1000, 1024])
def test_probe_select_list_capacities(cuda_device, n_probe):
    """n_probe across the steps of list_capacity (32 .. 1024 slots) on 16384 cells."""
    check_coarse(_randn((8, 37), n_probe), _randn((8, 16384), 7), n_probe)


def test_probe_select_ties(cuda_device):
    """Duplicated centroid columns tie exactly: the lower cell comes first.  All centroids equal: cells 0..n_probe-1."""
    cb = _randn((24, 300), 1)
    cb[:, 150:] = cb[:, :150]
    x = _randn((24, 70), 2)
    cells = check_coarse(x, cb, 64)
    assert (cells[:, 1::2] == cells[:, ::2] + 150).all()       # each pair ties: the lower copy first, its twin next
    for C, n_probe in ((300, 64), (1027, 1024)):
        same = np.repeat(_randn((24, 1), 3), C, axis=1)
        cells = check_coarse(x, same, n_probe)
        assert (cells == np.arange(n_probe)).all()


@pytest.mark.parametrize("scale", [1e3, 1e-3])
def test_coarse_cancellation(cuda_device, scale):
    """Queries close to centroids of a codebook scaled by 1e3 / 1e-3: sims are differences of nearly equal large terms,
    so the epilogue's rounding order shows."""
    cb = _randn((40, 257), 5, scale)
    pick = np.random.default_rng(6).integers(0, 257, 150)
    x = (cb[:, pick] + _randn((40, 150), 7, scale * 1e-3)).astype(F32)
    check_coarse(x, cb, 257)


@pytest.mark.parametrize("d", [1, 33, 960])
def test_normalize_columns(cuda_device, d):
    import torchpq_b200 as T
    x = _randn((d, 129), d, 3.0)
    x[:, ::17] = 0                                             # zero columns: 0 / (0 + 1e-9)
    x[:, 5] = 1e-20
    got = T.fn.normalize(g(x)).cpu().numpy()
    assert_bits(got, X.normalize_columns(x))


# ----------------------------------------------------------------------------------------- LUT
@pytest.mark.parametrize("M", [1, 8, 64, 120, 192])
@pytest.mark.parametrize("dsub", [1, 2, 3, 4, 8, 16])
def test_precompute_adc(cuda_device, M, dsub):
    import torchpq_b200 as T
    d = M * dsub
    pq = _randn((M, dsub, 256), M + dsub)
    for nq in (1, 17):
        x = _randn((d, nq), nq + M)
        for distance in ("euclidean", "cosine"):
            got = T.fn.precompute_adc(g(x), g(pq), distance).cpu().numpy()
            assert_bits(got, X.build_lut(x, pq, distance))


@pytest.mark.parametrize("M,dsub", [(8, 128), (4, 460), (1, 7300)])
def test_precompute_adc_wide(cuda_device, M, dsub):
    """Wide sub-vectors: lut_kernel's shared-memory tile above 48 KB (128), with fewer sub-quantizers per CTA (460), and
    with one query and one sub-quantizer per CTA (7300)."""
    import torchpq_b200 as T
    pq = _randn((M, dsub, 256), M + dsub)
    x = _randn((M * dsub, 17), dsub)
    for distance in ("euclidean", "cosine"):
        assert_bits(T.fn.precompute_adc(g(x), g(pq), distance).cpu().numpy(), X.build_lut(x, pq, distance))


@pytest.mark.parametrize("M", [8, 64, 120])
@pytest.mark.parametrize("dsub", [1, 2, 3])
def test_part2_scan(cuda_device, M, dsub):
    """The residual index's per-cell half of the LUT (ScanLayout.part2_scan) in scan layout: the m_pad rows equal their
    restatement, and the rest of a partly used last 64-sub-quantizer group is +0."""
    st = B.randn_state(M * dsub, M, 50, 1000, seed=M + dsub)
    lay = make_residual_index(st).layout()
    mp, mg = lay.m_pad, (lay.m_pad + 63) // 64
    got = lay.part2_scan.view(st.n_cells, mg, 256, 64).transpose(2, 3).reshape(st.n_cells, mg * 64, 256).cpu().numpy()
    assert_bits(got[:, :mp], X.part2(st.vq_codebook, st.pq_codebook))
    assert not got[:, mp:].view(np.uint32).any()


@pytest.mark.parametrize("nq", [15, 16, 1000])
def test_precompute_adc_query_tiles(cuda_device, nq):
    """Query counts around and across the LUT kernel's query tiles."""
    import torchpq_b200 as T
    pq = _randn((8, 3, 256), 9)
    x = _randn((24, nq), nq)
    for distance in ("euclidean", "cosine"):
        assert_bits(T.fn.precompute_adc(g(x), g(pq), distance).cpu().numpy(), X.build_lut(x, pq, distance))


def test_reference_layout_chain(cuda_device):
    """fn.precompute_adc feeding fn.IVFPQTopk.topk (reference layouts, m-ascending sums): equal to the restated LUT
    scanned by the oracle's m-ascending sum, values and addresses."""
    import torchpq_b200 as T
    st = B.randn_state(64, 16, 16, 5000, seed=3)
    st.n_probe = 6
    x = _randn((64, 40), 4)
    s, cells, npl = gpu_coarse(x, st.vq_codebook, 6, True, 1.0)
    lut = T.fn.precompute_adc(g(x), g(st.pq_codebook), "euclidean")
    wlut = X.build_lut(x, st.pq_codebook, "euclidean")
    assert_bits(lut.cpu().numpy(), wlut)
    cs, cz = st.cell_start[cells], st.cell_size[cells]
    v, a = T.fn.IVFPQTopk(16).topk(g(st.storage), lut, g(cs), g(cz), g(st.is_empty), g(npl), k=30)
    ov, oa = O.ivfpq_topk(st.storage, wlut, st.is_empty, cs, cz, npl, 30)
    assert_bits(v.cpu().numpy(), ov)
    assert np.array_equal(a.cpu().numpy(), oa)


# ----------------------------------------------------------------------------------------- smart probing vs float64
def check_smart(s, n, n_probe, temperature):
    r = X.smart_probing_check(s, n, n_probe, temperature)
    for key in ("exact_ok", "range_ok", "nan_ok", "amb_ok"):
        bad = np.flatnonzero(~r[key])
        assert bad.size == 0, (key, bad[:5], n[bad[:5]], r["v"][bad[:5]], r["margin"][bad[:5]], r["pmin"][bad[:5]])
    return r


def test_smart_probing_against_float64(cuda_device):
    """Ordinary temperatures: the list length is exactly ceil(H * n_probe) wherever float64 puts that value farther
    than the derived margin from an integer, and floor or ceil inside it -- a small fraction of rows.  Low temperatures:
    rows whose smallest softmax probability is clearly below 2^-150 (0 in fp32, so p log2 p is NaN) give INT64_MIN,
    rows clearly above 2^-149 (fp32 subnormals count as nonzero) do not; the temperatures put many rows on each side."""
    d, Cn, nq, n_probe = 32, 1024, 1000, 64
    cb = _randn((d, Cn), 0)
    x = (_randn((d, nq), 1) * 2.0 ** np.random.default_rng(2).uniform(-1, 5, nq)).astype(F32)
    rows = inside = 0
    for temperature in (1.0, 0.3, 0.1):
        s, c, n = gpu_coarse(x, cb, n_probe, True, temperature)
        r = check_smart(s, n, n_probe, temperature)
        assert r["num_rows"].all()
        rows += nq
        inside += int(r["inside"].sum())
    print(f"smart probing: {inside} of {rows} rows ({inside / rows:.2%}) within the fp32 margin of an integer")
    assert inside <= 0.05 * rows
    n_nan = n_num = n_amb = 0
    for temperature in (0.02, 0.015, 0.012):
        s, c, n = gpu_coarse(x, cb, n_probe, True, temperature)
        r = check_smart(s, n, n_probe, temperature)
        n_nan += int(r["nan_rows"].sum())
        n_num += int(r["num_rows"].sum())
        n_amb += int(r["amb_rows"].sum())
    print(f"NaN boundary: {n_nan} rows clearly below 2^-150 (INT64_MIN), {n_num} clearly above 2^-149, {n_amb} between")
    assert n_nan >= 0.25 * 3 * nq and n_num >= 0.25 * 3 * nq


# ----------------------------------------------------------------------------------------- end-to-end search
def make_residual_index(st):
    import torchpq_b200 as T
    ix = T.IVFPQIndex(st.d_vector, st.n_subvectors, st.n_cells, initial_size=1, device="cuda:0", pq_use_residual=True)
    return ix.load_state(st)


def lut_is_staged(ix, nq, n_probe, k):
    """The search workspace holds a LUT per query exactly when the LUT is staged through global memory (or the
    cell-major path writes them): the in-CTA build needs none."""
    import torchpq_b200 as T
    lay = ix.layout()
    lut_bytes = (lay.m_pad + 63) // 64 * 65536
    return T._lib.lib.tpq_search_workspace_bytes(C.byref(lay.cindex), nq, n_probe, k) >= min(nq, 16384) * lut_bytes


def run_search(st, x, k, *, residual=False, smart=True, temperature=1.0, m_pad=None, staged=None, ix=None, rows=None):
    """The GPU's search against search_cells_fp32 fed the GPU's own probe lists (which must equal the restated coarse
    stage, and whose smart-probing lengths must pass the float64 check); values bit for bit, addresses, ids."""
    st.use_smart_probing, st.smart_probing_temperature = smart, temperature
    ix = ix or (make_residual_index(st) if residual else make_index(st))
    ix.n_probe, ix.use_smart_probing, ix.smart_probing_temperature = st.n_probe, smart, temperature
    nq = x.shape[1]
    if m_pad is not None:
        assert ix.layout().m_pad == m_pad
    if staged is not None:
        assert lut_is_staged(ix, nq, st.n_probe, k) == staged
    xu = X.normalize_columns(x) if st.distance == "cosine" else x
    s, cells, npl = gpu_coarse(xu, st.vq_codebook, st.n_probe, smart, temperature)
    ws, wc = X.coarse_probe(xu, st.vq_codebook, st.n_probe)
    assert_bits(s, ws)
    assert np.array_equal(cells, wc)
    if smart and st.n_probe > 1:
        check_smart(s, npl, st.n_probe, temperature)
    v, i, a = ix.search(g(x), k=k, return_address=True)
    v, i, a = v.cpu().numpy(), i.cpu().numpy(), a.cpu().numpy()
    rows = np.arange(nq) if rows is None else rows
    wv, wa = X.search_cells_fp32(st, xu[:, rows], cells[rows], npl[rows], k, base_sims=s[rows], residual=residual)
    assert_bits(v[rows], wv)
    assert np.array_equal(a[rows], wa)
    assert np.array_equal(i[rows], O.get_id_by_address(st.address2id, wa))
    return ix


@pytest.mark.parametrize("dsub", [1, 2, 4, 8])
def test_search_in_cta_lut(cuda_device, dsub):
    st = B.randn_state(16 * dsub, 16, 24, 6000, seed=dsub)
    st.n_probe = 6
    run_search(st, _randn((16 * dsub, 64), dsub), 50, m_pad=32, staged=False)


@pytest.mark.parametrize("dsub", [3, 12, 96, 128])
def test_search_staged_lut(cuda_device, dsub):
    st = B.randn_state(16 * dsub, 16, 24, 6000, seed=dsub)
    st.n_probe = 6
    run_search(st, _randn((16 * dsub, 64), dsub), 50, m_pad=32, staged=True)


@pytest.mark.parametrize("M,dsub,m_pad,staged", [(96, 1, 96, False), (120, 2, 128, False), (192, 3, 192, True)])
def test_search_wide_codes(cuda_device, M, dsub, m_pad, staged):
    """Two and three 64-sub-quantizer units per block, the 32-byte last unit at M = 96, padding sub-quantizers."""
    st = B.randn_state(M * dsub, M, 16, 3000, seed=M)
    st.n_probe = 5
    run_search(st, _randn((M * dsub, 40), M), 40, m_pad=m_pad, staged=staged)


@pytest.mark.parametrize("nq", [1, 3])
def test_search_sliced_batches(cuda_device, nq):
    st = B.randn_state(32, 16, 32, 20000, seed=nq)
    st.n_probe = 16
    run_search(st, _randn((32, nq), nq), 64)


@pytest.mark.parametrize("k", [1, 100, 1024])
def test_search_k_and_many_probes(cuda_device, k):
    st = B.randn_state(64, 16, 300, 30000, seed=k)
    st.n_probe = 200
    run_search(st, _randn((64, 12), k), k, temperature=0.3)


def test_search_cosine(cuda_device):
    st = B.randn_state(96, 24, 32, 8000, seed=11, distance="cosine")
    st.n_probe = 8
    run_search(st, _randn((96, 50), 11, 4.0), 50)


def test_search_is_empty_holes(cuda_device):
    st = B.randn_state(64, 32, 16, 8000, seed=12)
    rng = np.random.default_rng(12)
    st.is_empty[rng.choice(np.flatnonzero(st.is_empty == 0), 2000, replace=False)] = 1
    st.n_probe = 6
    run_search(st, _randn((64, 40), 12), 30)


def test_search_cell_major(cuda_device):
    """The cell-major scan (600 queries, 2000 live vectors per cell): a subset of the queries against the restatement."""
    st = B.randn_state(128, 64, 8, 16000, seed=13)
    st.n_probe = 4
    ix = cell_major_index(st)
    rows = np.r_[0:24, 300:308, CELL_NQ - 8:CELL_NQ]
    run_search(st, _randn((128, CELL_NQ), 13), 100, ix=ix, rows=rows, m_pad=64)


@pytest.mark.parametrize("M,d,staged", [(8, 32, False), (64, 128, False), (64, 512, True), (96, 192, True),
                                        (120, 240, True)])
def test_search_residual(cuda_device, M, d, staged):
    """Residual IVFPQ: query half built in the CTA (d/M 4, 2) or staged (d/M 8, M > 64); per-cell LUT = part1 + part2,
    scores seeded with the cell's coarse similarity."""
    st = B.randn_state(d, M, 16, 4000, seed=M + d)
    st.n_probe = 6
    run_search(st, _randn((d, 24), M), 20, residual=True, staged=staged)


# ----------------------------------------------------------------------------------------- internal == exported coarse
@pytest.mark.parametrize("kind", ["euclidean", "cosine", "residual"])
def test_internal_coarse_stage_equals_exported(cuda_device, kind):
    """search(x) equals search_cells(x, cells, base_sims, n_probe_list) fed from fn.coarse_probe (on fn.normalize(x)
    for cosine), bit for bit."""
    import torchpq_b200 as T
    st = B.randn_state(64, 16, 32, 8000, seed=14, distance="cosine" if kind == "cosine" else "euclidean")
    st.n_probe, st.use_smart_probing, st.smart_probing_temperature = 8, True, 1.0
    ix = make_residual_index(st) if kind == "residual" else make_index(st)
    x = g(_randn((64, 100), 14))
    v, i, a = ix.search(x, k=25, return_address=True)
    xu = T.fn.normalize(x) if kind == "cosine" else x
    s, cells, npl = T.fn.coarse_probe(xu, g(st.vq_codebook), 8, True, 1.0)
    v2, i2, a2 = ix.search_cells(xu, cells, base_sims=s, n_probe_list=npl, k=25, return_address=True)
    assert_bits(v.cpu().numpy(), v2.cpu().numpy())
    assert torch.equal(a, a2) and torch.equal(i, i2)
