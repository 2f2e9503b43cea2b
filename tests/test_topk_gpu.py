"""GPU: torchpq_b200.topk (fn.Topk) against the numpy oracle, bit for bit: values bit-identical (a NaN as a NaN) and
indices identical, no tolerance and no row left out.  Both plan shapes (a warp per row; a CTA per row slice, with and
without the second pass over the slices' sorted parts), every list capacity, misaligned rows, 64-bit offsets and
rank-adversarial rows; then fp16 against fp32, torch.topk and, where oracle/_ref has them, the reference's own kernels."""
import numpy as np
import pytest
import torch

from oracle import select_oracle as SO

pytestmark = pytest.mark.gpu

ROWS_PLAN_M = 16 * 132        # at and above this many rows (on a 132-SM H100) every row gets one warp


def _T():
    import torchpq_b200 as T
    return T


def _check(x, k):
    """x: CUDA tensor.  Our top-k equals the oracle's on every row."""
    v, i = _T().topk(x, k=k)
    torch.cuda.synchronize()
    assert v.dtype == x.dtype and i.dtype == torch.int64 and v.shape == (x.shape[0], k) == i.shape
    ov, oi = SO.topk(x.cpu().numpy(), k)
    vn, inn = v.float().cpu().numpy(), i.cpu().numpy()
    bad = np.nonzero(~((vn.view(np.uint32) == ov.view(np.uint32)) | (np.isnan(vn) & np.isnan(ov))).all(1)
                     | ~(inn == oi).all(1))[0]
    assert bad.size == 0, f"{bad.size} rows differ, first {bad[:5]}: ours {inn[bad[0], :8]} oracle {oi[bad[0], :8]}"
    return v, i


def _data(m, n, dtype, seed, kind="randn"):
    g = torch.Generator(device="cuda").manual_seed(seed)
    if kind == "randn":
        x = torch.randn(m, n, device="cuda", generator=g)
    else:                                                    # few distinct values: ties everywhere
        x = torch.randint(0, 16, (m, n), device="cuda", generator=g).float()
    return x.to(dtype).contiguous()


KS = (1, 2, 31, 32, 33, 100, 256, 1000, 1024)
SHAPES = [
    # many short rows: a warp per row
    (70000, 1, 1), (70000, 31, 2), (70000, 32, 31), (70000, 33, 32), (3000, 1000, 33), (3000, 1000, 100),
    (2500, 4096, 256), (2200, 4096, 1000), (2200, 4096, 1024), (3000, 1000, 1024),
    # few rows, one CTA per row
    (1, 1, 1), (3, 31, 33), (3, 32, 1024), (3, 33, 2), (1000, 1000, 31), (1000, 4096, 256), (1000, 4096, 1024),
    (1000, 33, 1), (3, 4096, 100),
    # few long rows: slices and the second pass
    (1, 1 << 20, 1), (1, 1 << 20, 2), (1, 1 << 20, 31), (1, 1 << 20, 32), (1, 1 << 20, 33), (1, 1 << 20, 100),
    (1, 1 << 20, 256), (1, 1 << 20, 1000), (1, 1 << 20, 1024), (3, 1 << 20, 33), (3, 1 << 20, 1024),
]


@pytest.mark.parametrize("m,n,k", SHAPES)
@pytest.mark.parametrize("kind", ["randn", "ties"])
def test_topk_shapes_fp32(m, n, k, kind):
    _check(_data(m, n, torch.float32, m * 7 + n + k, kind), k)


@pytest.mark.parametrize("m,n,k", [(3000, 1000, 32), (1000, 4096, 100), (1, 1 << 20, 1024), (3, 1 << 20, 7),
                                   (70000, 33, 1), (2500, 4096, 1024)])
@pytest.mark.parametrize("kind", ["randn", "ties"])
def test_topk_shapes_fp16(m, n, k, kind):
    _check(_data(m, n, torch.float16, m + n * 3 + k, kind), k)


# n % 4 != 0 (fp32) / n % 8 != 0 (fp16) with m > 1: rows start at every 16-byte phase; scalar head and tail
@pytest.mark.parametrize("m,n,k", [(3, 4097, 100), (5, 100003, 100), (7, 65541, 1024), (2300, 1001, 32),
                                   (2300, 4103, 256), (9, 8191, 1), (4, 65535, 33)])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_topk_misaligned_rows(m, n, k, dtype):
    _check(_data(m, n, dtype, n + k, "randn"), k)


def test_topk_fp16_row_beyond_2_31():
    """One fp16 row of 2^31 + 5 entries: columns above 2^31 must come back whole (64-bit offsets, 32-bit columns)."""
    n = (1 << 31) + 5
    g = torch.Generator(device="cuda").manual_seed(11)
    x = (torch.rand(1, n, device="cuda", generator=g, dtype=torch.float16) * 0.5).contiguous()   # all < 0.5
    plant = {n - 1: 3.0, (1 << 31): float("nan"), (1 << 31) + 1: 2.0, 1 << 30: 2.0, (1 << 31) - 1: 1.5, 0: 1.0,
             12345: 1.0}
    for c, val in plant.items():
        x[0, c] = val
    v, i = _T().topk(x, k=7)
    torch.cuda.synchronize()
    assert i[0].tolist() == [1 << 31, n - 1, 1 << 30, (1 << 31) + 1, (1 << 31) - 1, 0, 12345]
    vf = v[0].float().cpu().numpy()
    assert np.isnan(vf[0]) and vf[1:].tolist() == [3.0, 2.0, 2.0, 1.5, 1.0, 1.0]
    del x


def test_topk_rows_beyond_2_31_elements():
    """m * n > 2^31 with a warp per row: the row offset r * n needs 64 bits."""
    m, n = ROWS_PLAN_M + 3, (1 << 20) + 3
    x = torch.zeros(m, n, device="cuda", dtype=torch.float16)
    x[-1, n - 2] = 4.0
    x[-1, 5] = 4.0
    x[-2, 77] = -1.0
    v, i = _T().topk(x, k=3)
    torch.cuda.synchronize()
    assert i[-1].tolist() == [5, n - 2, 0] and v[-1].float().tolist() == [4.0, 4.0, 0.0]
    assert i[-2].tolist() == [0, 1, 2] and i[0].tolist() == [0, 1, 2]


# ----------------------------------------------------------------------------- rank-adversarial rows
PLANS = [(1, 1 << 20), (3, 200003), (1000, 4096), (ROWS_PLAN_M, 4096)]


@pytest.mark.parametrize("m,n", PLANS)
@pytest.mark.parametrize("k", [1, 32, 100, 1024])
def test_topk_ascending_and_descending_rows(m, n, k):
    base = torch.arange(n, device="cuda", dtype=torch.float32)          # exact up to 2^24
    x = base.repeat(m, 1).contiguous()
    _, i = _check(x, k)
    assert i[0].tolist() == list(range(n - 1, n - 1 - k, -1))           # every element passes the filter
    _, i = _check(x.flip(1).contiguous(), k)
    assert i[0].tolist() == list(range(k))


@pytest.mark.parametrize("m,n", PLANS)
@pytest.mark.parametrize("k", [1, 33, 1024])
@pytest.mark.parametrize("value", [0.0, -0.0, 1.0, float("-inf"), float("nan")])
def test_topk_constant_rows(m, n, k, value):
    x = torch.full((m, n), value, device="cuda", dtype=torch.float32)
    _, i = _check(x, k)
    assert (i == torch.arange(k, device="cuda")).all()


@pytest.mark.parametrize("m,n", [(1, 1 << 20), (3, 200003), (1, 10 ** 7)])
@pytest.mark.parametrize("k", [32, 100, 1024])
def test_topk_ties_across_slices(m, n, k):
    """Equal values spread over every slice and on both sides of every multiple of 64 columns (slice starts): the lower
    column must win across parts."""
    x = torch.randn(m, n, device="cuda").clamp_(max=4.0)
    x[:, ::997] = 5.0
    for c in range(8192, n, 8192):
        x[:, c - 3:c + 3] = 6.0
    _check(x, k)


@pytest.mark.parametrize("m,n", [(1, 1 << 20), (3, 200003), (1, 10 ** 7)])
@pytest.mark.parametrize("k", [1, 100, 1024])
def test_topk_whole_answer_in_last_slice(m, n, k):
    x = torch.randn(m, n, device="cuda")
    x[:, n - 2 * k:] += 100.0
    _, i = _check(x, k)
    assert (i >= n - 2 * k).all()


@pytest.mark.parametrize("k", [1, 32, 100, 1024])
@pytest.mark.parametrize("m", [1, 3, ROWS_PLAN_M])
@pytest.mark.parametrize("dn", [-1, 0, 1])
def test_topk_rows_of_k_minus_one_k_k_plus_one(k, m, dn):
    n = k + dn
    if n < 1:
        pytest.skip("an empty row")
    v, i = _check(_data(m, n, torch.float32, k + dn, "randn"), k)
    if dn < 0:
        assert (i[:, -1] == -1).all() and torch.isneginf(v[:, -1]).all()


@pytest.mark.parametrize("m,n", PLANS)
@pytest.mark.parametrize("k", [1, 32, 1024])
@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_topk_special_values(m, n, k, dtype):
    """+-0, NaN of both signs and payloads, +-inf among random values."""
    g = torch.Generator(device="cuda").manual_seed(n + k)
    x = torch.randn(m, n, device="cuda", generator=g).to(dtype)
    bits = torch.tensor([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFFFFFFFF], dtype=torch.int64).to(torch.int32)
    nans = bits.view(torch.float32).to("cuda")
    specials = torch.cat([nans, torch.tensor([0.0, -0.0, float("inf"), float("-inf")], device="cuda")]).to(dtype)
    sel = torch.randint(0, n, (m, max(1, n // 50)), device="cuda", generator=g)
    x.scatter_(1, sel, specials[torch.randint(0, 8, sel.shape, device="cuda", generator=g)])
    x[:, :: max(1, n // 7)] = -0.0
    x[:, 1:: max(1, n // 5)] = 0.0
    _check(x.contiguous(), k)


# ----------------------------------------------------------------------------- fp16, torch.topk, the reference
@pytest.mark.parametrize("m,n,k", [(3000, 1000, 32), (3, 1 << 20, 1024), (1000, 4096, 100)])
def test_topk_fp16_equals_fp32_on_widened_data(m, n, k):
    x16 = _data(m, n, torch.float16, 5, "randn")
    v16, i16 = _T().topk(x16, k=k)
    v32, i32 = _T().topk(x16.float(), k=k)
    assert torch.equal(i16, i32) and torch.equal(v16.float(), v32)


def _tie_free_rows(x, k):
    """Rows whose k + 1 largest values are all distinct (torch.topk's order among ties is unspecified)."""
    t = torch.topk(x.float(), min(k + 1, x.shape[1]), dim=1).values
    return (t[:, 1:] != t[:, :-1]).all(1)


@pytest.mark.parametrize("m,n,k", [(1000, 4096, 32), (10000, 4096, 32), (3, 1 << 20, 1024), (1, 10 ** 7, 100),
                                   (100, 100000, 256), (2500, 1000, 1)])
def test_topk_matches_torch_topk(m, n, k):
    x = _data(m, n, torch.float32, 9, "randn")
    v, i = _T().topk(x, k=k)
    tv, ti = torch.topk(x, k, dim=1)
    assert torch.equal(v, tv)
    rows = _tie_free_rows(x, k)
    assert rows.float().mean() > 0.5
    assert torch.equal(i[rows], ti[rows])


def test_topk_issue_example():
    T = _T()
    x = torch.randn(1000, 4096, device="cuda")
    v, i = T.topk(x, k=32)
    tv, ti = torch.topk(x, 32, dim=1)
    assert i.dtype == torch.int64 and (v[:, 1:] <= v[:, :-1]).all()
    rows = _tie_free_rows(x, 32)
    assert torch.equal(i[rows], ti[rows]) and torch.equal(v, tv)


REF_CASES = [(1, torch.float32), (1, torch.float16), (20, torch.float32), (32, torch.float16), (64, torch.float32),
             (100, torch.float32), (256, torch.float32), (512, torch.float32), (1000, torch.float32)]


@pytest.mark.parametrize("k,dtype", REF_CASES)
def test_topk_matches_reference_kernels(k, dtype):
    from oracle import ref_select as R
    tag = R.tag_of(k)
    if not R.available((tag,)):
        pytest.skip("oracle/_ref has no reference select kernels")
    x = _data(64, 5000, dtype, k, "randn")
    rv, ri = R.topk(x, k)
    v, i = _T().topk(x, k=k)
    torch.cuda.synchronize()
    assert torch.equal(v.float(), rv.float())
    rows = _tie_free_rows(x, k)
    assert torch.equal(i[rows], ri[rows])


def test_topk_python_asserts_and_unsupported():
    T = _T()
    x = torch.randn(4, 100, device="cuda")
    with pytest.raises(NotImplementedError):
        T.topk(x, k=1025)
    with pytest.raises(AssertionError):
        T.topk(x.to(torch.bfloat16), k=2)
    with pytest.raises(AssertionError):
        T.topk(x.to(torch.float64), k=2)
    with pytest.raises(AssertionError):
        T.topk(x[:, ::2], k=2)
    with pytest.raises(AssertionError):
        T.topk(x, k=2, dim=0)
    with pytest.raises(AssertionError):
        T.topk(x[None], k=2)
    v, i = T.topk(x, k=2, dim=-1)
    assert v.shape == (4, 2)
    v, i = T.topk(torch.empty(0, 100, device="cuda"), k=5)
    assert v.shape == (0, 5) and i.shape == (0, 5)
    v, i = T.topk(torch.empty(3, 0, device="cuda"), k=2)
    assert (i == -1).all() and torch.isneginf(v).all()
