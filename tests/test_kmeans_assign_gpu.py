"""GPU: tpq_kmeans_assign (the TF32 wgmma kernel for large k and d, and its dispatch), manhattan in the exact kernel,
and the public KMeans / MultiKMeans classes."""
import numpy as np
import pytest
import torch

from oracle import kmeans_oracle as K
import kmeans_ref as R

pytestmark = pytest.mark.gpu


def _int_data(shape, gen, lo=-4, hi=4):
    return torch.randint(lo, hi + 1, shape, generator=gen).float()


def _exact_int_reference(data, cent, distance="euclidean"):
    """Labels and similarities for INTEGER data, computed exactly in float64 on the GPU: every fp32 product and sum of
    the exact kernel's fmaf chain is exact for these magnitudes, so this equals kmeans_oracle.max_sim bit for bit
    (checked on a small case in test_int_reference_equals_oracle).  Ties -> lowest index."""
    x, c = data.double().cuda(), cent.double().cuda()
    ip = x.transpose(1, 2) @ c                                             # [l, n, k]
    if distance == "euclidean":
        sims = 2 * ip - (x * x).sum(1)[:, :, None] - (c * c).sum(1)[:, None, :]
    else:
        sims = ip
    best = sims.max(dim=2, keepdim=True).values
    ar = torch.arange(sims.shape[2], device=sims.device).expand_as(sims)
    labels = torch.where(sims == best, ar, sims.shape[2]).min(dim=2).values
    return best[:, :, 0].float().cpu(), labels.cpu()


def test_int_reference_equals_oracle(cuda_device):
    g = torch.Generator().manual_seed(5)
    data, cent = _int_data((2, 24, 300), g), _int_data((2, 24, 40), g)
    for dist in ("euclidean", "cosine"):
        s, lab = _exact_int_reference(data, cent, dist)
        os_, ol = K.max_sim(data.numpy(), cent.numpy(), dist)
        assert np.array_equal(lab.numpy(), ol) and np.array_equal(s.numpy(), os_)


@pytest.mark.parametrize("l", [1, 3])
@pytest.mark.parametrize("k", [257, 1000, 4096, 16384])
@pytest.mark.parametrize("d", [8, 72, 128, 256])
def test_wide_kernel_integer_data_exact(cuda_device, d, k, l):
    """Integer data in [-4, 4]: every TF32 product and sum is exact and |score| < 2^13, so labels (lowest index on
    ties) and exact maxsims match the oracle bit for bit; n straddles the 128-point tile boundaries."""
    import torchpq_b200 as T
    g = torch.Generator().manual_seed(d * 7 + k + l)
    n = {8: 124, 72: 260, 128: 128, 256: 132}[d] + (0 if k < 4096 else 128)
    data, cent = _int_data((l, d, n), g), _int_data((l, d, k), g)
    ref_s, ref_l = _exact_int_reference(data, cent)
    s, lab = T.fn.kmeans_assign(data.cuda(), cent.cuda(), "euclidean", exact_values=True)
    assert np.array_equal(lab.cpu().numpy(), ref_l.numpy())
    assert np.array_equal(s.cpu().numpy(), ref_s.numpy())
    s0, lab0 = T.fn.kmeans_assign(data.cuda(), cent.cuda(), "euclidean", exact_values=False)
    assert np.array_equal(lab0.cpu().numpy(), ref_l.numpy())
    assert torch.allclose(s0.cpu(), ref_s, rtol=1e-3, atol=0.5)       # 2 * key - |x|^2: the key's 8 low bits are the index
    cs, cl = T.fn.kmeans_assign(data.cuda(), cent.cuda(), "cosine", exact_values=True)
    ref_cs, ref_cl = _exact_int_reference(data, cent, "cosine")
    assert np.array_equal(cl.cpu().numpy(), ref_cl.numpy())
    assert np.array_equal(cs.cpu().numpy(), ref_cs.numpy())


def _tie_case(metric, sign):
    """Centroids [1, 64, 8192] with duplicates of a winning column at j, j + 256, j + 4096 (different N tiles) and
    points whose best score (the kernel's internal score) has the requested sign."""
    g = torch.Generator().manual_seed(11)
    d, k, n = 64, 8192, 256
    js = [3, 130, 200]
    if metric == "cosine":
        cent = _int_data((1, d, k), g, -1, 1)
        cent[0, 0] = {1: -1.0, 0: -1.0, -1: -2.0}[sign]                   # every centroid: this value on feature 0
        x = torch.zeros(1, d, n)
        x[0, 0] = 1.0                                                      # points e_0: score = feature 0 of the centroid
        for j in js:
            win = torch.zeros(d)
            win[0] = {1: 3.0, 0: 0.0, -1: -1.0}[sign]
            for jj in (j, j + 256, j + 4096):
                cent[0, :, jj] = win
    else:
        cent = _int_data((1, d, k), g, -4, 4)
        cent[0, 0] = 4.0                                                   # |c|^2 >= 16 for every other centroid
        x = torch.zeros(1, d, n)
        for j in js:
            win = torch.zeros(d)
            if sign != 0:
                win[1] = 1.0                                               # |c|^2 = 1: the nearest to x = 0 or to x = win
            for jj in (j, j + 256, j + 4096):
                cent[0, :, jj] = win
        if sign > 0:
            x[0, 1] = 1.0                                                  # x = win: score = <x,c> - |c|^2/2 = +1/2
        # sign == 0: x = 0, win = 0 -> score 0; sign < 0: x = 0, |win|^2 = 1 -> score -1/2
    return x, cent, js


@pytest.mark.parametrize("sign", [1, 0, -1])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
def test_wide_kernel_ties_across_tiles(cuda_device, metric, sign):
    import torchpq_b200 as T
    x, cent, js = _tie_case(metric, sign)
    ref_s, ref_l = _exact_int_reference(x, cent, metric)
    assert (ref_l == min(js)).all()
    for ev in (True, False):
        s, lab = T.fn.kmeans_assign(x.cuda(), cent.cuda(), metric, exact_values=ev)
        assert (lab.cpu() == min(js)).all(), f"{(lab.cpu() != min(js)).sum()} labels miss the lowest tied index"
    assert np.array_equal(T.fn.kmeans_assign(x.cuda(), cent.cuda(), metric)[0].cpu().numpy(), ref_s.numpy())


@pytest.mark.parametrize("l,d,n,k", [(1, 128, 1 << 20, 4096), (1, 256, 1 << 18, 16384)])
def test_wide_kernel_randn_at_scale(cuda_device, l, d, n, k):
    """randn data, centroids = data points: labels agree with the exact kernel on at least 99 % of the points (a label
    can differ only between centroids whose similarities are within TF32 rounding); where they agree the exact maxsims
    are bit-identical; where they differ the chosen centroid is worse by less than 5e-3 relative."""
    import torchpq_b200 as T
    torch.manual_seed(d)
    data = torch.randn(l, d, n, device="cuda")
    cent = data[:, :, torch.randperm(n, device="cuda")[:k]].contiguous()
    se, le = T.fn.max_sim(data, cent, exact=True)
    st, lt = T.fn.kmeans_assign(data, cent, "euclidean", exact_values=True)
    agree = lt == le
    frac = float(agree.float().mean())
    assert frac >= 0.99, frac
    assert torch.equal(st[agree], se[agree])
    if not agree.all():
        gap = ((se - st) / se.abs())[~agree]
        assert float(gap.max()) < 5e-3, float(gap.max())


def _exact(data, cent, metric):
    import torchpq_b200 as T
    return T.fn.max_sim(data, cent, metric, exact=True)


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("l,d,n,k", [(2, 12, 1000, 300), (1, 264, 512, 300), (2, 64, 130, 300), (1, 40, 1002, 2000)])
def test_dispatch_outside_range_is_exact(cuda_device, metric, l, d, n, k):
    import torchpq_b200 as T
    torch.manual_seed(d + n)
    data, cent = torch.randn(l, d, n, device="cuda"), torch.randn(l, d, k, device="cuda")
    s, lab = T.fn.kmeans_assign(data, cent, metric, exact_values=False)
    es, el = _exact(data, cent, metric)
    assert torch.equal(lab, el) and torch.equal(s, es)


def test_dispatch_misaligned_pointer_is_exact(cuda_device):
    import torchpq_b200 as T
    l, d, n, k = 1, 64, 1024, 512
    torch.manual_seed(3)
    buf = torch.randn(l * d * n + 1, device="cuda")
    data = buf[1:].view(l, d, n)                                           # 4-byte aligned, not 16
    assert data.data_ptr() % 16 != 0
    cent = torch.randn(l, d, k, device="cuda")
    s, lab = T.fn.kmeans_assign(data, cent, exact_values=False)
    es, el = _exact(data, cent, "euclidean")
    assert torch.equal(lab, el) and torch.equal(s, es)


@pytest.mark.parametrize("l,d,n,k", [(2, 64, 1024, 256), (3, 32, 700, 100), (1, 8, 128, 8)])
def test_dispatch_assign_tc_range_matches_max_sim(cuda_device, l, d, n, k):
    import torchpq_b200 as T
    torch.manual_seed(k)
    data, cent = torch.randn(l, d, n, device="cuda"), torch.randn(l, d, k, device="cuda")
    for ev in (False, True):
        s, lab = T.fn.kmeans_assign(data, cent, exact_values=ev)
        ms, ml = T.fn.max_sim(data, cent, exact=False, exact_values=ev)
        assert torch.equal(lab, ml) and torch.equal(s, ms)


def test_cosine_goes_through_tensor_cores(cuda_device):
    """In assign_tc_kernel's range cosine takes the streaming TF32 kernel: TF32-derived maxsims (the score with its
    index field) differ from the exact ones, labels on integer data do not."""
    import torchpq_b200 as T
    g = torch.Generator().manual_seed(1)
    data, cent = _int_data((2, 64, 1024), g).cuda(), _int_data((2, 64, 256), g).cuda()
    s, lab = T.fn.kmeans_assign(data, cent, "cosine", exact_values=False)
    es, el = _exact(data, cent, "cosine")
    assert torch.equal(lab, el)
    assert not torch.equal(s, es)
    assert torch.equal(T.fn.kmeans_assign(data, cent, "cosine", exact_values=True)[0], es)


def test_manhattan_exact_kernel(cuda_device):
    import torchpq_b200 as T
    g = torch.Generator().manual_seed(2)
    data, cent = _int_data((2, 20, 700), g, -2, 2), _int_data((2, 20, 300), g, -2, 2)   # many ties
    os_, ol = R.max_sim(data.numpy(), cent.numpy(), "manhattan")
    for f in (lambda a, b: T.fn.max_sim(a, b, "manhattan"), lambda a, b: T.fn.kmeans_assign(a, b, "manhattan")):
        s, lab = f(data.cuda(), cent.cuda())
        assert np.array_equal(lab.cpu().numpy(), ol) and np.array_equal(s.cpu().numpy(), os_)
    data, cent = torch.randn(1, 64, 1000, generator=g), torch.randn(1, 64, 500, generator=g)
    os_, ol = R.max_sim(data.numpy(), cent.numpy(), "manhattan")
    s, lab = T.fn.kmeans_assign(data.cuda(), cent.cuda(), "manhattan")
    assert np.array_equal(lab.cpu().numpy(), ol) and np.array_equal(s.cpu().numpy(), os_)


def test_manhattan_rejected_by_lut(cuda_device):
    import torchpq_b200 as T
    with pytest.raises(AssertionError):
        T.fn.precompute_adc(torch.randn(32, 4, device="cuda"), torch.randn(8, 4, 256, device="cuda"), "manhattan")


# ------------------------------------------------------------------ public API
def _clustered(l, d, n, k, seed):
    """Integer data in well separated clusters: centres in multiples of 8, points = centre + [-2, 2] noise, so the
    assignment is the same under TF32 and exact arithmetic and the member means are exact."""
    g = torch.Generator().manual_seed(seed)
    centres = 8 * torch.randint(-4, 5, (l, d, k), generator=g).float()
    who = torch.randint(0, k, (l, n), generator=g)
    data = torch.gather(centres, 2, who[:, None, :].expand(l, d, n)) + torch.randint(-2, 3, (l, d, n), generator=g).float()
    init = torch.stack([data[i][:, [int((who[i] == j).nonzero()[0]) for j in range(k)]] for i in range(l)])
    return data.contiguous(), init.contiguous()


@pytest.mark.parametrize("distance", ["euclidean", "cosine", "manhattan"])
@pytest.mark.parametrize("multi", [False, True])
def test_fit_from_given_centroids_equals_oracle(cuda_device, distance, multi):
    import torchpq_b200 as T
    l = 2 if multi else 1
    data, init = _clustered(l, 96, 4096, 24, seed=7)
    oc, ol, _, on = R.fit(data.numpy(), init.numpy(), 50, tol=1e-4, distance=distance)
    if multi:
        km = T.MultiKMeans(24, max_iter=50, distance=distance)
        lab = km.fit(data.cuda(), init.cuda())
        cent = km.centroids
    else:
        km = T.KMeans(24, max_iter=50, distance=distance)
        lab = km.fit(data[0].cuda(), init[0].cuda())[None]
        cent = km.centroids[None]
        assert km.centroids.shape == (96, 24)
    assert np.array_equal(lab.cpu().numpy(), ol)
    assert np.array_equal(cent.cpu().numpy(), oc)
    assert km.n_iter_ == on


@pytest.mark.parametrize("init_mode", ["random", "kmeans++"])
def test_fit_same_seed_bit_identical(cuda_device, init_mode):
    import torchpq_b200 as T
    torch.manual_seed(0)
    data = torch.randn(128, 20000, device="cuda")
    runs = []
    for _ in range(2):
        km = T.KMeans(300, max_iter=5, init_mode=init_mode, seed=3)
        runs.append((km.fit(data), km.centroids.clone()))
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


@pytest.mark.parametrize("distance", ["euclidean", "cosine", "manhattan"])
def test_predict_and_topk_equal_oracle(cuda_device, distance):
    import torchpq_b200 as T
    torch.manual_seed(1)
    km = T.MultiKMeans(50, max_iter=3, distance=distance)
    km.fit(torch.randn(2, 40, 3000, device="cuda"))
    q = torch.randn(2, 40, 500)
    if distance == "cosine":                                               # the same normalised copies, then inner products
        qc = q.cuda()
        qn = (qc / (qc.norm(dim=-2, keepdim=True) + 1e-8)).cpu().numpy()
        cn = (km.centroids / (km.centroids.norm(dim=-2, keepdim=True) + 1e-8)).cpu().numpy()
        os_, ol = K.max_sim(qn, cn, "inner")
    else:
        os_, ol = R.max_sim(q.numpy(), km.centroids.cpu().numpy(), distance)
    assert np.array_equal(km.predict(q.cuda()).cpu().numpy(), ol)
    v, i = km.topk(q.cuda(), k=1)
    assert v.shape == (2, 500, 1) and i.shape == (2, 500, 1)
    assert np.array_equal(i[..., 0].cpu().numpy(), ol) and np.array_equal(v[..., 0].cpu().numpy(), os_)
    with pytest.raises(NotImplementedError):
        km.topk(q.cuda(), k=2)
    k1 = T.KMeans(50, distance=distance)
    k1.load_state_dict({"centroids": km.centroids[0].clone()})
    v1, i1 = k1.topk(q[0].cuda(), k=1)
    assert v1.shape == (500, 1) and np.array_equal(i1[:, 0].cpu().numpy(), ol[0])
    with pytest.raises(NotImplementedError):
        k1.topk(q[0].cuda(), k=3)


@pytest.mark.parametrize("distance", ["euclidean", "cosine", "manhattan"])
def test_kmeanspp_picks_equal_oracle(cuda_device, distance):
    import torchpq_b200 as T
    torch.manual_seed(4)
    data = torch.randn(2, 16, 2000, device="cuda")
    km = T.MultiKMeans(40, distance=distance, init_mode="kmeans++", seed=9)
    cent = km.kmeanspp(data)
    first = int(torch.randint(2000, (1,), generator=torch.Generator().manual_seed(9)))
    if distance == "cosine":                                               # the same normalised copy, then inner products
        xn = (data / (data.norm(dim=-2, keepdim=True) + 1e-8)).cpu().numpy()
        oc = R.kmeanspp(xn, 40, first, "inner")
    else:
        oc = R.kmeanspp(data.cpu().numpy(), 40, first, distance)
    assert np.array_equal(cent.cpu().numpy(), oc)
    k1 = T.KMeans(40, distance=distance, init_mode="kmeans++", seed=9)
    assert torch.equal(k1.kmeanspp(data[0].contiguous()), cent[0])


def test_state_dict_round_trip(cuda_device):
    import torchpq_b200 as T
    ref_sd = {"centroids": torch.randn(2, 16, 30, device="cuda")}          # what the reference's MultiKMeans saves
    km = T.MultiKMeans(30)
    km.load_state_dict(ref_sd)
    assert torch.equal(km.centroids, ref_sd["centroids"])
    km2 = T.MultiKMeans(30)
    km2.load_state_dict(km.state_dict())
    assert torch.equal(km2.centroids, ref_sd["centroids"])
    q = torch.randn(2, 16, 100, device="cuda")
    assert torch.equal(km2.predict(q), km.predict(q))


def test_cosine_leaves_caller_tensors_unchanged(cuda_device):
    import torchpq_b200 as T
    torch.manual_seed(6)
    data = torch.randn(64, 5000, device="cuda") * 3
    init = data[:, :100].clone() * 0.7
    d0, i0 = data.clone(), init.clone()
    km = T.KMeans(100, max_iter=3, distance="cosine")
    km.fit(data, init)
    km.predict(data)
    km.get_labels(data, init)
    T.KMeans(100, distance="cosine", init_mode="kmeans++").kmeanspp(data)
    assert torch.equal(data, d0) and torch.equal(init, i0)
