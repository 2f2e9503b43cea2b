"""GPU parity of tpq_max_sim / tpq_compute_centroids / tpq_pq_decode against the oracle and against the
reference's own kernels (oracle/_ref)."""
import numpy as np
import pytest
import torch

from oracle import kmeans_oracle as K, ref_kernels as R

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("l,d,n,k", [(3, 2, 1000, 256), (2, 16, 700, 40), (1, 64, 513, 256), (4, 8, 300, 300)])
@pytest.mark.parametrize("distance", ["euclidean", "cosine"])
def test_max_sim(cuda_device, l, d, n, k, distance):
    import torchpq_b200 as T
    torch.manual_seed(l * 7 + d)
    data, cent = torch.randn(l, d, n), torch.randn(l, d, k)
    osim, olab = K.max_sim(data.numpy(), cent.numpy(), distance)
    sim, lab = T.fn.max_sim(data.cuda(), cent.cuda(), distance)
    sim, lab = sim.cpu().numpy(), lab.cpu().numpy()
    assert np.array_equal(sim, osim)                       # same fmaf chain -> bit-identical
    assert np.array_equal(lab, olab)
    if R.aux_available():                                  # the reference's own max_sim_tn kernel
        rv, ri = R.max_sim_tn(data.cuda(), cent.cuda(), "euclidean" if distance == "euclidean" else "inner", dim=2)
        assert np.array_equal(rv.cpu().numpy(), osim)
        # the reference's label write races across its 128-wide centroid tiles (max_sim.cu:173-178):
        # compare where the winner is unique
        rl = ri.cpu().numpy()
        assert (rl == olab).mean() > (0.999 if k <= 128 else 0.99)   # k > 128: two racing tiles per row


def test_max_sim_integer_ties_lowest_index(cuda_device):
    import torchpq_b200 as T
    rng = np.random.default_rng(0)
    data = torch.from_numpy(rng.integers(-2, 3, (2, 4, 500)).astype(np.float32))
    cent = torch.from_numpy(rng.integers(-2, 3, (2, 4, 300)).astype(np.float32))   # many duplicate centroids
    osim, olab = K.max_sim(data.numpy(), cent.numpy())
    sim, lab = T.fn.max_sim(data.cuda(), cent.cuda())
    assert np.array_equal(lab.cpu().numpy(), olab) and np.array_equal(sim.cpu().numpy(), osim)


@pytest.mark.parametrize("l,d,n,k", [(3, 2, 5000, 256), (2, 16, 3000, 16), (1, 130, 20000, 256), (2, 8, 100, 1000),
                                     (1, 40, 30000, 1500), (2, 3, 5000, 4096)])
def test_compute_centroids(cuda_device, l, d, n, k):
    import torchpq_b200 as T
    torch.manual_seed(d)
    data = torch.randn(l, d, n)
    labels = torch.randint(0, max(1, k - 3), (l, n))       # the last clusters stay empty -> 0
    oc = K.compute_centroids(data.numpy(), labels.numpy(), k)
    c = T.fn.compute_centroids(data.cuda(), labels.cuda(), k).cpu().numpy()
    assert np.allclose(c, oc, rtol=1e-5, atol=1e-6)
    assert np.array_equal(c, K.compute_centroids_seq(data.numpy(), labels.numpy(), k))   # sums in point order
    assert np.array_equal(T.fn.compute_centroids(data.cuda(), labels.cuda(), k).cpu().numpy(), c)   # run to run: bit for bit
    assert (c[:, :, k - 3:] == 0).all()
    if R.aux_available() and k in (16, 256):
        rc = R.compute_centroids(data.cuda(), labels.cuda(), k).cpu().numpy()
        assert np.allclose(rc, oc, rtol=1e-5, atol=1e-6)


def _centroids_bitexact(data, labels, k):
    """GPU update == compute_centroids_seq bit for bit (fp32 sums in point order, one rounded division)."""
    import torchpq_b200 as T
    c = T.fn.compute_centroids(data.cuda(), labels.cuda(), k).cpu().numpy()
    oc = K.compute_centroids_seq(data.numpy(), labels.numpy(), k)
    assert c.shape == oc.shape
    bad = np.argwhere(c.view(np.uint32) != oc.view(np.uint32))
    assert len(bad) == 0, f"{len(bad)} centroid entries differ, first [l, e, j] = {bad[:5].tolist()}"


# k = 256 / 257, 512 / 513, 1024 / 1025: one / two / four clusters per thread of the streaming kernel, then the
# owner kernel; d = 16 / 17 and 32 / 33: the streaming kernel's 16-feature group and the owner kernel's 32-feature block
@pytest.mark.parametrize("k", [1, 255, 256, 257, 512, 513, 1024, 1025, 4099])
@pytest.mark.parametrize("d", [1, 3, 16, 17, 32, 33, 130])
def test_compute_centroids_bitexact_shapes(cuda_device, k, d):
    g = torch.Generator().manual_seed(k * 1000 + d)
    n = 4097                                                       # one point past the streaming kernel's 4096-point tile
    data = torch.randn(2, d, n, generator=g)
    labels = torch.randint(0, k, (2, n), generator=g)
    _centroids_bitexact(data, labels, k)


@pytest.mark.parametrize("n", [0, 1, 4095, 4096, 4097, 3 * 4096 + 5])
@pytest.mark.parametrize("k", [256, 1025])
def test_compute_centroids_bitexact_point_counts(cuda_device, n, k):
    g = torch.Generator().manual_seed(n + k)
    data = torch.randn(2, 17, n, generator=g)
    labels = torch.randint(0, k, (2, n), generator=g)
    _centroids_bitexact(data, labels, k)


@pytest.mark.parametrize("skew", ["all_first", "all_last", "sorted", "reverse_sorted"])
@pytest.mark.parametrize("k", [257, 1025])
def test_compute_centroids_bitexact_skewed_labels(cuda_device, skew, k):
    """Long member lists cross tiles (4096 points in the streaming kernel, 1024 in the owner kernel) and every sum
    must still be taken in point order."""
    g = torch.Generator().manual_seed(len(skew) + k)
    n = 3 * 4096 + 5
    data = torch.randn(2, 33, n, generator=g)
    labels = torch.randint(0, k, (2, n), generator=g)
    if skew == "all_first":
        labels[:] = 0
    elif skew == "all_last":
        labels[:] = k - 1
    elif skew == "sorted":
        labels = labels.sort(dim=1).values
    else:
        labels = labels.sort(dim=1, descending=True).values
    _centroids_bitexact(data, labels, k)


@pytest.mark.parametrize("k", [256, 513, 4099])
def test_compute_centroids_ignores_out_of_range_labels(cuda_device, k):
    """Labels -1, k and 2^40 belong to no cluster (compute_centroids.cu:61-64): they add nothing and count nothing."""
    g = torch.Generator().manual_seed(k)
    n = 6000
    data = torch.randn(2, 20, n, generator=g)
    labels = torch.randint(0, k, (2, n), generator=g)
    which = torch.randint(0, 4, (2, n), generator=g)
    labels[which == 1] = -1
    labels[which == 2] = k
    labels[which == 3] = 2 ** 40
    _centroids_bitexact(data, labels, k)
    import torchpq_b200 as T
    c = T.fn.compute_centroids(data.cuda(), labels.cuda(), k).cpu().numpy()
    assert np.allclose(c, K.compute_centroids(data.numpy(), labels.numpy(), k), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("M,dsub,n", [(8, 4, 1000), (64, 2, 4096), (3, 8, 17), (120, 8, 333)])
def test_pq_decode(cuda_device, M, dsub, n):
    import torchpq_b200 as T
    torch.manual_seed(M)
    cb = torch.randn(M, dsub, 256)
    code = torch.randint(0, 256, (M, n), dtype=torch.uint8)
    o = K.pq_decode(cb.numpy(), code.numpy())
    g = T.fn.pq_decode(cb.cuda(), code.cuda()).cpu().numpy()
    assert np.array_equal(g, o)
    if R.aux_available():
        assert np.array_equal(R.pq_decode(cb.cuda(), code.cuda()).cpu().numpy(), o)


def _exact_sim_of(data, cent, labels):
    """fp32 fmaf-chain similarity of every point to the centroid `labels` picks (oracle arithmetic)."""
    l, d, n = data.shape
    out = np.zeros((l, n), np.float32)
    for li in range(l):
        c = cent[li][:, labels[li]]                           # [d, n]
        acc = np.zeros(n, np.float32)
        for e in range(d):
            dif = (data[li, e] - c[e]).astype(np.float32)
            acc = K._fma32(-dif, dif, acc)
        out[li] = acc
    return out


@pytest.mark.parametrize("l,d,n,k", [(3, 64, 4096, 256), (2, 16, 1000, 40), (1, 8, 132, 256), (5, 32, 300, 100), (64, 64, 2048, 256),
                                     (2, 40, 1000, 160), (1, 24, 640, 192), (3, 56, 2000, 64)])
def test_max_sim_tensor_core(cuda_device, l, d, n, k):
    """TF32 wgmma assignment: labels equal the exact ones except between near-equidistant centroids, and the
    reported similarity is the EXACT fp32 value of the chosen centroid."""
    import torchpq_b200 as T
    torch.manual_seed(l + d + k)
    data, cent = torch.randn(l, d, n), torch.randn(l, d, k)
    osim, olab = K.max_sim(data.numpy(), cent.numpy())
    sim, lab = T.fn.max_sim(data.cuda(), cent.cuda(), exact=False)
    sim_fast, lab_fast = T.fn.max_sim(data.cuda(), cent.cuda(), exact=False, exact_values=False)
    torch.cuda.synchronize()
    assert torch.equal(lab, lab_fast)                                  # same labels, TF32-derived values
    assert torch.allclose(sim_fast, sim, rtol=5e-3, atol=5e-2)
    sim, lab = sim.cpu().numpy(), lab.cpu().numpy()
    assert lab.min() >= 0 and lab.max() < k
    agree = (lab == olab).mean()
    assert agree >= 0.985, f"label agreement {agree}"
    assert np.array_equal(sim, _exact_sim_of(data.numpy(), cent.numpy(), lab))
    # where the label differs the chosen centroid is (almost) as close as the best one
    bad = lab != olab
    if bad.any():
        rel = (osim[bad] - sim[bad]) / np.abs(osim[bad])
        assert rel.min() >= 0 and rel.max() < 5e-3


def _int_tensor(rng, shape, lo=-8, hi=8):
    return torch.from_numpy(rng.integers(lo, hi + 1, shape).astype(np.float32))


def _tc_matches_oracle_on_exact_data(data, cent):
    """Integer data and centroids in [-8, 8], d <= 64: every product, |c|^2/2 (one TF32 (hi, lo) pair) and every partial
    sum of the score <x,c> - |c|^2/2 is an integer or half-integer below 2^13, exact in TF32 operands and in the fp32
    accumulator, and the 8 masked mantissa bits still separate half-integers.  So the TF32 kernel must return exactly
    the oracle's labels (lowest index on ties) and, with exact_values, exactly its maxsims; with TF32-derived values
    the only error left is the index field in the key: |2 key - 2 score| < 2 * 2^-15 |score|, plus the final rounding."""
    import torchpq_b200 as T
    osim, olab = K.max_sim(data.numpy(), cent.numpy())
    sim, lab = T.fn.max_sim(data.cuda(), cent.cuda(), exact=False, exact_values=True)
    sim_f, lab_f = T.fn.max_sim(data.cuda(), cent.cuda(), exact=False, exact_values=False)
    sim, lab, sim_f, lab_f = (t.cpu().numpy() for t in (sim, lab, sim_f, lab_f))
    x2 = (data.numpy().astype(np.float64) ** 2).sum(axis=1)
    score = (osim.astype(np.float64) + x2) / 2                     # exact: <x,c> - |c|^2/2 of the best centroid
    bad = lab != olab
    assert not bad.any(), (f"{bad.sum()} of {bad.size} labels differ (best score < 0: {(bad & (score < 0)).sum()}, "
                           f"= 0: {(bad & (score == 0)).sum()}, > 0: {(bad & (score > 0)).sum()}); first [l, i, got, "
                           f"want] = {[[*ix, lab[tuple(ix)], olab[tuple(ix)]] for ix in np.argwhere(bad)[:4].tolist()]}")
    assert np.array_equal(sim, osim)
    assert np.array_equal(lab_f, olab)
    err = np.abs(sim_f.astype(np.float64) - osim.astype(np.float64))
    assert (err <= 2.0 ** -14 * np.abs(score) + np.spacing(np.abs(osim))).all(), err.max()
    return osim, olab


@pytest.mark.parametrize("k", [8, 60, 64, 100, 128, 132, 192, 196, 252, 256])
@pytest.mark.parametrize("d", [8, 16, 24, 32, 40, 48, 56, 64])
def test_max_sim_tensor_core_exact_data(cuda_device, d, k):
    """Every (d / 8, ceil(k / 64)) instantiation of assign_tc_kernel, k a multiple of 64 and not."""
    rng = np.random.default_rng(d * 1000 + k)
    _tc_matches_oracle_on_exact_data(_int_tensor(rng, (2, d, 520)), _int_tensor(rng, (2, d, k)))


@pytest.mark.parametrize("k,groups", [(100, [(3, 10), (20, 50, 51), (15, 67), (5, 74), (40, 99)]),
                                      (256, [(3, 10), (12, 67), (5, 74), (6, 130, 131), (64, 200), (1, 65, 129, 193),
                                             (150, 255)])])
@pytest.mark.parametrize("d", [16, 64])
def test_max_sim_tensor_core_ties_lowest_index(cuda_device, d, k, groups):
    """Duplicated centroid columns inside a 64-column chunk and across chunks; rows drawn near them with a positive
    best score (x near c), a zero one (x = c / 2) and a negative one (x pulled towards the origin: farther from its
    nearest centroid than from 0).  The lowest column of each group must win, as in the exact kernel, for every sign."""
    rng = np.random.default_rng(d + k)
    l, n = 2, 1024
    # every centroid far from the origin (entries +-5..8), so the one a row is drawn around stays its nearest even when
    # the row is pulled towards the origin; duplicated columns get even entries, so that c / 2 is an integer
    cent = (rng.integers(5, 9, (l, d, k)) * rng.choice([-1, 1], (l, d, k))).astype(np.float32)
    for gr in groups:
        cent[:, :, list(gr)] = (2 * (cent[:, :, gr[0]] // 2))[:, :, None]
    data = np.zeros((l, d, n), np.float32)
    kind = np.arange(n) % 3                                         # 0: positive, 1: zero, 2: negative best score
    for li in range(l):
        for i in range(n):
            c = cent[li, :, groups[i % len(groups)][0]]
            if kind[i] == 0:
                data[li, :, i] = c + rng.integers(-1, 2, d)
            elif kind[i] == 1:
                data[li, :, i] = c / 2
            else:
                data[li, :, i] = np.trunc(c * rng.uniform(0.25, 0.45))
    osim, olab = _tc_matches_oracle_on_exact_data(torch.from_numpy(data), torch.from_numpy(cent))
    # the rows do land on the duplicated columns, with each sign of the best score
    x2 = (data.astype(np.float64) ** 2).sum(axis=1)
    score = (osim.astype(np.float64) + x2) / 2
    firsts = {gr[0] for gr in groups}
    on_dup = np.isin(olab, list(firsts))
    for sel in (score > 0, score == 0, score < 0):
        assert (on_dup & sel).sum() >= n // 8, (on_dup & sel).sum()


@pytest.mark.parametrize("sign", [-1, 1])
@pytest.mark.parametrize("d", [8, 64])
def test_max_sim_tensor_core_signed_zero_ties(cuda_device, d, sign):
    """The packed arg-max key ranks -0 below +0, so the kernel relies on its accumulator never holding -0.  The worst
    case for that: a zero centroid whose every product with x is -0 (x < 0 against +0 entries, or x > 0 against -0
    entries; then -|c|^2/2 = -0 as well), tied at score 0 with the centroid 2x placed at a HIGHER column, every other
    centroid far away.  If the zero centroid's score came out as -0, the higher column would win."""
    rng = np.random.default_rng(d * 10 + sign)
    l, n, k = 64, 128, 256
    x = (sign * rng.integers(1, 5, (l, d))).astype(np.float32)             # no zero entry: every product is -0
    cent = np.repeat((-8.0 * np.sign(x))[:, :, None], k, axis=2).astype(np.float32)   # far: opposite orthant
    cent += rng.integers(0, 2, (l, d, k)) * np.sign(x)[:, :, None]           # (distinct far centroids)
    z = rng.integers(0, k - 1, l)
    b = np.array([rng.integers(zi + 1, k) for zi in z])
    for li in range(l):
        cent[li, :, z[li]] = -0.0 if sign > 0 else 0.0
        cent[li, :, b[li]] = 2 * x[li]
    assert (np.signbit(cent[np.arange(l), :, z]) == (sign > 0)).all()
    data = np.repeat(x[:, :, None], n, axis=2)
    osim, olab = _tc_matches_oracle_on_exact_data(torch.from_numpy(data), torch.from_numpy(cent))
    assert (olab == z[:, None]).all() and (osim == -(x.astype(np.float64) ** 2).sum(axis=1)[:, None]).all()


@pytest.mark.parametrize("n", [128, 132, 160, 196])
def test_max_sim_tensor_core_last_tile(cuda_device, n):
    """n at the eligibility limit: the last 64-point tile partly (or, past the last 32-point box, wholly) out of
    bounds, zero-filled by TMA and not stored."""
    rng = np.random.default_rng(n)
    _tc_matches_oracle_on_exact_data(_int_tensor(rng, (3, 32, n)), _int_tensor(rng, (3, 32, 100)))


@pytest.mark.parametrize("l,n", [(500, 128), (301, 192), (1, 128)])
def test_max_sim_tensor_core_many_kmeans_per_cta(cuda_device, l, n):
    """Many k-means of one to three tiles each in one CTA: the centroid set is reloaded between segments and the two
    consumer warpgroups alternate tiles across them.  l = 1, n = 128: fewer tiles than SMs."""
    rng = np.random.default_rng(l + n)
    _tc_matches_oracle_on_exact_data(_int_tensor(rng, (l, 24, n)), _int_tensor(rng, (l, 24, 100)))


def _storage_offset(t):
    """The same values at a 4-byte storage offset (contiguous, not 16-byte aligned)."""
    buf = torch.empty(t.numel() + 1, device="cuda")
    out = buf[1:].view(t.shape)
    out.copy_(t)
    return out


@pytest.mark.parametrize("case", ["n124", "n130", "d12", "d72", "k6", "k258", "k260", "cosine", "data_offset",
                                  "cent_offset", "eligible"])
def test_max_sim_tensor_core_dispatch(cuda_device, case):
    """Shapes the tensor-core kernel does not take run the exact kernel: exact=False returns the exact kernel's values
    bit for bit, even with TF32-derived values requested.  The eligible control shows the comparison would notice."""
    import torchpq_b200 as T
    shape = {"l": 2, "d": 16, "n": 256, "k": 64}                  # eligible; each case moves one thing out of range
    if case[0] in "ndk" and case[1:].isdigit():
        shape[case[0]] = int(case[1:])
    l, d, n, k = shape["l"], shape["d"], shape["n"], shape["k"]
    distance = "cosine" if case == "cosine" else "euclidean"
    g = torch.Generator().manual_seed(len(case))
    data, cent = torch.randn(l, d, n, generator=g).cuda(), torch.randn(l, d, k, generator=g).cuda()
    esim, elab = T.fn.max_sim(data, cent, distance, exact=True)
    if case == "data_offset":
        data = _storage_offset(data)
    if case == "cent_offset":
        cent = _storage_offset(cent)
    sim, lab = T.fn.max_sim(data, cent, distance, exact=False, exact_values=False)
    if case == "eligible":
        assert not torch.equal(sim, esim)                          # TF32-derived values: the tensor-core kernel ran
    else:
        assert torch.equal(sim, esim) and torch.equal(lab, elab)


def test_max_sim_tensor_core_c5_scale(cuda_device):
    """The benchmark's C5 shape at l = 2 (d = 64, k = 256, n = 2^20, randn, centroids = data points) against the exact
    GPU kernel (pinned to the oracle by the tests above): same labels except between near-equidistant centroids, exact
    similarities wherever the label agrees."""
    import torchpq_b200 as T
    g = torch.Generator().manual_seed(5)
    data = torch.randn(2, 64, 1 << 20, generator=g).cuda()
    cent = data[:, :, :256].contiguous()
    esim, elab = T.fn.max_sim(data, cent, exact=True)
    sim, lab = T.fn.max_sim(data, cent, exact=False, exact_values=True)
    lab_f = T.fn.max_sim(data, cent, exact=False, exact_values=False)[1]
    assert torch.equal(lab, lab_f)
    same = lab == elab
    agree = same.float().mean().item()
    assert agree >= 0.985, agree
    assert torch.equal(sim[same], esim[same])
    rel = ((esim - sim) / esim.abs())[~same]
    if rel.numel():
        assert rel.min().item() >= 0 and rel.max().item() < 5e-3, (rel.min().item(), rel.max().item())


def test_fit_matches_oracle_loop(cuda_device):
    """build.fit = the reference's MultiKMeans.fit loop (clustering/MultiKMeans.py:415-453): from identical initial
    centroids on integer-valued data (sums of members are exact in fp32, so every Lloyd step is order-independent)
    the exact-assignment GPU loop and the CPU restatement agree bit for bit: centroids, labels, iteration count."""
    from torchpq_b200 import build
    rng = np.random.default_rng(3)
    data = torch.from_numpy(rng.integers(-8, 9, (3, 4, 3000)).astype(np.float32))
    c0 = data[:, :, rng.choice(3000, 16, replace=False)].clone()
    ocent, olab, oinertia, oit = K.fit(data.numpy(), c0.numpy(), max_iter=12, tol=1e-4)
    cent, lab, inertia, it = build.fit(data.cuda().contiguous(), 16, max_iter=12, tol=1e-4, centroids=c0.cuda(), exact=True)
    assert it == oit
    assert np.array_equal(lab.cpu().numpy(), olab)
    assert np.allclose(cent.cpu().numpy(), ocent, rtol=1e-6, atol=1e-6)
    assert abs(inertia - oinertia) <= 1e-4 * max(1.0, abs(oinertia))


def test_fit_stops_on_sum_of_squares_and_picks_best_redo(cuda_device):
    """error = sum((new - old)^2) <= tol stops the loop (not a mean shift); with n_redo > 1 the lowest-inertia run wins."""
    from torchpq_b200 import build
    torch.manual_seed(0)
    centers = torch.randn(1, 8, 4) * 20
    data = (centers[:, :, torch.randint(0, 4, (2000,))] + torch.randn(1, 8, 2000)).cuda().contiguous()
    cent, lab, inertia, it = build.fit(data, 4, max_iter=50, tol=1e-4, n_redo=1, seed=1)
    assert it < 50                                                   # converged by the tolerance, not by max_iter
    runs = [build.fit(data, 4, max_iter=50, tol=1e-4, n_redo=1, seed=s)[2] for s in (5, 6, 7)]
    best = build.fit(data, 4, max_iter=50, tol=1e-4, n_redo=3, seed=5)[2]
    assert abs(best - min(runs)) <= 1e-3 * abs(min(runs))
