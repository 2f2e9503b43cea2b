"""GPU parity: the CUDA path (through the C ABI) against the CPU oracle on identical state."""
import numpy as np
import pytest
import torch

from oracle import ivfpq_oracle as O, build_state as B
from helpers import make_index, tie_free_rows, assert_close_results

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,d,C,n,k,n_probe", [
    (8, 32, 16, 3000, 10, 4),
    (64, 128, 32, 6000, 100, 8),
    (32, 64, 8, 2000, 1, 3),
    (120, 240, 16, 4000, 100, 16),
])
@pytest.mark.parametrize("smart", [False, True])
def test_integer_kat_exact(cuda_device, M, d, C, n, k, n_probe, smart):
    """Integer-valued state: every score is exact, so values must be identical and ids identical
    on every query that is tie-free at the k-th boundary."""
    st, queries = B.integer_state(d, M, C, n, seed=M + k)
    st.n_probe, st.use_smart_probing = n_probe, smart
    x = queries(64)
    ov, oi, oa = O.search(st, x, k=k + 1, return_address=True)
    ix = make_index(st)
    v, i, a = ix.search(x.cuda(), k=k, return_address=True)
    v, i, a = v.cpu().numpy(), i.cpu().numpy(), a.cpu().numpy()
    assert np.array_equal(v, ov[:, :k])                       # values are exact whatever the tie order
    ok = tie_free_rows(ov, k)                                  # k-th and (k+1)-th scores differ
    assert np.array_equal(np.sort(i[ok], axis=1), np.sort(oi[ok, :k], axis=1))   # the id SET is tie-rule independent
    # with the shared total order (score desc, address asc) even tied rows agree
    assert np.array_equal(a, oa[:, :k])


@pytest.mark.parametrize("distance,M,d", [("euclidean", 8, 128), ("euclidean", 64, 128), ("cosine", 24, 96)])
def test_randn_close(cuda_device, distance, M, d):
    torch.manual_seed(7)
    base = torch.randn(d, 8000)
    st = B.build_state(base, M, 32, distance=distance, vq_iters=3, pq_iters=2, n_train=4000)
    st.n_probe = 8
    x = torch.randn(d, 100)
    for smart in (False, True):
        st.use_smart_probing = smart
        ov, oi = O.search(st, x, k=50)
        ix = make_index(st)
        v, i = ix.search(x.cuda(), k=50)
        assert_close_results(v.cpu().numpy(), i.cpu().numpy(), ov, oi, rtol=1e-3, min_overlap=0.995)


def test_fewer_than_k_and_empty_cells(cuda_device):
    st, queries = B.integer_state(32, 8, 64, 40, seed=3)     # 40 vectors in 64 cells: most cells empty
    st.n_probe, st.use_smart_probing = 8, False
    x = queries(16)
    ov, oi, oa = O.search(st, x, k=20, return_address=True)
    ix = make_index(st)
    v, i, a = ix.search(x.cuda(), k=20, return_address=True)
    assert np.array_equal(v.cpu().numpy(), ov)
    assert np.array_equal(a.cpu().numpy(), oa)
    assert np.array_equal(i.cpu().numpy(), oi)
    assert (oi == -1).any() and np.isinf(ov).any()


def test_is_empty_holes(cuda_device):
    st, queries = B.integer_state(32, 8, 8, 1000, seed=5)
    rng = np.random.default_rng(0)
    live = np.flatnonzero(st.is_empty == 0)
    holes = rng.choice(live, 200, replace=False)
    st.is_empty[holes] = 1
    st.n_probe, st.use_smart_probing = 4, False
    x = queries(32)
    ov, oi, oa = O.search(st, x, k=10, return_address=True)
    ix = make_index(st)
    v, i, a = ix.search(x.cuda(), k=10, return_address=True)
    assert np.array_equal(a.cpu().numpy(), oa) and np.array_equal(v.cpu().numpy(), ov)
    assert not np.isin(a.cpu().numpy(), holes).any()


@pytest.mark.parametrize("k", [1, 10, 100, 256, 1024])
def test_k_sweep(cuda_device, k):
    st, queries = B.integer_state(64, 16, 8, 5000, seed=11, lo=-8, hi=9)
    st.n_probe, st.use_smart_probing = 6, False
    x = queries(8)
    ov, oi, oa = O.search(st, x, k=k, return_address=True)
    ix = make_index(st)
    v, i, a = ix.search(x.cuda(), k=k, return_address=True)
    assert np.array_equal(v.cpu().numpy(), ov)
    assert np.array_equal(a.cpu().numpy(), oa)


def test_reference_layout_op(cuda_device):
    """fn.IVFPQTopk.topk drop-in (reference storage layout, reference LUT layout, reference sum order):
    values are bit-identical to the oracle's m-ascending fp32 sums even on randn data."""
    import torchpq_b200 as T
    torch.manual_seed(3)
    base = torch.randn(64, 5000)
    st = B.build_state(base, 16, 16, vq_iters=2, pq_iters=2)
    st.n_probe, st.use_smart_probing = 5, True
    x = torch.randn(64, 40)
    xx, sims, cells, npl = O.coarse_probe(st, x)
    lut = O.precompute_adc(xx, torch.from_numpy(st.pq_codebook), st.distance)
    cs, cz = st.cell_start[cells.numpy()], st.cell_size[cells.numpy()]
    ov, oa = O.ivfpq_topk(st.storage, lut.numpy(), st.is_empty, cs, cz, npl.numpy(), 30)
    op = T.fn.IVFPQTopk(16)
    v, a = op.topk(torch.from_numpy(st.storage).cuda(), lut.cuda(), torch.from_numpy(cs).cuda(),
                   torch.from_numpy(cz).cuda(), torch.from_numpy(st.is_empty).cuda(), npl.cuda(), k=30)
    assert np.array_equal(v.cpu().numpy(), ov)
    assert np.array_equal(a.cpu().numpy(), oa)


def test_lut_and_coarse(cuda_device):
    """Against the reference's torch arithmetic, to a tolerance; the bit-exact counterpart, against restatements of
    these kernels' own arithmetic, is tests/test_fp32_exact_gpu.py."""
    import torchpq_b200 as T
    torch.manual_seed(5)
    for distance in ("euclidean", "cosine"):
        base = torch.randn(96, 3000)
        st = B.build_state(base, 24, 64, distance=distance, vq_iters=2, pq_iters=1)
        st.n_probe = 16
        x = torch.randn(96, 50)
        xx, sims, cells, npl = O.coarse_probe(st, x)
        xg = x.cuda()
        if distance == "cosine":
            xg = T.fn.normalize(xg)
            assert torch.allclose(xg.cpu(), xx, rtol=1e-5, atol=1e-7)
        lut = T.fn.precompute_adc(xg, torch.from_numpy(st.pq_codebook).cuda(), distance).cpu()
        olut = O.precompute_adc(xx, torch.from_numpy(st.pq_codebook), distance)
        assert torch.allclose(lut, olut, rtol=1e-4, atol=1e-4)
        gs, gc, gn = T.fn.coarse_probe(xg, torch.from_numpy(st.vq_codebook).cuda(), 16, True, 30.0)
        assert torch.allclose(gs.cpu(), sims, rtol=1e-4, atol=1e-3)
        assert (gc.cpu() == cells).float().mean() > 0.99
        assert (gn.cpu() == npl).float().mean() > 0.98


def test_sharded_scan_equals_unsharded(cuda_device):
    """Cell-sharded search (dist.py) without NCCL: run every shard on this GPU, stack the packed keys the
    way the all-gather would, merge with tpq_merge_topk -> bit-identical to the unsharded search."""
    import torchpq_b200 as T
    torch.manual_seed(9)
    st = B.build_state(torch.randn(64, 6000), 16, 32, vq_iters=2, pq_iters=1)
    st.n_probe = 8
    x = torch.randn(64, 300).cuda()
    ix = make_index(st)
    v0, i0, a0 = ix.search(x, k=40, return_address=True)
    for world in (2, 3, 8):
        parts = []
        for r in range(world):
            ix.set_shard(r, world)
            parts.append(ix.search(x, k=40, return_keys=True)[2])
        v, i, a = T.fn.merge_topk(torch.stack(parts).contiguous(), ix._address2id)
        assert torch.equal(v, v0) and torch.equal(a, a0) and torch.equal(i, i0)
    ix.set_shard(0, 1)


def test_small_batch_slices(cuda_device):
    """nq small -> each query is split over several CTAs (slices) and merged: same answer as the oracle."""
    st, queries = B.integer_state(64, 16, 32, 20000, seed=21, lo=-6, hi=7)
    st.n_probe, st.use_smart_probing = 16, False
    ix = make_index(st)
    for nq in (1, 3, 40):
        x = queries(nq, qseed=nq)
        ov, oi, oa = O.search(st, x, k=64, return_address=True)
        v, i, a = ix.search(x.cuda(), k=64, return_address=True)
        assert np.array_equal(v.cpu().numpy(), ov) and np.array_equal(a.cpu().numpy(), oa)


def test_build_side_matches_oracle_placement(cuda_device):
    """container_add on the GPU (torch ops, build.py) places items exactly where the oracle's restatement of
    CellContainer.add does, including an expansion and a second add."""
    from torchpq_b200 import build
    import torchpq_b200 as T
    rng = np.random.default_rng(4)
    st = O.empty_state(32, 8, 16, 8)
    ix = T.IVFPQIndex(32, 8, 16, initial_size=8, device="cuda:0")
    for n in (700, 300):
        codes = rng.integers(0, 256, (8, n)).astype(np.uint8)
        cells = rng.integers(0, 16, n)
        _, adr = O.container_add(st, codes, cells)
        _, gadr = build.container_add(ix, torch.from_numpy(codes).cuda(), torch.from_numpy(cells).cuda(), return_address=True)
        assert np.array_equal(gadr.cpu().numpy(), adr)
    for name, ref in (("_storage", st.storage), ("_is_empty", st.is_empty), ("_cell_start", st.cell_start),
                      ("_cell_size", st.cell_size), ("_cell_capacity", st.cell_capacity), ("_address2id", st.address2id)):
        assert np.array_equal(getattr(ix, name).cpu().numpy(), ref), name


def test_train_add_search_end_to_end(cuda_device):
    """train -> add -> search through the public API only; recall equals the oracle's on the same state."""
    import torchpq_b200 as T
    torch.manual_seed(1)
    base = torch.randn(32, 20000, device="cuda")
    ix = T.IVFPQIndex(32, 16, 64, initial_size=64, device="cuda:0")
    ix.train(base[:, :8000].contiguous())
    ids = ix.add(base)
    assert ids.shape[0] == 20000 and ix.n_items == 20000
    ix.n_probe = 16
    x = torch.randn(32, 200, device="cuda")
    v, i = ix.search(x, k=10)
    import bench
    st = bench.to_oracle_state(ix)
    ov, oi = O.search(st, x.cpu(), k=10)
    assert_close_results(v.cpu().numpy(), i.cpu().numpy(), ov, oi, rtol=1e-3, min_overlap=0.995)
    truth = O.exact_topk(base.cpu(), x.cpu(), 10, "euclidean").numpy()
    assert abs(O.recall_at_k(i.cpu().numpy(), truth) - O.recall_at_k(oi, truth)) <= 1e-3


def test_remove_then_search_and_refill(cuda_device):
    """remove() makes holes the scan skips; results equal the oracle on the same (holed) state; the next add
    refills the holes first (CellContainer.add placement rule)."""
    import torchpq_b200 as T
    import bench
    torch.manual_seed(2)
    base = torch.randn(32, 6000, device="cuda")
    ix = T.IVFPQIndex(32, 8, 16, initial_size=512, device="cuda:0")
    ix.train(base[:, :3000].contiguous())
    ids = ix.add(base)
    gone = ids[::7]
    adr_gone = ix.get_address_by_id(gone)
    ix.remove(ids=gone)
    assert ix.n_items == 6000 - gone.shape[0]
    assert (ix.get_address_by_id(gone) == -1).all()
    ix.n_probe = 8
    x = torch.randn(32, 64, device="cuda")
    v, i = ix.search(x, k=20)
    assert not torch.isin(i, gone).any()
    ov, oi = O.search(bench.to_oracle_state(ix), x.cpu(), k=20)
    assert_close_results(v.cpu().numpy(), i.cpu().numpy(), ov, oi, rtol=1e-3, min_overlap=0.995)
    new_ids, new_adr = ix.add(base[:, :200].contiguous(), return_address=True)
    assert torch.isin(new_adr, adr_gone).all()            # holes are reused before fresh slots


@pytest.mark.parametrize("M,d", [(8, 64), (12, 36), (16, 16)])
def test_staged_lut_and_odd_subvector_sizes(cuda_device, M, d):
    """d/M = 8, 3, 1: the LUT is staged through HBM (8, 3) or built in the scan CTA (1); all must match the oracle."""
    st, queries = B.integer_state(d, M, 8, 3000, seed=d, lo=-4, hi=5)
    st.n_probe, st.use_smart_probing = 5, True
    x = queries(40)
    ov, oi, oa = O.search(st, x, k=33, return_address=True)
    ix = make_index(st)
    v, i, a = ix.search(x.cuda(), k=33, return_address=True)
    assert np.array_equal(v.cpu().numpy(), ov) and np.array_equal(a.cpu().numpy(), oa)


def test_large_batch_is_chunked(cuda_device):
    """nq above the library's per-launch query chunk (16384): same answers as small batches."""
    st, queries = B.integer_state(32, 8, 8, 2000, seed=8)
    st.n_probe, st.use_smart_probing = 3, False
    ix = make_index(st)
    x = queries(20000).cuda()
    v, i = ix.search(x, k=7)
    for s in (0, 16380, 19990):
        v2, i2 = ix.search(x[:, s:s + 10].contiguous(), k=7)
        assert torch.equal(v[s:s + 10], v2) and torch.equal(i[s:s + 10], i2)


def test_many_probes_and_wide_k(cuda_device):
    st, queries = B.integer_state(32, 8, 300, 20000, seed=13, lo=-5, hi=6)
    st.n_probe, st.use_smart_probing = 200, True
    x = queries(12)
    ov, oi, oa = O.search(st, x, k=1000, return_address=True)
    ix = make_index(st)
    v, i, a = ix.search(x.cuda(), k=1000, return_address=True)
    assert np.array_equal(v.cpu().numpy(), ov) and np.array_equal(a.cpu().numpy(), oa)


def test_argument_errors(cuda_device):
    st, queries = B.integer_state(32, 8, 8, 500, seed=1)
    ix = make_index(st)
    with pytest.raises(AssertionError):
        ix.search(queries(3).cuda(), k=0)                       # IVFPQIndex.py:473
    with pytest.raises(AssertionError):
        ix.search(queries(3).cuda(), k=1025)
    with pytest.raises(AssertionError):
        ix.search(torch.zeros(31, 3, device="cuda"), k=1)       # IVFPQIndex.py:472
    ix.n_probe = 9                                              # > n_cells
    with pytest.raises(AssertionError):
        ix.search(queries(3).cuda(), k=1)


def test_patch_reference_shaped_object(cuda_device):
    """torchpq_b200.patch() on an object that only has the REFERENCE class's attributes (no torchpq_b200 base
    class): index.search then runs the sm_90a path and matches the oracle."""
    import torchpq_b200 as T

    class Codec:                                   # what torchpq's VQCodec / PQCodec expose to search
        def __init__(self, cb):
            self.codebook, self.is_trained = cb, True

    class RefShaped:                               # attribute names of torchpq.index.IVFPQIndex
        def search(self, x, k=1):
            raise RuntimeError("CuPy path")

    st, queries = B.integer_state(64, 16, 16, 4000, seed=4, lo=-6, hi=7)
    st.n_probe = 5
    g = lambda a: torch.as_tensor(a).cuda().contiguous()
    ref = RefShaped()
    ref.d_vector, ref.n_subvectors, ref.n_cells, ref.distance, ref.device = 64, 16, 16, "euclidean", "cuda:0"
    ref._storage, ref._is_empty, ref._cell_start = g(st.storage), g(st.is_empty), g(st.cell_start)
    ref._cell_size, ref._address2id = g(st.cell_size), g(st.address2id)
    ref.vq_codec, ref.pq_codec = Codec(g(st.vq_codebook)), Codec(g(st.pq_codebook))
    ref.n_probe, ref.use_smart_probing, ref.smart_probing_temperature = 5, True, 30.0
    T.patch(ref)
    x = queries(30)
    ov, oi, oa = O.search(st, x, k=12, return_address=True)
    v, i, a = ref.search(x.cuda(), k=12, return_address=True)
    assert np.array_equal(v.cpu().numpy(), ov) and np.array_equal(a.cpu().numpy(), oa) and np.array_equal(i.cpu().numpy(), oi)
    T.unpatch(ref)
    with pytest.raises(RuntimeError):
        ref.search(x.cuda(), k=12)


@pytest.mark.parametrize("M,d", [(96, 96), (160, 320), (192, 192), (100, 300)])
def test_wide_codes_unit_pipeline(cuda_device, M, d):
    """M = 96 / 160 / 192 / 100: two or three 64-sub-quantizer units per block (odd and even unit counts, a short last
    unit, padding sub-quantizers), 16-warp CTAs, fused (d/M = 1, 2) and staged (d/M = 3) LUTs."""
    st, queries = B.integer_state(d, M, 8, 3000, seed=M, lo=-3, hi=4)
    st.n_probe, st.use_smart_probing = 4, True
    x = queries(24)
    ov, oi, oa = O.search(st, x, k=50, return_address=True)
    ix = make_index(st)
    v, i, a = ix.search(x.cuda(), k=50, return_address=True)
    assert np.array_equal(v.cpu().numpy(), ov) and np.array_equal(a.cpu().numpy(), oa) and np.array_equal(i.cpu().numpy(), oi)


def test_scan_push_single_gpu(cuda_device):
    """tpq_ivfpq_scan_push (the fused scan + exchange of dist.sharded_search) with this GPU as its only 'peer': the keys
    each CTA pushes into slot 0 of the gather buffer are exactly the keys search() returns, for both the in-kernel coarse
    probe and caller-supplied probe lists; a batch small enough to be sliced is refused (the caller then gathers)."""
    import ctypes as C
    import torchpq_b200 as T
    st, queries = B.integer_state(64, 16, 32, 20000, seed=31, lo=-6, hi=7)
    st.n_probe, st.use_smart_probing = 8, True
    ix = make_index(st)
    x = queries(700).cuda()                                       # >= 592 queries: one CTA per query, no slices
    k = 50
    v, i, keys = ix.search(x, k=k, return_keys=True)
    buf = torch.zeros(1, 700, k, dtype=torch.int64, device="cuda")
    ptrs = (C.c_void_p * 1)(buf.data_ptr())
    ix.scan_push(x, k, ptrs, 1, 0)
    torch.cuda.synchronize()
    assert torch.equal(buf[0], keys)
    sims, cells, npl = T.fn.coarse_probe(x, ix.vq_codec.codebook, 8, True, 30.0)
    buf.zero_()
    ix.scan_push(x, k, ptrs, 1, 0, cells=cells, base_sims=sims, n_probe_list=npl)
    torch.cuda.synchronize()
    assert torch.equal(buf[0], keys)
    v2, i2, a2 = T.fn.merge_topk(buf, ix._address2id)
    assert torch.equal(v2, v) and torch.equal(i2, i)
    with pytest.raises(NotImplementedError):
        ix.scan_push(x[:, :40].contiguous(), k, ptrs, 1, 0)


def test_drop_reference_layout(cuda_device):
    """A search-only index: after drop_reference_layout() the reference-layout code store is gone, results are unchanged."""
    st, queries = B.integer_state(64, 16, 32, 20000, seed=33, lo=-6, hi=7)
    st.n_probe, st.use_smart_probing = 8, True
    ix = make_index(st)
    x = queries(50).cuda()
    v0, i0 = ix.search(x, k=20)
    before = ix.resident_bytes()
    ix.drop_reference_layout()
    assert ix._storage is None and ix._is_empty is None and ix.resident_bytes() < before
    v1, i1 = ix.search(x, k=20)
    assert torch.equal(v0, v1) and torch.equal(i0, i1)
    with pytest.raises(AssertionError):
        ix.add(queries(5).cuda())


def test_empty_batch_and_empty_index(cuda_device):
    """Edge cases: a batch of zero queries returns [0, k] tensors; an index that holds no vectors returns (-inf, -1)."""
    import torchpq_b200 as T
    st, queries = B.integer_state(32, 8, 8, 500, seed=3)
    st.n_probe, st.use_smart_probing = 4, True
    ix = make_index(st)
    v, i = ix.search(torch.empty(32, 0, device="cuda"), k=5)
    assert v.shape == (0, 5) and i.shape == (0, 5)
    empty = T.IVFPQIndex(32, 8, 8, initial_size=16, device="cuda:0")
    empty.vq_codec.set_codebook(torch.from_numpy(st.vq_codebook).cuda())
    empty.pq_codec.set_codebook(torch.from_numpy(st.pq_codebook).cuda())
    empty.n_probe = 4
    v, i, a = empty.search(queries(9).cuda(), k=7, return_address=True)
    assert torch.isinf(v).all() and (v < 0).all() and (i == -1).all() and (a == -1).all()
