"""CPU: the SQ codec oracle against the reference's torch expressions (torchpq/codec/SQCodec.py, restated below op for
op on CPU torch), SQCodec's and IVFSQIndex's constructors, buffers and checkpoint keys, and the argument errors of
tpq_sq_encode, tpq_sq_decode and tpq_ivfsq_search (which return before any launch).  No GPU needed."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ivfsq_oracle as SO


# ---------------------------------------------------------------- the reference's expressions (SQCodec.py), CPU torch
def _ref_train(x, mode, alpha=1.0):
    if mode == "minmax":
        lower, upper = x.min(dim=-1)[0], x.max(dim=-1)[0]
    else:
        means, stds = x.mean(dim=-1), x.std(dim=-1)
        lower, upper = means - alpha * stds, means + alpha * stds
    return lower, upper, upper - lower + 1e-8


def _ref_encode8(x, lower, rng):
    t = x - lower[:, None]
    t.div_(rng[:, None])
    t.mul_(256)
    t.round_()
    t.clamp_(min=0, max=255)
    return t.byte()


def _ref_decode8(code, lower, rng):
    out = code.float()
    out.div_(256)
    out.mul_(rng[:, None])
    out.add_(lower[:, None])
    return out


def _bits(a):
    return np.asarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("mode", ["minmax", "meanstd"])
def test_oracle_codec_equals_reference_expressions(mode):
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((16, 3000)).astype(np.float32) * 3)
    lower, upper, rg = _ref_train(x, mode, 0.7)
    lo, r = lower.numpy(), rg.numpy()
    # randn, then values exactly half-way between two codes, x = lower, x = upper and values outside [lower, upper]
    half = (lower[:, None] + ((torch.arange(40, dtype=torch.float32) + 0.5) / 256)[None, :] * rg[:, None])
    extra = torch.cat([half, lower[:, None], upper[:, None], lower[:, None] - 5, upper[:, None] + 5,
                       torch.full((16, 1), 1e30), torch.full((16, 1), -1e30)], 1)
    xs = torch.cat([x, extra], 1).contiguous()
    want = _ref_encode8(xs.clone(), lower, rg)
    got = SO.encode(xs.numpy(), 8, lo, r)
    assert np.array_equal(got, want.numpy())
    assert np.array_equal(_bits(SO.decode(got, 8, lo, r)), _bits(_ref_decode8(want, lower, rg).numpy()))
    all_codes = np.tile(np.arange(256, dtype=np.uint8), (16, 1))
    assert np.array_equal(_bits(SO.decode(all_codes, 8, lo, r)),
                          _bits(_ref_decode8(torch.from_numpy(all_codes), lower, rg).numpy()))


def test_oracle_codec_quirks():
    x = torch.tensor([[0.0, 1.0, 0.5, 2.0]])
    lower, upper, rg = _ref_train(x, "minmax")
    lo, r = lower.numpy(), rg.numpy()
    code = SO.encode(x.numpy(), 8, lo, r)
    assert code[0, 3] == 255                                    # x == upper: 256, clamped to 255
    back = SO.decode(np.array([[255]], np.uint8), 8, lo, r)
    assert back[0, 0] < upper[0].item()                          # code 255 never decodes to upper
    assert back[0, 0] == np.float32(np.float32(255 / 256) * r[0]) + lo[0]


def test_oracle_fp16_equals_reference():
    rng = np.random.default_rng(1)
    x = np.concatenate([rng.standard_normal((4, 500)).astype(np.float32) * 1000,
                        np.array([[65504, 65520, 7e4, -7e4]] * 4, np.float32)], 1)
    t = torch.from_numpy(x)
    code = SO.encode(x, 16)
    assert np.array_equal(code.view(np.uint16), t.half().numpy().view(np.uint16))
    assert np.isinf(code[:, -2:]).all() and np.isinf(code[:, -3]).all()     # beyond +-65504 (after rounding): +-inf
    assert np.array_equal(_bits(SO.decode(code, 16)), _bits(t.half().float().numpy()))


# ---------------------------------------------------------------- constructors and checkpoints
def test_sqcodec_constructor_and_buffers():
    import torchpq_b200 as T
    for bits in (8, 16, 32):
        c = T.codec.SQCodec(bits=bits)
        assert c.n_bins == 2 ** bits and not c.is_trained
        assert set(c._buffers) == {"_is_trained", "lower", "upper", "binsize", "range"}
        assert c.binsize is None and c.lower is None
    for bits in (4, 2, 12):
        with pytest.raises(NotImplementedError):
            T.codec.SQCodec(bits=bits)
    c = T.codec.SQCodec(bits=16)
    c.train(torch.randn(4, 10))
    assert c.is_trained and c.lower is None                     # 16 bits: nothing to fit


def test_sqcodec_train_is_the_reference_expression():
    import torchpq_b200 as T
    x = torch.randn(6, 200)
    for mode, alpha in (("minmax", 1.0), ("meanstd", 0.5)):
        c = T.codec.SQCodec(mode=mode, alpha=alpha)
        c.train(x)
        lower, upper, rg = _ref_train(x, mode, alpha)
        assert torch.equal(c.lower, lower) and torch.equal(c.upper, upper) and torch.equal(c.range, rg)
        assert sorted(c.state_dict()) == ["_is_trained", "lower", "range", "upper"]   # binsize is None: not saved


def test_reference_shaped_state_dict_loads():
    import torchpq_b200 as T
    sd = {"_is_trained": torch.tensor(True), "lower": torch.zeros(8), "upper": torch.ones(8),
          "range": torch.ones(8) + 1e-8}
    c = T.codec.SQCodec()
    c.load_state_dict(sd)
    assert c.is_trained and torch.equal(c.upper, torch.ones(8)) and c.binsize is None
    ix = T.IVFSQIndex(8, 2, initial_size=1, device="cpu")
    full = ix.state_dict()
    full.update({"sq_codec." + k: v for k, v in sd.items()})
    ix2 = T.IVFSQIndex(8, 2, initial_size=0, device="cpu")
    ix2.load_state_dict(full)
    assert ix2.sq_codec.is_trained and torch.equal(ix2.sq_codec.lower, torch.zeros(8)) and ix2.capacity == 2


def _index(**kw):
    import torchpq_b200 as T
    return T.IVFSQIndex(device="cpu", **kw)


def test_ivfsq_constructor_validation_and_buffers():
    for bits in (4, 32, 7):
        with pytest.raises(NotImplementedError):
            _index(d_vector=8, bits=bits)
    for name in ("inner", "manhattan"):
        with pytest.raises(NotImplementedError, match=name):
            _index(d_vector=8, distance=name)
    with pytest.raises(AssertionError):
        _index(d_vector=6, bits=8)                             # 8 bits: d % 4 == 0
    with pytest.raises(AssertionError):
        _index(d_vector=5, bits=16)                            # 16 bits: d % 2 == 0
    ix = _index(d_vector=12, n_cells=4, initial_size=3, distance="cosine")
    assert ix._storage.dtype == torch.uint8 and ix._storage.shape == (3, 12, 4) and ix.code_size == 12
    assert (ix.n_probe, ix.use_smart_probing, ix.smart_probing_temperature) == (1, True, 30.0)
    ix16 = _index(d_vector=6, n_cells=4, initial_size=3, bits=16)
    assert ix16._storage.shape == (3, 12, 4) and ix16.code_size == 12
    assert ix16.sq_codec.bits == 16 and not ix16.sq_codec.is_trained


def test_ivfsq_state_dict_keys():
    import torchpq_b200 as T
    ix = _index(d_vector=8, n_cells=2, initial_size=1)
    base = {"_address2id", "_storage", "_cell_start", "_cell_size", "_cell_capacity", "_is_empty",
            "vq_codec._is_trained", "sq_codec._is_trained"}
    assert set(ix.state_dict()) == base                        # None buffers are not saved
    ix.sq_codec.train(torch.randn(8, 50))
    assert set(ix.state_dict()) == base | {"sq_codec.lower", "sq_codec.upper", "sq_codec.range"}
    assert "binsize" in ix.sq_codec._buffers and ix.sq_codec.binsize is None
    pq = set(T.IVFPQIndex(8, 4, 2, initial_size=1, device="cpu").state_dict())
    assert {k for k in base if not k.startswith("sq_codec")} <= pq   # IVFPQIndex's names


# ---------------------------------------------------------------- C ABI argument errors
def test_sq_codec_abi_argument_errors():
    import torchpq_b200 as T
    L, E = T._lib.lib, T._lib
    fake = C.c_void_p(256)                                     # never dereferenced: every call fails its checks first
    for f in (L.tpq_sq_encode, L.tpq_sq_decode):
        assert f(fake, 8, 10, 4, fake, fake, fake, None) == E.TPQ_ERR_UNSUPPORTED
        assert f(fake, 8, 10, 12, fake, fake, fake, None) == E.TPQ_ERR_UNSUPPORTED
        assert f(fake, 0, 10, 8, fake, fake, fake, None) == E.TPQ_ERR_BAD_ARG and "bad sizes" in E.last_error()
        assert f(fake, 8, -1, 8, fake, fake, fake, None) == E.TPQ_ERR_BAD_ARG
        assert f(None, 8, 10, 8, fake, fake, fake, None) == E.TPQ_ERR_BAD_ARG and "null input" in E.last_error()
        assert f(fake, 8, 10, 8, fake, fake, None, None) == E.TPQ_ERR_BAD_ARG
        assert f(fake, 8, 10, 8, None, fake, fake, None) == E.TPQ_ERR_BAD_ARG and "lower or range" in E.last_error()
        assert f(fake, 8, 10, 8, fake, None, fake, None) == E.TPQ_ERR_BAD_ARG
        assert f(None, 8, 0, 8, fake, fake, None, None) == E.TPQ_OK            # n == 0 launches nothing


def test_ivfsq_abi_argument_errors():
    import torchpq_b200 as T
    L, E = T._lib.lib, T._lib
    fake = C.c_void_p(256)
    lo = C.c_void_p(512)                                       # 16-byte aligned

    def search(k=10, metric=0, nq=4, n_probe=2, cells=None, npl=None, capacity=100, ws_bytes=1 << 40, n_cells=8,
               values=fake, bits=8, d=8, lower=lo, range_=lo):
        return L.tpq_ivfsq_search(fake, d, nq, fake, n_cells, fake, bits, lower, range_, capacity, fake, fake, fake,
                                  fake, metric, cells, npl, n_probe, 0, 30.0, k, fake, values, fake, None, fake,
                                  ws_bytes, None)

    for bits in (4, 32, 0):
        assert search(bits=bits) == E.TPQ_ERR_UNSUPPORTED and "8 and 16 only" in E.last_error()
    assert search(d=6) == E.TPQ_ERR_BAD_ARG and "multiple of 4" in E.last_error()
    assert search(d=5, bits=16) == E.TPQ_ERR_BAD_ARG and "multiple of 2" in E.last_error()
    assert search(lower=None) == E.TPQ_ERR_BAD_ARG and "null lower or range" in E.last_error()
    assert search(range_=None) == E.TPQ_ERR_BAD_ARG and "null lower or range" in E.last_error()
    assert search(lower=C.c_void_p(260)) == E.TPQ_ERR_BAD_ARG and "16-byte aligned" in E.last_error()
    assert search(k=0) == E.TPQ_ERR_BAD_ARG and "k must be in (0, 1024]" in E.last_error()
    assert search(k=1025) == E.TPQ_ERR_UNSUPPORTED
    for m in (E.METRIC["inner"], E.METRIC["manhattan"], 7):
        assert search(metric=m) == E.TPQ_ERR_UNSUPPORTED and "euclidean and cosine only" in E.last_error()
    assert search(nq=-1) == E.TPQ_ERR_BAD_ARG and "bad sizes" in E.last_error()
    assert search(n_probe=0) == E.TPQ_ERR_BAD_ARG
    assert search(capacity=1 << 32) == E.TPQ_ERR_BAD_ARG and "32-bit address" in E.last_error()
    assert search(cells=fake) == E.TPQ_ERR_BAD_ARG and "go together" in E.last_error()
    assert search(n_probe=9) == E.TPQ_ERR_BAD_ARG and "n_probe=9 must be in [1, n_cells=8]" in E.last_error()
    assert search(values=None) == E.TPQ_ERR_BAD_ARG and "null output" in E.last_error()
    assert "tpq_ivfsq_search" in E.last_error()
    assert search(nq=0) == E.TPQ_OK
    assert search(nq=0, bits=16, lower=None, range_=None) == E.TPQ_OK     # 16 bits read no bounds
    need = L.tpq_ivfflat_workspace_bytes(8, 4, 8, 2, 10)                  # the workspace is IVFFlat's
    assert search(ws_bytes=need - 1) == E.TPQ_ERR_WORKSPACE and "workspace too small" in E.last_error()
