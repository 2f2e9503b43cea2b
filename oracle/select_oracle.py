"""CPU oracle of row-wise top-k (torchpq_b200.topk / tpq_topk; TEST INFRASTRUCTURE ONLY).

Restates the library's total order in numpy on the integer image of the float, the map of score_to_ord
(csrc/common.cuh): sign bit set -> all bits flipped, else the sign bit set; every NaN, of either sign, maps to the
largest image (above +inf).  A row is sorted stably by image descending, so equal images keep column order: value
descending, then column ascending, +0 above -0.  The values are the images decoded again, so a NaN comes back as the
NaN 0x7fffffff.  (ivfpq_oracle.select_topk sorts float64 values and ties +0 with -0; it cannot serve here.)
"""
import numpy as np


def order_image(x):
    """fp32 / fp16 array -> uint32 image under the total order (fp16 is widened exactly first)."""
    f = np.ascontiguousarray(x, dtype=np.float32)
    b = f.view(np.uint32)
    img = np.where(b & np.uint32(0x80000000), ~b, b | np.uint32(0x80000000)).astype(np.uint32)
    img[np.isnan(f)] = np.uint32(0xFFFFFFFF)
    return img


def image_value(img):
    """The inverse of order_image on non-NaN images; 0xFFFFFFFF decodes as the NaN 0x7fffffff."""
    img = np.asarray(img, dtype=np.uint32)
    b = np.where(img & np.uint32(0x80000000), img ^ np.uint32(0x80000000), ~img).astype(np.uint32)
    return b.view(np.float32)


def topk(x, k):
    """x [m, n] fp32 / fp16 -> (values [m, k] f32, indices [m, k] i64), rows shorter than k padded (-inf, -1)."""
    x = np.asarray(x)
    assert x.ndim == 2 and k >= 1
    m, n = x.shape
    img = order_image(x)
    kk = min(k, n)
    # stable sort of the complement ascending == image descending, ties by column ascending
    order = np.argsort(~img, axis=1, kind="stable")[:, :kk]
    values = np.full((m, k), -np.inf, dtype=np.float32)
    indices = np.full((m, k), -1, dtype=np.int64)
    values[:, :kk] = image_value(np.take_along_axis(img, order, axis=1))
    indices[:, :kk] = order
    return values, indices


def same_values(a, b):
    """Bit-identical float32 arrays, a NaN equal to a NaN (of any payload)."""
    a, b = np.asarray(a, dtype=np.float32), np.asarray(b, dtype=np.float32)
    if a.shape != b.shape:
        return False
    na, nb = np.isnan(a), np.isnan(b)
    return bool(np.array_equal(na, nb) and np.array_equal(a.view(np.uint32)[~na], b.view(np.uint32)[~nb]))
