"""CPU restatement of the k-means / codec neighbours of the search path (TEST INFRASTRUCTURE).

    max_sim            kernels/cuda/max_sim.cu:182-309 (thread_nseuclidean :78-98 / thread_matmul, reduce_dim_2 :152-180)
                       as called by MultiKMeans.get_labels (clustering/MultiKMeans.py:314-333)
    compute_centroids  kernels/cuda/compute_centroids.cu:9-86
    pq_decode          kernels/cuda/pq_decode.cu:7-53 ; PQCodec._decode_cpu codec/PQCodec.py:95-111
"""
import numpy as np

from .fp32_exact import fma32


def _fma32(a, b, c):
    """fp32 fused multiply-add with one rounding (fp32_exact.fma32: float64 sum, corrected where it double-rounds)."""
    return fma32(a, b, c)


def max_sim(data, cent, distance="euclidean", chunk=4096):
    """data [l, d, n], cent [l, d, k] -> (maxsims [l, n] f32, labels [l, n] i64).
    Similarity accumulated feature by feature with fmaf(-dif, dif, acc) (euclidean) or fmaf(a, b, acc)
    (inner), e ascending, as the kernel does; arg-max = lowest index among equal maxima."""
    data, cent = np.asarray(data, np.float32), np.asarray(cent, np.float32)
    l, d, n = data.shape
    k = cent.shape[2]
    sims = np.empty((l, n), np.float32)
    labels = np.empty((l, n), np.int64)
    for li in range(l):
        for s in range(0, n, chunk):
            x = data[li, :, s:s + chunk]                         # [d, m]
            acc = np.zeros((x.shape[1], k), np.float32)
            for e in range(d):
                a = x[e][:, None]
                b = cent[li, e][None, :]
                if distance == "euclidean":
                    dif = (a - b).astype(np.float32)
                    acc = _fma32(-dif, dif, acc)
                else:
                    acc = _fma32(np.broadcast_to(a, acc.shape), np.broadcast_to(b, acc.shape), acc)
            labels[li, s:s + chunk] = acc.argmax(axis=1)
            sims[li, s:s + chunk] = acc.max(axis=1)
    return sims, labels


def compute_centroids(data, labels, k):
    """data [l, d, n], labels [l, n] -> centroids [l, d, k] (member mean in float64, empty cluster -> 0).
    Labels outside [0, k) belong to no cluster (compute_centroids.cu:61-64 skips them)."""
    data = np.asarray(data, np.float32)
    labels = np.asarray(labels, np.int64)
    l, d, n = data.shape
    out = np.zeros((l, d, k), np.float64)
    for li in range(l):
        ok = (labels[li] >= 0) & (labels[li] < k)
        lab = labels[li][ok]
        cnt = np.bincount(lab, minlength=k).astype(np.float64)
        for e in range(d):
            out[li, e] = np.bincount(lab, weights=data[li, e][ok].astype(np.float64), minlength=k)
        nz = cnt > 0
        out[li][:, nz] /= cnt[nz]
        out[li][:, ~nz] = 0
    return out.astype(np.float32)


def compute_centroids_seq(data, labels, k):
    """data [l, d, n], labels [l, n] -> centroids [l, d, k] in the arithmetic the GPU update promises: each member sum
    is taken in fp32, starting from 0 and adding one member at a time in point order; the mean is fp32(sum) /
    fp32(count), rounded once; an empty cluster is 0; labels outside [0, k) are ignored.  That is a fixed function of
    the inputs, so the GPU kernels must match it bit for bit.

    Vectorised over clusters: step r adds, for every cluster at once, its member of rank r (its r-th point in point
    order), so the loop runs max(count) times, not n times."""
    data = np.asarray(data, np.float32)
    labels = np.asarray(labels, np.int64)
    l, d, n = data.shape
    out = np.zeros((l, d, k), np.float32)
    for li in range(l):
        pts = np.nonzero((labels[li] >= 0) & (labels[li] < k))[0]
        if len(pts) == 0:
            continue
        lab = labels[li][pts]
        pts = pts[np.argsort(lab, kind="stable")]               # grouped by cluster, point order kept inside each
        cnt = np.bincount(lab, minlength=k)
        start = np.concatenate(([0], np.cumsum(cnt)[:-1]))      # first sorted position of each cluster
        by_cnt = np.argsort(-cnt, kind="stable")                # clusters with a member of rank r: a prefix of by_cnt
        cnt_desc = cnt[by_cnt]
        sums = np.zeros((d, k), np.float32)
        for r in range(int(cnt_desc[0])):
            cl = by_cnt[:np.searchsorted(-cnt_desc, -r, side="left")]   # clusters with count > r
            sums[:, cl] += data[li][:, pts[start[cl] + r]]      # fp32 + fp32, rounded once
        nz = cnt > 0
        out[li][:, nz] = sums[:, nz] / cnt[nz].astype(np.float32)
    return out


def pq_decode(codebook, code):
    """codebook [M, dsub, 256], code [M, n] u8 -> [M*dsub, n] f32."""
    M, dsub, _ = codebook.shape
    n = code.shape[1]
    out = np.empty((M, dsub, n), np.float32)
    for m in range(M):
        out[m] = codebook[m][:, code[m]]
    return out.reshape(M * dsub, n)


def fit(data, centroids0, max_iter, tol=1e-4):
    """MultiKMeans.fit for one redo from given initial centroids, euclidean (clustering/MultiKMeans.py:431-441):
    labels = arg-max similarity, new centroids = member means, error = sum((new - old)^2), stop when error <= tol.
    -> (centroids, labels of the last assignment, inertia = mean(-maxsims), iterations)."""
    cent = np.asarray(centroids0, np.float32)
    k = cent.shape[2]
    n_iter = 0
    for _ in range(max_iter):
        sims, labels = max_sim(data, cent, "euclidean")
        new = compute_centroids(data, labels, k)
        diff = (new - cent).astype(np.float32)
        error = float((diff * diff).astype(np.float32).sum(dtype=np.float32))
        cent = new
        n_iter += 1
        if error <= tol:
            break
    return cent, labels, float((-sims).mean()), n_iter
