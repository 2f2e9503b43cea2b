"""Public k-means: ``KMeans`` and ``MultiKMeans``, mirrors of torchpq.clustering.KMeans / MultiKMeans
(clustering/KMeans.py, clustering/MultiKMeans.py) on the library's CUDA kernels.

Data layout as in the reference: ``[d, n]`` for KMeans, ``[l, d, n]`` for MultiKMeans (KMeans is the l = 1 case), and
the trained ``centroids`` buffer is ``[d, k]`` / ``[l, d, k]``, so a reference ``state_dict`` loads here and ours loads
back.  CUDA tensors only: there is no CPU path.

    fit                 the Lloyd loop of build.fit with the tensor-core assignment (fn.kmeans_assign): TF32 wgmma
                        wherever a kernel takes the shape, euclidean and cosine; manhattan on the exact kernel
    predict, get_labels, topk(k=1)
                        the exact fp32 kernel (fn.max_sim), so labels follow the reference's arithmetic
    compute_centroids   member means, summed in point order (bit-reproducible)

Where this differs from the reference, on purpose:
  * initial centroids come from a generator seeded with ``seed`` (random: k distinct points; kmeans++: the first pick),
    not from the unseeded numpy generator, so two fits with the same seed are identical;
  * cosine normalises copies of the data and centroids; the reference divides and re-multiplies the caller's tensors
    in place (KMeans.py:305-323 and kmeanspp), which changes them by rounding;
  * kmeans++ keeps a running per-point best similarity that each new centroid updates (one k = 1 assignment) instead of
    re-scoring every chosen centroid at every step: the same picks in O(n k d) instead of O(n k^2 d);
  * ``topk`` with k > 1 needs a fused distance-GEMM + top-k kernel (the reference's TopkBMMCuda) that this library
    does not have: it raises NotImplementedError.
"""
from __future__ import annotations

import torch

from . import build, fn
from .modules import StateModule

DISTANCES = ("euclidean", "cosine", "manhattan")
INIT_MODES = ("random", "kmeans++")


def _normalized(x):
    """x / (||x|| + 1e-8) along the feature axis, out of place (the reference's cos_sim / get_labels normalisation)."""
    return x / (x.norm(dim=-2, keepdim=True) + 1e-8)


class MultiKMeans(StateModule):
    """l independent k-means over data [l, d, n] (clustering/MultiKMeans.py).  ``sm_size`` is accepted and ignored;
    ``seed`` seeds the initialisation (build.fit)."""

    def __init__(self, n_clusters, n_redo=1, max_iter=100, tol=1e-4, distance="euclidean", init_mode="random",
                 verbose=0, sm_size=48 * 256 * 4, seed=0):
        super().__init__()
        assert distance in DISTANCES, f"distance must be one of {DISTANCES}"
        assert init_mode in INIT_MODES, f"init_mode must be one of {INIT_MODES}"
        self.n_clusters, self.n_redo, self.max_iter, self.tol = n_clusters, n_redo, max_iter, tol
        self.distance, self.init_mode, self.verbose, self.sm_size, self.seed = distance, init_mode, verbose, sm_size, seed
        self.register_buffer("centroids", None)

    # ------------------------------------------------------------------ reference helpers
    @staticmethod
    def calculate_error(a, b):
        """Sum of squared differences (MultiKMeans.py:141-148), the Lloyd loop's stopping error."""
        return (a - b).pow(2).sum()

    @staticmethod
    def calculate_inertia(a):
        return (-a).mean()

    def _max_sim(self, data, centroids):
        """Exact-kernel assignment of data [l, d, n] to centroids [l, d, k] -> (maxsims [l, n], labels [l, n])."""
        if self.distance == "cosine":
            data, centroids = _normalized(data), _normalized(centroids)
        return fn.max_sim(data.contiguous(), centroids.contiguous(), self.distance, exact=True)

    def get_labels(self, data, centroids):
        """data [l, d, n], centroids [l, d, k] -> (maxsims [l, n], labels [l, n]) on the exact kernel."""
        return self._max_sim(data, centroids)

    def compute_centroids(self, data, labels):
        """data [l, d, n], labels [l, n] -> centroids [l, d, k] (member means, empty cluster -> 0)."""
        return fn.compute_centroids(data, labels, self.n_clusters)

    def kmeanspp(self, data, seed=None):
        """data [l, d, n] -> centroids [l, d, k] by k-means++ (see _kmeanspp)."""
        return self._kmeanspp(data, seed)

    def initialize_centroids(self, data, seed=None):
        """data [l, d, n] -> centroids [l, d, k] by init_mode (random: k distinct points from the seeded generator)."""
        return self._initialize(data, seed)

    def _kmeanspp(self, data, seed=None):
        """k-means++ (MultiKMeans.py:232-268): the first centroid is a random point (the same column for every
        k-means), each next one the point whose best similarity to the chosen centroids is lowest (first such point).
        For cosine the picks are normalised points, as in the reference.  -> centroids [l, d, k]."""
        l, d, n = data.shape
        x = (_normalized(data) if self.distance == "cosine" else data).contiguous()
        gen = torch.Generator(device="cpu").manual_seed(self.seed if seed is None else seed)
        first = int(torch.randint(n, (1,), generator=gen))
        cent = torch.zeros(l, d, self.n_clusters, device=data.device, dtype=data.dtype)
        cent[:, :, 0] = x[:, :, first]
        best = fn.max_sim(x, cent[:, :, :1].contiguous(), self.distance, exact=True)[0]      # [l, n] running best
        rows = torch.arange(l, device=data.device)
        for i in range(1, self.n_clusters):
            pick = x[rows, :, best.argmin(dim=-1)]                                          # [l, d]; argmin: first minimum
            cent[:, :, i] = pick
            best = torch.maximum(best, fn.max_sim(x, pick[:, :, None].contiguous(), self.distance, exact=True)[0])
        return cent

    def _initialize(self, data, seed=None):
        seed = self.seed if seed is None else seed
        if self.init_mode == "kmeans++":
            return self._kmeanspp(data, seed)
        return build._init_centroids(data, self.n_clusters, seed)

    # ------------------------------------------------------------------ public API
    def fit(self, data, centroids=None):
        """Cluster data [l, d, n] (optionally from given initial centroids [l, d, k]) -> labels [l, n] of the last
        assignment; the trained centroids land in ``self.centroids``."""
        assert data.is_contiguous(), "use .contiguous()"
        if centroids is not None:
            assert centroids.shape == (data.shape[0], data.shape[1], self.n_clusters)
            centroids = centroids.contiguous()
        cent, labels, inertia, n_iter = build.fit(
            data, self.n_clusters, self.max_iter, tol=self.tol, n_redo=self.n_redo, seed=self.seed,
            centroids=centroids, distance=self.distance, kmeans_assign=True,
            init=lambda x, k, seed: self._initialize(x, seed))
        self.n_iter_, self.inertia_ = n_iter, inertia
        self.print_message(f"finished {self.n_redo} redos, {n_iter} iterations, inertia {inertia}", 1)
        self.register_buffer("centroids", cent)
        return labels

    def predict(self, query):
        """query [l, d, n] -> labels [l, n] of the closest centroid (exact kernel)."""
        assert self.centroids is not None, "kmeans is not trained"
        return self.get_labels(query, self.centroids)[1]

    def topk(self, query, k=1):
        """The best centroid of every query point: (sims [l, n, 1], labels [l, n, 1]).  k > 1 is not implemented."""
        assert self.centroids is not None, "kmeans is not trained"
        assert k <= self.n_clusters, "k is larger than number of clusters"
        if k != 1:
            raise NotImplementedError("topk with k > 1 needs a fused distance-GEMM + top-k kernel, which this library "
                                      "does not have; use k = 1")
        v, i = self.get_labels(query, self.centroids)
        return v[..., None], i[..., None]


class KMeans(MultiKMeans):
    """k-means over data [d, n] (clustering/KMeans.py): MultiKMeans with l = 1; ``centroids`` is [d, k]."""

    def get_labels(self, data, centroids):
        """data [d, n], centroids [d, k] -> (maxsims [n], labels [n]) on the exact kernel."""
        v, i = self._max_sim(data[None], centroids[None])
        return v[0], i[0]

    def compute_centroids(self, data, labels):
        return fn.compute_centroids(data[None], labels[None], self.n_clusters)[0]

    def kmeanspp(self, data, seed=None):
        """data [d, n] -> centroids [d, k]."""
        return self._kmeanspp(data[None], seed)[0]

    def initialize_centroids(self, data, seed=None):
        """data [d, n] -> centroids [d, k]."""
        return self._initialize(data[None], seed)[0]

    def fit(self, data, centroids=None):
        """Cluster data [d, n] -> labels [n]; the trained centroids [d, k] land in ``self.centroids``."""
        assert data.is_contiguous(), "use .contiguous()"
        labels = super().fit(data[None], None if centroids is None else centroids[None])
        self.register_buffer("centroids", self.centroids[0])
        return labels[0]

    def predict(self, query):
        """query [d, n] -> labels [n]."""
        assert self.centroids is not None, "kmeans is not trained"
        return self.get_labels(query, self.centroids)[1]

    def topk(self, query, k=1):
        """(sims [n, 1], labels [n, 1]); k > 1 is not implemented."""
        assert self.centroids is not None, "kmeans is not trained"
        assert k <= self.n_clusters, "k is larger than number of clusters"
        if k != 1:
            raise NotImplementedError("topk with k > 1 needs a fused distance-GEMM + top-k kernel, which this library "
                                      "does not have; use k = 1")
        v, i = self.get_labels(query, self.centroids)
        return v[:, None], i[:, None]
