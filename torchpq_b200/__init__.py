"""torchpq_b200 -- H100-native (sm_90a) IVFPQ search path behind torchpq.index.IVFPQIndex.search(), IVFPQ search
re-ranked on a second PQ code (IVFPQRIndex), exact flat search (FlatIndex), inverted-file search with exact distances
(IVFFlatIndex), inverted-file search over scalar-quantized vectors (IVFSQIndex, codec.SQCodec), IVFPQ search
over 4-bit PQ codes (IVFPQ4Index), exact fp32 re-ranking of any
of these indexes' candidates (RefineFlatIndex), row-wise top-k (topk = fn.Topk()), and k-means
(clustering.KMeans / MultiKMeans).

Importing this package loads ``libtpq_b200.so``; there is no CPU / PyTorch fallback.
"""
from . import _lib  # noqa: F401  (raises ImportError when the CUDA library is missing)
from .index import IVFPQIndex, ScanLayout
from .flat_index import FlatIndex
from .ivfpqr_index import IVFPQRIndex
from .ivfflat_index import IVFFlatIndex
from .ivfsq_index import IVFSQIndex
from .ivfpq4_index import IVFPQ4Index
from .refine_index import RefineFlatIndex
from . import codec
from . import fn
from . import clustering
from .clustering import KMeans, MultiKMeans
from .patch import patch, unpatch

topk = fn.Topk()                     # torchpq.topk (torchpq/__init__.py:22)

__all__ = ["IVFPQIndex", "IVFPQRIndex", "IVFFlatIndex", "IVFSQIndex", "IVFPQ4Index", "FlatIndex", "RefineFlatIndex", "codec", "ScanLayout", "KMeans", "MultiKMeans", "clustering", "fn", "topk", "patch", "unpatch"]
