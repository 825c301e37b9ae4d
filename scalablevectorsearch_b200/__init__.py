"""scalablevectorsearch_b200 -- H100-native Vamana batched search behind the SVS interface.

Only the hot path of SURVEY.md §8 lives here: ``csrc/`` (CUDA kernels + C ABI -> ``libsvsb200.so``),
the host-side mirror of the reference's search interface (:mod:`.vamana`), and the file formats
around it (:mod:`.io`).
"""
from .vamana import (DataType, DistanceType, GraphLoader, SearchBufferConfig, ShardedVamana, Vamana,
                     VamanaBuildParameters, VamanaSearchParameters, VectorDataLoader, build_graph, lvq8_compress)
from ._lib import Svsb200Error

__all__ = ["DataType", "DistanceType", "GraphLoader", "SearchBufferConfig", "Vamana", "VamanaSearchParameters",
           "VectorDataLoader", "Svsb200Error", "lvq8_compress", "ShardedVamana", "VamanaBuildParameters", "build_graph"]
