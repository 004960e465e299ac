"""pg_embedding_b200 -- H100-native (sm_90a) HNSW candidate-scoring path for pg_embedding.

The product is the C-ABI shared library ``libpgemb_b200.so`` (include/pgemb_b200.h); this package holds
its CUDA sources (csrc/), the build script and a thin host-side mirror of the reference's interface for
the hot path (index.py).  Importing the symbols below requires the built library: there is no CPU
fallback.
"""
from .index import (DIST_COSINE, DIST_L2, DIST_MANHATTAN, HnswIndex, cosine_distance, device_count,  # noqa: F401
                    dist_batch, l2_distance, manhattan_distance)

__all__ = ["HnswIndex", "l2_distance", "cosine_distance", "manhattan_distance", "dist_batch", "device_count",
           "DIST_L2", "DIST_COSINE", "DIST_MANHATTAN"]
