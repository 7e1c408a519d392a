"""jvector_b200 — H100 (sm_90a) implementation of JVector's distance / quantised-scoring hot path.

The product is the C-ABI library `lib/libjvector_b200.so` (include/jvector_b200.h). This package is the host-side
mirror of the reference's interface for that path, used by the tests and the bench:

  VectorSimilarityFunction                      base:vector/VectorSimilarityFunction.java
  F32Vectors / PQVectors / BQVectors / NVQVectors   RandomAccessVectorValues / CompressedVectors (device resident)
  ProductQuantization.compute / refine          base:quantization/ProductQuantization.java (trained on the device)
  ScoreFunction (similarityTo / similarityToBatch)  base:graph/similarity/ScoreFunction.java
  GraphIndex, GraphSearcher.search              base:graph/GraphSearcher.java:222
  ExhaustiveSearcher.search                     GraphSearcher.search's arguments over every accepted row (no graph)
  SegmentSearcher.search                        GraphSearcher.search over several segment graphs, answers merged on the device
  GraphIndexBuilder.build                       base:graph/GraphIndexBuilder.java:436
  GraphIndexBuilder.refine                      base:graph/GraphIndexBuilder.java:472-538 (cleanup's improveConnections)
  GraphIndexCompactor.compact                   graph/disk/OnDiskGraphIndexCompactor.java (the per-node merge, fp32, FusedPQ or
                                                sidecar PQ with PQRetrainer's retraining; not the file)
"""
from . import api
from .api import (BQVectors, ExhaustiveSearcher, F32Vectors, GraphIndex, GraphIndexBuilder, GraphIndexCompactor, GraphSearcher, NVQVectors, PQVectors,
                  ProductQuantization, QueryBatch, ScoreFunction, SearchResult, SegmentSearcher, SegmentSearchResult, VectorSimilarityFunction, bq_encode_all, kmeans_assign, nvq_encode_all, nvq_encode_resident,
                  pack_accept_bits, pq_encode_all, pq_encode_all_anisotropic, pq_encode_resident, score_multi, topk_bruteforce)
from ._native import JVectorB200Error, init, load

__all__ = ["VectorSimilarityFunction", "F32Vectors", "PQVectors", "BQVectors", "NVQVectors", "ProductQuantization", "ScoreFunction", "GraphIndex",
           "GraphSearcher", "ExhaustiveSearcher", "SegmentSearcher", "SegmentSearchResult", "GraphIndexBuilder", "GraphIndexCompactor", "SearchResult", "score_multi", "topk_bruteforce", "bq_encode_all",
           "pq_encode_all", "pq_encode_all_anisotropic", "pq_encode_resident", "nvq_encode_all", "nvq_encode_resident", "QueryBatch", "kmeans_assign", "pack_accept_bits", "JVectorB200Error", "init", "load"]
