"""morphik-core_b200 -- H100-native ColPali late-interaction (MaxSim) path for Morphik.

Host side is Python (like the reference) calling hand-written sm_90a CUDA through the C-ABI in
include/b200ms.h (ctypes).  Modules:
  _native   ctypes binding of libb200ms.so (fails loudly when the library is missing; there is no CPU fallback)
  index     MaxSimIndex: device-resident packed corpus + search (torch only holds the tensors)
  models    DocumentChunk, the record type of core/models/chunk.py
  store     B200MultiVectorStore, the BaseVectorStore plugin (core/vector_store/base_vector_store.py:7-65)
  sharded   document-sharded multi-GPU search (torch.distributed / NCCL all-gather of per-shard top-k)
  sharded_store  the BaseVectorStore plugin over all GPUs of a box (rank 0 serves, ranks > 0 run worker_loop)
  fde       FixedDimensionalEncodingConfig / generate_*_encoding (MUVERA FDE) and TwoStageIndex (FDE candidates -> MaxSim rerank)
  shardfile packed shard files (the HBM layout on disk) + importers for the reference's .npy / BIT(128)[] forms
  reranker  embedding-based MaxSim reranker adapter
"""
__version__ = "0.1.1"
