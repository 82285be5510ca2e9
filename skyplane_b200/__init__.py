"""skyplane_b200 -- H100-native chunk-processing stage (LZ4 frame + MD5) for Skyplane's gateway.

Scope: the one data-parallel hot path of the gateway (SURVEY.md section 8).  Public surface:
  chunk         Chunk / ChunkRequest / ChunkState / WireProtocolHeader (reference-compatible)
  gateway_queue GatewayQueue / GatewayANDQueue
  chunk_store   ChunkStore
  operators     GatewayOperator (plugin base) and GatewayCompressHash (the H100 stage)
  stage         ChunkStage: pinned staging + fused kernel launches
  native        ctypes binding of libskychunk.so (C ABI in include/skychunk.h)
There is no CPU fallback: the compute path requires the CUDA library and a GPU.
"""
__version__ = "0.1.0"

from skyplane_b200.chunk import Chunk, ChunkRequest, ChunkState, WireProtocolHeader  # noqa: F401
