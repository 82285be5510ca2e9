"""The reference's three file-only operators, so complete local pipelines can be wired around the H100 stage
(``gen_data -> compress_hash -> ... -> decompress_verify -> write_local``) without any cloud or socket code.

Behavioural mirrors of skyplane/gateway/operators/gateway_operator.py:
  GatewayWaitReceiver  (:125-150)  forwards a chunk once ``<chunk_id>.chunk`` holds chunk_length_bytes bytes,
                                   otherwise returns False (re-queued) -- uses a stat instead of reading the file;
  GatewayRandomDataGen (:417-452)  creates the chunk file of ``size_mb`` MiB and records its length on the chunk
                                   (the reference calls fallocate, i.e. ZERO-filled data; ``fill="random"`` is ours);
  GatewayWriteLocal    (:455-472)  terminal no-op: the chunk already sits in the chunk directory.
"""
from __future__ import annotations

import os
from multiprocessing import Queue
from typing import Optional

from skyplane_b200.chunk import ChunkRequest
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayOperator

MB = 1 << 20  # skyplane/utils/definitions.py:7


class GatewayWaitReceiver(GatewayOperator):
    def process(self, chunk_req: ChunkRequest, *args) -> bool:
        path = self.chunk_store.get_chunk_file_path(chunk_req.chunk.chunk_id)
        try:
            size = os.stat(path).st_size
        except FileNotFoundError:
            return False  # not downloaded yet
        want = chunk_req.chunk.chunk_length_bytes
        if size < want:
            return False  # still being written
        assert size == want, f"Downloaded chunk length does not match expected length: {size}, {want}"
        return True


class GatewayRandomDataGen(GatewayOperator):
    def __init__(self, handle: str, region: str, input_queue: GatewayQueue, output_queue: Optional[GatewayQueue], error_event,
                 error_queue: Queue, chunk_store: ChunkStore, size_mb: float, n_processes: Optional[int] = 1, fill: str = "zeros"):
        super().__init__(handle, region, input_queue, output_queue, error_event, error_queue, chunk_store, n_processes)
        if fill not in ("zeros", "random"):
            raise ValueError("fill must be 'zeros' (the reference's fallocate behaviour) or 'random'")
        self.size_mb = size_mb
        self.fill = fill

    def process(self, chunk_req: ChunkRequest, *args) -> bool:
        nbytes = int(self.size_mb * MB)
        assert nbytes > 0, f"Invalid size {nbytes} for generated chunk"
        path = self.chunk_store.get_chunk_file_path(chunk_req.chunk.chunk_id)
        tmp = path.with_suffix(".partial")  # downstream readiness checks look at <id>.chunk only
        with open(tmp, "wb") as f:
            if self.fill == "zeros":
                f.truncate(nbytes)
            else:
                left = nbytes
                while left:
                    piece = os.urandom(min(left, 8 * MB))
                    f.write(piece)
                    left -= len(piece)
        os.replace(tmp, path)
        chunk_req.chunk.chunk_length_bytes = os.path.getsize(path)
        return True


class GatewayWriteLocal(GatewayOperator):
    def process(self, chunk_req: ChunkRequest, *args) -> bool:
        return True  # nothing to do: the chunk file is already in the chunk directory
