"""Chunk directory + status log of one gateway (API-compatible with skyplane/gateway/chunk_store.py:14-109).

Layout the stage relies on:
  <chunk_dir>/<chunk_id>.chunk       the chunk's bytes (tmpfs in production, compute/server.py:341)
  <chunk_dir>/<chunk_id>.chunk.lz4   ours: the LZ4 frame produced by / delivered to the H100 stage (or its SecretBox)
  <chunk_dir>/<chunk_id>.chunk.box   ours: the SecretBox of a chunk of a compressed transfer that was sent as itself
                                     (skip_incompressible); such a chunk sent unsealed has no payload file of its own
Operators report state changes with ``log_chunk_state``; the records travel through ``chunk_status_queue`` to
whoever plays the gateway API's role (gateway_daemon_api.py:89-155).
"""
from __future__ import annotations

import shutil
from datetime import datetime, timezone
from multiprocessing import Queue
from os import PathLike
from pathlib import Path
from typing import Dict, Optional, Tuple

from skyplane_b200.chunk import ChunkRequest, ChunkState
from skyplane_b200.gateway_queue import GatewayQueue

CHUNK_SUFFIX = ".chunk"
FRAME_SUFFIX = ".chunk.lz4"
BOX_SUFFIX = ".chunk.box"


def _utc_stamp() -> str:
    return datetime.now(timezone.utc).replace(tzinfo=None).isoformat()


class ChunkStore:
    def __init__(self, chunk_dir: PathLike):
        self.chunk_dir = Path(chunk_dir)
        self.chunk_dir.mkdir(parents=True, exist_ok=True)
        self._purge_leftovers()
        self.region_key_upload_id_mappings: Dict[str, str] = {}
        self.chunk_requests: Dict[str, GatewayQueue] = {}  # partition id -> queue feeding the operator graph
        self.chunk_status_queue: Queue = Queue()  # status records, operators -> API

    def _purge_leftovers(self) -> None:
        """A gateway always starts with an empty chunk directory (chunk_store.py:21-24)."""
        for pattern in ("*" + CHUNK_SUFFIX, "*" + FRAME_SUFFIX, "*" + BOX_SUFFIX):
            for leftover in self.chunk_dir.glob(pattern):
                leftover.unlink()

    # -- multipart bookkeeping --------------------------------------------------------------------
    def set_upload_ids_map(self, maps: Dict[str, str]) -> None:
        self.region_key_upload_id_mappings.update(maps)

    def get_upload_ids_map(self) -> Dict[str, str]:
        return self.region_key_upload_id_mappings

    def get_upload_id_map_path(self) -> Path:
        return self.chunk_dir / "upload_id_map.json"

    # -- partitions and incoming requests ---------------------------------------------------------
    def add_partition(self, partition_id: str, queue: Optional[GatewayQueue] = None) -> None:
        if partition_id in self.chunk_requests:
            raise ValueError(f"Partition {partition_id} already exists")
        self.chunk_requests[partition_id] = GatewayQueue() if queue is None else queue

    def add_chunk_request(self, chunk_request: ChunkRequest, state: ChunkState = ChunkState.registered) -> Tuple[int, bool]:
        """Called for every request the gateway API receives. -> (queue depth, accepted?)"""
        partition = chunk_request.chunk.partition_id
        target = self.chunk_requests.get(partition)
        if target is None:
            raise ValueError(f"Partition {partition} does not exist in {self.chunk_requests} - was the gateway program loaded?")
        try:
            target.put_nowait(chunk_request)
        except Exception as exc:  # queue.Full: tell the caller to back off
            print("Error adding chunk", exc)
            return target.size(), False
        self.log_chunk_state(chunk_request, state)
        return target.size(), True

    def add_chunk_requests(self, chunk_requests, state: ChunkState = ChunkState.registered) -> None:
        """Batch form of ``add_chunk_request`` (all requests of one partition): one queue element, one status element."""
        reqs = list(chunk_requests)
        if not reqs:
            return
        target = self.chunk_requests.get(reqs[0].chunk.partition_id)
        if target is None:
            raise ValueError(f"Partition {reqs[0].chunk.partition_id} does not exist in {self.chunk_requests} - was the gateway program loaded?")
        target.put_many(reqs)
        self.log_chunk_states(reqs, state)

    # -- status log -------------------------------------------------------------------------------
    def log_chunk_state(
        self,
        chunk_req: ChunkRequest,
        new_status: ChunkState,
        worker_id: Optional[int] = None,
        operator_handle: Optional[str] = None,
        metadata: Optional[Dict] = None,
    ) -> None:
        record = dict(
            chunk_id=chunk_req.chunk.chunk_id,
            partition=chunk_req.chunk.partition_id,
            state=new_status.name,
            time=_utc_stamp(),
            handle=operator_handle,
            worker_id=worker_id,
        )
        if metadata:
            record.update(metadata)  # e.g. compressed_size_bytes / uncompressed_size_bytes from the H100 stage
        self.chunk_status_queue.put(record)

    def log_chunk_states(self, chunk_reqs, new_status: ChunkState, worker_id: Optional[int] = None, operator_handle: Optional[str] = None,
                         metadata: Optional[list] = None) -> None:
        """Batch form of ``log_chunk_state``: the same records, shipped as ONE queue element (a list).  A consumer of
        ``chunk_status_queue`` sees either a dict (the reference's form) or a list of such dicts (``iter_status_records``)."""
        stamp = _utc_stamp()
        records = []
        for i, r in enumerate(chunk_reqs):
            rec = dict(chunk_id=r.chunk.chunk_id, partition=r.chunk.partition_id, state=new_status.name, time=stamp, handle=operator_handle,
                       worker_id=worker_id)
            if metadata and metadata[i]:
                rec.update(metadata[i])
            records.append(rec)
        if records:
            self.chunk_status_queue.put(records)

    @staticmethod
    def iter_status_records(item):
        """Normalise one element taken from ``chunk_status_queue`` to its records."""
        return item if isinstance(item, list) else (item,)

    # -- files ------------------------------------------------------------------------------------
    def get_chunk_file_path(self, chunk_id: str) -> Path:
        return self.chunk_dir / (chunk_id + CHUNK_SUFFIX)

    def get_compressed_file_path(self, chunk_id: str) -> Path:
        return self.chunk_dir / (chunk_id + FRAME_SUFFIX)

    def get_box_file_path(self, chunk_id: str) -> Path:
        return self.chunk_dir / (chunk_id + BOX_SUFFIX)

    def wire_payload(self, chunk_id: str) -> Tuple[Path, bool]:
        """What a sender of a compressed transfer puts on the wire for a chunk the H100 stage has handled (INTEGRATION §2):
        -> (payload file, WireProtocolHeader.is_compressed).  ``.chunk.lz4`` is a frame or the box of a frame; ``.chunk.box``
        is the box of a chunk sent as itself; with neither, ``<chunk_id>.chunk`` itself goes, uncompressed.  (With
        ``compress: false`` every payload is uncompressed, whatever its file.)"""
        for path, compressed in ((self.get_compressed_file_path(chunk_id), True), (self.get_box_file_path(chunk_id), False)):
            if path.exists():
                return path, compressed
        return self.get_chunk_file_path(chunk_id), False

    def remaining_bytes(self) -> int:
        try:
            return shutil.disk_usage(self.chunk_dir).free
        except OSError:
            return 0
