"""In-process gateway harness: ChunkStore + GatewayQueue + GatewayCompressHash workers.

The reference has no fake backend (SURVEY.md section 4); this is ours.  It reproduces what
``gateway_daemon`` wires around an operator (gateway_daemon.py:126-341): a chunk directory, an input
queue fed with ChunkRequests, forked operator workers (one per GPU, worker_id -> device) and a drained
status / output queue.  The calling process must NOT have initialised CUDA: workers are forked.

Run as a module for BASELINE config 4-style streams:
    python -m skyplane_b200.harness --gpus 8 --chunks 12800 --chunk-mib 8 --pool 64
"""
from __future__ import annotations

import argparse
import json
import multiprocessing as mp
import os
import queue
import shutil
import tempfile
import time
import uuid
from pathlib import Path
from typing import Callable, Dict, List, Optional, Sequence

from skyplane_b200.chunk import Chunk, ChunkRequest
from skyplane_b200.chunk_store import ChunkStore
from skyplane_b200.gateway_queue import GatewayQueue
from skyplane_b200.operators import GatewayCompressHash


def _drain_status(store: ChunkStore, acc: Dict):
    try:
        while True:
            for rec in store.iter_status_records(store.chunk_status_queue.get_nowait()):
                acc["states"][rec["state"]] = acc["states"].get(rec["state"], 0) + 1
                acc["comp"] += rec.get("compressed_size_bytes", 0)
                acc["raw"] += rec.get("uncompressed_size_bytes", 0)
                if "frame_verify_status" in rec:
                    acc["verify"][rec["chunk_id"]] = rec["frame_verify_status"]
                if rec.get("passed_through"):
                    acc["passed_through"].add(rec["chunk_id"])
    except queue.Empty:
        pass


def run_stream(
    chunk_dir: os.PathLike,
    pool_files: Sequence[os.PathLike],
    pool_lens: Sequence[int],
    n_requests: int,
    n_workers: int = 1,
    n_gpus: Optional[int] = None,
    max_batch_chunks: int = 64,
    max_batch_bytes: int = 1 << 30,
    keep_frames: bool = True,
    window: int = 512,
    timeout_s: float = 600.0,
    on_done: Optional[Callable[[ChunkRequest], None]] = None,
    warmup_requests: int = 0,
    operator_cls=GatewayCompressHash,
    n_slots: int = 4,
    **operator_options,
) -> Dict:
    """Stream ``n_requests`` chunk requests (recycling ``pool_files`` by hard link) through the operator.

    The first ``warmup_requests`` completions are not timed (worker start-up: CUDA context, pinned staging).
    ``operator_options`` are handed to ``operator_cls`` as they are (GatewayCompressHash's sender options, e.g.
    ``high_ratio=True`` or ``compression_level=9``).
    Returns {"wall_s", "bytes", "records": [{chunk_id, pool_index, md5, raw_len, frame_path}], "status": {...},
    "frame_verify": {chunk_id: status of every chunk whose frame failed the check},
    "passed_through": [chunk_id of every chunk sent as itself]}.
    """
    chunk_dir = Path(chunk_dir)
    store = ChunkStore(chunk_dir)
    qin, qout = GatewayQueue(), GatewayQueue()
    store.add_partition("0", qin)
    err_ev, err_q = mp.Event(), mp.Queue()
    op = operator_cls(
        "compress_hash", "local:box", qin, qout, err_ev, err_q, store, n_processes=n_workers,
        max_batch_chunks=max_batch_chunks, max_batch_bytes=max_batch_bytes, n_gpus=n_gpus, keep_frames_on_disk=keep_frames, n_slots=n_slots,
        **operator_options,
    )
    op.start_workers()
    records: List[Dict] = []
    status_acc = {"states": {}, "comp": 0, "raw": 0, "verify": {}, "passed_through": set()}
    pool_of: Dict[str, int] = {}
    sent = done = 0
    total_bytes = 0
    t0 = None
    try:
        deadline = time.time() + timeout_s
        while done < n_requests:
            if err_ev.is_set():
                raise RuntimeError("operator failed:\n" + err_q.get(timeout=5))
            if time.time() > deadline:
                raise TimeoutError(f"harness timed out with {done}/{n_requests} chunks done")
            fresh = []
            while sent < n_requests and sent - done < window and len(fresh) < 256:
                k = sent % len(pool_files)
                cid = uuid.uuid4().hex
                dst = store.get_chunk_file_path(cid)
                try:
                    os.link(pool_files[k], dst)
                except OSError:
                    shutil.copyfile(pool_files[k], dst)
                pool_of[cid] = k
                req = ChunkRequest(Chunk(src_key=f"obj/{k}", dest_key=f"obj/{k}", chunk_id=cid, chunk_length_bytes=pool_lens[k], partition_id="0"))
                if t0 is None and warmup_requests == 0:
                    t0 = time.perf_counter()
                fresh.append(req)
                sent += 1
            store.add_chunk_requests(fresh)  # (what the gateway API does per POST of a chunk-request list)
            _drain_status(store, status_acc)
            finished = qout.get_batch_nowait(1024)
            if not finished:
                time.sleep(0.0005)
                continue
            for r in finished:
                done += 1
                if done <= warmup_requests:
                    if done == warmup_requests:
                        t0 = time.perf_counter()
                else:
                    total_bytes += r.chunk.chunk_length_bytes
                cid = r.chunk.chunk_id
                rec = {
                    "chunk_id": cid,
                    "pool_index": pool_of.pop(cid),
                    "md5": r.chunk.md5_hash.hex() if r.chunk.md5_hash else None,
                    "raw_len": r.chunk.chunk_length_bytes,
                    "frame_path": str(store.get_compressed_file_path(cid)) if keep_frames else None,
                }
                records.append(rec)
                if on_done is not None:
                    on_done(r)
                store.get_chunk_file_path(cid).unlink(missing_ok=True)  # what the API thread does after the terminal op
        wall = time.perf_counter() - t0 if t0 is not None else 0.0
    finally:
        # children flush their status records while exiting: keep draining or join() would block on a full pipe
        for flag in op.exit_flags:
            flag.set()
        while any(p.is_alive() for p in op.processes):
            _drain_status(store, status_acc)
            time.sleep(0.002)
        op.stop_workers()
    # this process logged the "registered" records itself: give its feeder thread a moment to flush them, drain, and do
    # not let interpreter exit block on records nobody will read
    for _ in range(50):
        _drain_status(store, status_acc)
        if sum(status_acc["states"].values()) >= 3 * sent:
            break
        time.sleep(0.01)
    store.chunk_status_queue.cancel_join_thread()
    status, comp, raw = status_acc["states"], status_acc["comp"], status_acc["raw"]
    return {"wall_s": wall, "bytes": total_bytes, "records": records, "status": status, "compressed_bytes": comp, "uncompressed_bytes": raw,
            "frame_verify": status_acc["verify"], "passed_through": sorted(status_acc["passed_through"])}


def main():
    ap = argparse.ArgumentParser(description="Stream synthetic chunks through GatewayCompressHash workers (one per GPU)")
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--chunks", type=int, default=256)
    ap.add_argument("--chunk-mib", type=float, default=8)
    ap.add_argument("--pool", type=int, default=32)
    ap.add_argument("--workload", choices=["random", "silesia", "mixed"], default="mixed")
    ap.add_argument("--batch", type=int, default=128, help="chunks per kernel launch")
    ap.add_argument("--slots", type=int, default=4, help="staging slots per worker (one being read into, the others on the GPU)")
    ap.add_argument("--warmup", type=int, default=-1, help="untimed leading requests (default: 4 batches per GPU)")
    ap.add_argument("--dir", default=None)
    a = ap.parse_args()
    from skyplane_b200 import synth

    n = int(a.chunk_mib * (1 << 20))
    base = Path(a.dir or tempfile.mkdtemp(prefix="skyb200_", dir="/dev/shm" if os.path.isdir("/dev/shm") else None))
    pool_dir = base / "pool"
    pool_dir.mkdir(parents=True, exist_ok=True)
    import hashlib

    files, lens, digests = [], [], []
    for k in range(a.pool):
        kind = a.workload if a.workload != "mixed" else ("random" if k % 2 else "silesia")
        data = synth.random_chunk(3000 + k, n) if kind == "random" else synth.silesia_like_chunk(3000 + k, n)
        p = pool_dir / f"{k}.bin"
        p.write_bytes(data)
        files.append(p)
        lens.append(n)
        digests.append(hashlib.md5(data).hexdigest())  # hashlib = the reference's own call (s3_interface.py:181)
    try:
        warm = a.warmup if a.warmup >= 0 else (a.slots + 1) * a.batch * a.gpus
        res = run_stream(base / "chunks", files, lens, a.chunks + warm, n_workers=a.gpus, n_gpus=a.gpus, max_batch_chunks=a.batch,
                         max_batch_bytes=max(n * a.batch, 64 << 20), keep_frames=False, window=max(256, (a.slots + 2) * a.batch * a.gpus), n_slots=a.slots,
                         warmup_requests=warm)
        bad = [r["chunk_id"] for r in res["records"] if r["md5"] != digests[r["pool_index"]]]
        if bad:
            raise SystemExit(f"{len(bad)} chunks came back with a wrong MD5, e.g. {bad[:3]}")
        gbs = res["bytes"] / res["wall_s"] / 1e9
        print(json.dumps({"metric": "gateway-queue end-to-end GB/s (raw input)", "value": gbs, "n_gpus": a.gpus, "chunks": a.chunks,
                          "chunk_mib": a.chunk_mib, "wall_s": res["wall_s"], "status": res["status"], "md5_verified": len(res["records"]),
                          "ratio": (res["uncompressed_bytes"] / res["compressed_bytes"]) if res["compressed_bytes"] else None}))
    finally:
        shutil.rmtree(base, ignore_errors=True)


if __name__ == "__main__":
    main()
