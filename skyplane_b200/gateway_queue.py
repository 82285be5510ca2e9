"""Inter-operator queues of the gateway (API-compatible with skyplane/gateway/gateway_queue.py:4-61).

* ``GatewayQueue``    -- one bounded multiprocessing queue shared by the workers of the consuming operator.
* ``GatewayANDQueue`` -- fan-out: every registered consumer handle gets its own ``GatewayQueue`` and sees every item.

``get_batch_nowait`` is ours: the H100 operator drains many requests per kernel launch.
"""
from __future__ import annotations

import multiprocessing
import queue as _queue
from collections import deque
from typing import Dict, Iterable, List

DEFAULT_DEPTH = 10000  # the reference's maxsize


class _Batch:
    """Several requests travelling as one queue element (see GatewayQueue.put_many)."""

    __slots__ = ("items",)

    def __init__(self, items):
        self.items = items


class GatewayQueue:
    """FIFO of ChunkRequests between two operators."""

    def __init__(self, maxsize: int = DEFAULT_DEPTH):
        self.q = multiprocessing.Queue(maxsize)
        self.handles: List[str] = []
        self._pending = deque()  # process-local: requests of a batch already taken off the queue

    # -- consumers ------------------------------------------------------------------------------
    def register_handle(self, requester_handle) -> None:
        self.handles.append(requester_handle)

    def get_handles(self) -> List[str]:
        return self.handles

    def get_nowait(self, requester_handle=None):
        """Next request or ``queue.Empty``.  (``put_many`` ships a whole list as one queue element -- one pickle, one pipe
        write, one wake-up instead of one per request; the consumer unpacks it here, so callers never see the difference.)"""
        if self._pending:
            return self._pending.popleft()
        item = self.q.get_nowait()
        if isinstance(item, _Batch):
            self._pending.extend(item.items)
            return self._pending.popleft()
        return item

    def get_batch_nowait(self, max_items: int, requester_handle=None) -> list:
        """Up to ``max_items`` requests that are available right now (possibly none)."""
        batch: list = []
        while len(batch) < max_items:
            try:
                batch.append(self.get_nowait(requester_handle))
            except _queue.Empty:
                break
        return batch

    def pop(self, requester_handle=None) -> None:
        if self._pending:
            self._pending.popleft()
            return
        item = self.q.get()
        if isinstance(item, _Batch):
            self._pending.extend(item.items[1:])

    # -- producers ------------------------------------------------------------------------------
    def put(self, chunk_req) -> None:
        self.q.put(chunk_req)

    def put_nowait(self, chunk_req) -> None:
        self.q.put_nowait(chunk_req)

    def put_many(self, chunk_reqs: Iterable) -> None:
        items = list(chunk_reqs)
        if len(items) == 1:
            self.q.put(items[0])
        elif items:
            self.q.put(_Batch(items))

    def size(self) -> int:
        return self.q.qsize() + len(self._pending)


class GatewayANDQueue(GatewayQueue):
    """Broadcast queue: ``put`` delivers to every consumer's private queue (used behind ``mux_and``)."""

    def __init__(self, maxsize: int = DEFAULT_DEPTH):
        self.maxsize = maxsize
        self.q: Dict[str, GatewayQueue] = {}  # handle -> private queue
        self.temp_q = multiprocessing.Queue(maxsize)

    def register_handle(self, requester_handle) -> None:
        self.q[requester_handle] = GatewayQueue(self.maxsize)

    def get_handles(self) -> List[str]:
        return list(self.q)

    def get_handle_queue(self, requester_handle) -> GatewayQueue:
        return self.q[requester_handle]

    def get_nowait(self, requester_handle):
        return self.q[requester_handle].get_nowait()

    def pop(self, requester_handle) -> None:
        self.q[requester_handle].pop()

    def put(self, chunk_req) -> None:
        for private in self.q.values():
            private.put(chunk_req)

    def put_many(self, chunk_reqs: Iterable) -> None:
        items = list(chunk_reqs)
        for private in self.q.values():
            private.put_many(items)

    def put_nowait(self, chunk_req) -> None:
        raise ValueError("GatewayANDQueue cannot be the first queue in a pipeline")

    def size(self) -> int:
        return max((private.size() for private in self.q.values()), default=0)
