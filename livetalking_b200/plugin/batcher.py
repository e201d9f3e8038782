"""Cross-session batching scheduler (SURVEY §8 f1).

The reference serves up to ``max_session`` sessions against ONE shared model (app.py:76-100, server/session_manager.py:56-83)
and runs one forward pass per session per step (avatars/base_avatar.py:337-381).  At 32 sessions per GPU that is 32
under-filled launches per 40 ms frame period; the engine is two orders of magnitude faster than any single session can
feed it.  Here sessions keep the reference's per-session threads and queues, but their ``inference_batch`` calls do not own a
network: every frame becomes a *slot request* (avatar handle, mirror-indexed frame number, mel window), a dispatcher
thread packs requests of ALL sessions into batches of up to B slots and serves each batch with one engine call
(``ltb_w2l_infer_slots``: one forward graph + one paste launch + one D2H), then hands every session its own frames.

Latency rule: a batch is dispatched when it is full or when its oldest request has waited ``max_wait_ms`` — a lone session is
never held back for longer than that.  Requests of one ``submit`` call keep their order and are never split across more
than the necessary number of batches."""
from __future__ import annotations

import os
import threading
import time
from collections import deque
from typing import List, Sequence

import numpy as np


class _Ticket:
    __slots__ = ("requests", "frames", "remaining", "done", "error")

    def __init__(self, requests):
        self.requests = requests
        self.frames: List = [None] * len(requests)
        self.remaining = len(requests)
        self.done = threading.Event()
        self.error = None


class CrossSessionBatcher:
    """``mux``: an engine session created with ``slots=True`` (``engine.W2LSession.infer_slots``) — or any object with the same
    ``infer_slots(requests) -> (n, H, W, 3) uint8`` method and a ``batch`` attribute."""

    def __init__(self, mux, max_wait_ms: float = 4.0):
        self.mux, self.B, self.max_wait = mux, int(mux.batch), max_wait_ms / 1000.0
        self._q = deque()                       # (ticket, position, request, t_submit)
        self._cv = threading.Condition()
        self._stop = False
        self.batches = 0                        # statistics: engine calls, slots served
        self.slots = 0
        self._thread = threading.Thread(target=self._run, name="ltb-cross-session-batcher", daemon=True)
        self._thread.start()

    # ---- session side
    def submit(self, requests: Sequence[tuple]) -> List[np.ndarray]:
        """requests: [(engine avatar, frame idx, mel (80,16) float32), ...] of ONE session step -> its composited frames, in order.
        Blocks the calling (inference) thread until all of them are served."""
        if not requests:
            return []
        t = _Ticket(list(requests))
        now = time.monotonic()
        with self._cv:
            if self._stop:
                raise RuntimeError("CrossSessionBatcher is closed")
            for i, r in enumerate(t.requests):
                self._q.append((t, i, r, now))
            self._cv.notify()
        t.done.wait()
        if t.error is not None:
            raise t.error
        return t.frames

    # ---- dispatcher
    def _take_batch(self):
        with self._cv:
            while not self._stop:
                if self._q:
                    oldest = self._q[0][3]
                    if len(self._q) >= self.B or time.monotonic() - oldest >= self.max_wait:
                        return [self._q.popleft() for _ in range(min(self.B, len(self._q)))]
                    self._cv.wait(timeout=max(0.0, self.max_wait - (time.monotonic() - oldest)))
                else:
                    self._cv.wait()
            return None

    def _run(self):
        while True:
            batch = self._take_batch()
            if batch is None:
                return
            try:
                frames = self.mux.infer_slots([b[2] for b in batch])
                err = None
            except Exception as e:               # noqa: BLE001 - handed to every waiting session, the dispatcher keeps running
                frames, err = None, e
            self.batches += 1
            self.slots += len(batch)
            for j, (t, pos, _r, _ts) in enumerate(batch):
                if err is not None:
                    t.error = err
                else:
                    t.frames[pos] = frames[j]
                t.remaining -= 1
                if t.remaining == 0:
                    t.done.set()

    def close(self):
        with self._cv:
            self._stop = True
            pending = list(self._q)
            self._q.clear()
            self._cv.notify_all()
        for t, _pos, _r, _ts in pending:
            t.error = RuntimeError("CrossSessionBatcher closed")
            t.done.set()
        self._thread.join(timeout=5)


_SHARED_LOCK = threading.Lock()


def shared_scheduler(owner, table_attr: str, key, make_mux) -> CrossSessionBatcher:
    """The CrossSessionBatcher of `key` in the table ``owner.<table_attr>``, created by the first session that asks and shared by all
    later ones.  make_mux() builds its engine mux; its dispatch deadline is LTB_MUX_WAIT_MS (default 4 ms).  The owner is the model
    whose weights the mux runs, so its schedulers live as long as it does."""
    with _SHARED_LOCK:
        table = getattr(owner, table_attr, None)
        if table is None:
            table = {}
            setattr(owner, table_attr, table)
        if key not in table:
            table[key] = CrossSessionBatcher(make_mux(), float(os.environ.get("LTB_MUX_WAIT_MS", "4")))
        return table[key]


class SharedFeatures:
    """An ASR's feature extractor in cross-session mode (HubertASR, WhisperASR): run(pcm) is one group request of a shared feature
    scheduler and blocks until its round is served.  The scheduler and its graph belong to the model, so close() releases nothing."""

    def __init__(self, batcher: CrossSessionBatcher):
        self.batcher = batcher

    def run(self, pcm: np.ndarray) -> np.ndarray:
        return self.batcher.submit([pcm])[0]

    def close(self):
        pass
