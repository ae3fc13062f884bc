"""What every chunk tier below the local pinned pool does the same way (b200kv/remote.py: the `lm://` cache
server, b200kv/disk.py: local disk):

* scheduler role: `prefetch_state(req_id, tokens)` — when the local pool holds less than the whole prompt, ask the
  tier which of the following chunks it has and fetch them INTO THE LOCAL PINNED POOL on a background thread, over
  several lanes at once; the connector answers vLLM "ask me again" (`(None, False)`,
  KVConnectorBase_V1.get_num_new_matched_tokens, base.py:453-486) until that is done or `wait_s` has passed, then
  the ordinary local lookup sees the chunks and the ordinary load path moves them to the GPU.  One prefetch per
  request; chunks that arrive late still land in the pool for the next request.
* worker role: `push(keys)` — after a store, copy the new chunks into the tier in the background, once their D2H
  has committed them to the pool, on `pushers` threads.  With `push_queue` > 0 the queue is bounded and a chunk that
  finds it full is skipped (counted), so the store path never waits for the tier.

A subclass supplies the transfers: `_prefix(keys)` (how many leading keys the tier holds), `_get(key)` and
`_put(key)` (0 or a negative code; raise on a failure of the tier itself), `_usable()` and `_failed(what, err)`.
"""
from __future__ import annotations

import queue
import threading
import time
from concurrent.futures import Future, ThreadPoolExecutor

import numpy as np

from . import _lib
from ._lib import B200KVError
from .engine import KVPool, chunk_keys


class LowerTier:
    PENDING, DONE = "pending", "done"
    name = "tier"

    def __init__(self, pool: KVPool, chunk: int, key_seed, owner: int = 0, include_partial: bool = True,
                 workers: int = 2, wait_s: float = 2.0, io_lanes: int = 4, push_queue: int = 0, pushers: int = 1,
                 prefix_lease_ms: int = 0):
        """key_seed: one seed, or one per tensor-parallel rank (the scheduler prefetches every rank's
        chunks of a prompt; each worker pushes its own).  prefix_lease_ms > 0: the chunks of the prompt already in
        the pool are leased that long when a prefetch starts, so the fetched chunks cannot evict the prefix they
        extend from a pool that is small against the prompt."""
        self.pool = pool
        self.key_seeds = [int(x) for x in (key_seed if isinstance(key_seed, (list, tuple)) else [key_seed])]
        self.chunk, self.owner, self.include_partial = chunk, owner, include_partial
        self.wait_s, self.prefix_lease_ms = wait_s, prefix_lease_ms
        self._exec = ThreadPoolExecutor(max_workers=workers, thread_name_prefix=f"b200kv-{self.name}")
        self._io = ThreadPoolExecutor(max_workers=max(1, io_lanes), thread_name_prefix=f"b200kv-{self.name}-io")
        self._io_lanes = max(1, io_lanes)
        self._jobs: dict[str, tuple[Future, float]] = {}
        self._asked: set[str] = set()                # requests whose one prefetch has been answered
        self._push_q: queue.Queue = queue.Queue(maxsize=push_queue)
        self._n_pushers = max(1, pushers)
        self._pushers: list[threading.Thread] = []
        self._closed = False
        self._inflight = 0                           # chunks queued or being copied
        self._inflight_mu = threading.Lock()         # guards _inflight and the push counters
        self.fetched_chunks = 0
        self.pushed_chunks = 0
        self.push_skipped = 0                        # not copied: tier unusable, queue full, no room, not stored
        self.push_present = 0                        # not copied: the tier had it already
        self.errors = 0

    # ---- what a tier supplies ---------------------------------------------------------------------
    def _usable(self) -> bool:
        return True

    def _failed(self, what: str, err):
        self.errors += 1

    def _prefix(self, keys) -> int:
        raise NotImplementedError

    def _get(self, key: int) -> int:
        raise NotImplementedError

    def _put(self, key: int) -> int:
        raise NotImplementedError

    # ---- scheduler role ---------------------------------------------------------------------------
    def _get_some(self, keys) -> int:
        got = 0
        for k in keys:
            if self._get(int(k)) != 0:      # evicted meanwhile / no local room: nothing behind it is useful
                break
            got += 1
        return got

    def _fetch(self, missing: list[np.ndarray]) -> int:
        try:
            got = 0
            for keys in missing:
                n = self._prefix(keys)
                lanes = min(self._io_lanes, n)
                futs = [self._io.submit(self._get_some, keys[i:n:lanes]) for i in range(lanes)]
                got += sum(f.result() for f in futs)
            self.fetched_chunks += got
            return got
        except Exception as e:
            self._failed("prefetch", e)
            return 0

    def prefetch_state(self, req_id: str, tokens) -> str:
        """PENDING while chunks of this prompt are on their way from the tier, else DONE.
        Never raises; a failed tier degrades to the local pool."""
        job = self._jobs.get(req_id)
        now = time.monotonic()
        if job is not None:
            fut, t0 = job
            if fut.done() or now - t0 > self.wait_s:
                self._jobs.pop(req_id, None)      # late chunks still land in the pool for the next turn
                self._asked.add(req_id)           # one prefetch per request, however often vLLM asks
                return self.DONE
            return self.PENDING
        if self._closed or not self._usable() or req_id in self._asked:
            return self.DONE
        missing = []
        for seed in self.key_seeds:
            keys = chunk_keys(tokens, self.chunk, seed, self.include_partial)
            n_local = self.pool.lookup_owner(keys)[0] if len(keys) else 0
            if n_local < len(keys):
                missing.append(keys[n_local:].copy())
                if n_local and self.prefix_lease_ms:
                    self.pool.contains(keys[:n_local], None, self.prefix_lease_ms)
        if not missing:
            return self.DONE
        self._jobs[req_id] = (self._exec.submit(self._fetch, missing), now)
        return self.PENDING

    def forget(self, req_id: str):
        self._jobs.pop(req_id, None)
        self._asked.discard(req_id)

    # ---- worker role ------------------------------------------------------------------------------
    def push(self, keys):
        """Copy these chunks into the tier once they are READY in the local pool (the D2H of a store is
        still in flight when this is called)."""
        if self._closed:
            return
        if not self._pushers:
            self._pushers = [threading.Thread(target=self._push_loop, name=f"b200kv-{self.name}-push", daemon=True)
                             for _ in range(self._n_pushers)]
            for t in self._pushers:
                t.start()
        for k in keys:
            with self._inflight_mu:
                self._inflight += 1
            try:
                self._push_q.put_nowait((int(k), time.monotonic()))
            except queue.Full:                      # the tier cannot keep up: this chunk is not copied
                self._settled("push_skipped")

    def _settled(self, counter: str | None = None):
        with self._inflight_mu:
            self._inflight -= 1
            if counter is not None:
                setattr(self, counter, getattr(self, counter) + 1)

    def _push_loop(self):
        while True:
            item = self._push_q.get()
            if item is None:
                return
            key, t0 = item
            if not self._usable():
                self._settled("push_skipped")
                continue
            counter = None
            try:
                rc = self._put(key)
                if rc == _lib.ENOENT and time.monotonic() - t0 < 10.0:
                    time.sleep(0.002)                       # not committed yet: try again shortly
                    try:
                        self._push_q.put_nowait((key, t0))
                        continue
                    except queue.Full:
                        pass
                if rc == 0:
                    counter = "pushed_chunks"
                elif rc == _lib.EEXIST:
                    counter = "push_present"
                elif rc in (_lib.ENOENT, _lib.ENOSPC):
                    counter = "push_skipped"
                else:
                    raise B200KVError(rc, f"{self.name} put")
            except Exception as e:
                self._failed("push", e)
            self._settled(counter)

    def flush(self, timeout_s: float = 30.0) -> bool:
        """Wait until the push queue is drained (tests, shutdown)."""
        t0 = time.monotonic()
        while time.monotonic() - t0 < timeout_s:
            with self._inflight_mu:
                if self._inflight <= 0:
                    return True
            time.sleep(0.005)
        return False

    def close(self):
        self._closed = True
        for _ in self._pushers:
            self._push_q.put(None)
        for t in self._pushers:
            t.join(timeout=5)
        self._exec.shutdown(wait=False, cancel_futures=True)
        self._io.shutdown(wait=False, cancel_futures=True)
