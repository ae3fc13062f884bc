"""Remote chunk tier: `LMCACHE_REMOTE_URL=lm://host:port` (helm/templates/deployment-vllm-multi.yaml:
338-345) and the cache server the chart deploys beside the engines
(helm/templates/deployment-cache-server.yaml:62-65 — `lmcache_server 0.0.0.0 <port>`).

* `RemoteServer` / `python -m b200kv.server host port` — the server (C++ threads inside libb200kv.so;
  chunks live in a b200kv pool with the usual LRU).
* `RemoteClient` — one connection (ctypes over the C ABI `b200kv_remote_*`).
* `RemoteTier` — what the connector uses, a `LowerTier` (b200kv/lower_tier.py):
    - scheduler role: `prefetch_state(req_id, tokens)` — fetch the chunks the server holds beyond the local
      pool's prefix INTO THE LOCAL PINNED POOL, while the connector answers vLLM "ask me again";
    - worker role: `push(keys)` — after a store, upload the new chunks in the background.
    A server that fails is not asked again for `retry_s`.
No byte of a chunk passes through Python: sockets <-> pool slots inside the library.
"""
from __future__ import annotations

import ctypes as C
import logging
import threading
import time

import numpy as np

from ._lib import B200KVError, PoolStats, check, lib
from .engine import KVPool
from .lower_tier import LowerTier

logger = logging.getLogger("b200kv")

EIO = -5


def parse_remote_url(url: str | None) -> tuple[str, int] | None:
    """`lm://host:port` (also `b200kv://`, or bare host:port).  None/"" -> no remote tier."""
    if not url:
        return None
    u = url.strip()
    for scheme in ("lm://", "b200kv://", "tcp://"):
        if u.startswith(scheme):
            u = u[len(scheme):]
            break
    else:
        if "://" in u:
            raise ValueError(f"LMCACHE_REMOTE_URL={url!r}: only lm://host:port is supported")
    u = u.rstrip("/")
    host, sep, port = u.rpartition(":")
    if not sep or not host or not port.isdigit():
        raise ValueError(f"LMCACHE_REMOTE_URL={url!r}: expected lm://host:port")
    return host, int(port)


class RemoteServer:
    """In-process cache server (threads live in the library)."""

    def __init__(self, host: str = "0.0.0.0", port: int = 0, pool_bytes: int = 8 << 30):
        h = C.c_void_p()
        check(lib().b200kv_server_start(host.encode(), port, pool_bytes, C.byref(h)), "b200kv_server_start")
        self._h = h
        self.port = lib().b200kv_server_port(h)

    def stats(self) -> dict:
        a = (C.c_uint64 * 5)()
        check(lib().b200kv_server_get_stats(self._h, a), "b200kv_server_get_stats")
        return dict(zip(("n_put", "n_get", "n_get_miss", "bytes_in", "bytes_out"), (int(x) for x in a)))

    def stop(self):
        if self._h:
            lib().b200kv_server_stop(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.stop()
        except Exception:
            pass


class RemoteClient:
    """One TCP connection to a server; calls are serialised inside the library."""

    def __init__(self, host: str, port: int, timeout_ms: int = 5000):
        h = C.c_void_p()
        check(lib().b200kv_remote_connect(host.encode(), port, timeout_ms, C.byref(h)), "b200kv_remote_connect")
        self._h = h

    def ping(self) -> bool:
        return lib().b200kv_remote_ping(self._h) == 0

    def exists(self, keys) -> int:
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        n = C.c_int32(0)
        check(lib().b200kv_remote_exists(self._h, keys.ctypes.data_as(C.POINTER(C.c_uint64)), len(keys), C.byref(n)),
              "b200kv_remote_exists")
        return n.value

    def put(self, pool: KVPool, key: int, owner: int = 0) -> int:
        """0 sent, -EEXIST server already has it, -ENOENT not READY locally, other < 0 = failure."""
        return lib().b200kv_remote_put(self._h, pool.handle, C.c_uint64(int(key)), owner)

    def get(self, pool: KVPool, key: int, owner: int = 0) -> int:
        return lib().b200kv_remote_get(self._h, pool.handle, C.c_uint64(int(key)), owner)

    def stats(self) -> dict:
        st = PoolStats()
        check(lib().b200kv_remote_stats(self._h, C.byref(st)), "b200kv_remote_stats")
        return {f: int(getattr(st, f)) for f, _ in PoolStats._fields_}

    def traffic(self) -> tuple[int, int]:
        up, down = C.c_uint64(0), C.c_uint64(0)
        lib().b200kv_remote_traffic(self._h, C.byref(up), C.byref(down))
        return up.value, down.value

    def close(self):
        if self._h:
            lib().b200kv_remote_close(self._h)
            self._h = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass


class RemoteTier(LowerTier):
    name = "remote"

    def __init__(self, pool: KVPool, host: str, port: int, chunk: int, key_seed, owner: int = 0,
                 include_partial: bool = True, workers: int = 2, wait_s: float = 2.0, timeout_ms: int = 5000,
                 retry_s: float = 5.0, io_conns: int = 4):
        """key_seed: one seed, or one per tensor-parallel rank (the scheduler prefetches every rank's
        chunks of a prompt; each worker pushes its own).  The chunk transfers of ONE prefetch run on
        `io_conns` connections: one TCP stream is bounded by one core's copy rate, the rate scales with
        connections."""
        super().__init__(pool, chunk, key_seed, owner, include_partial, workers=workers, wait_s=wait_s,
                         io_lanes=io_conns)
        self.host, self.port = host, port
        self.timeout_ms, self.retry_s = timeout_ms, retry_s
        self._tls = threading.local()
        self._down_until = 0.0                       # server unreachable: do not stall requests on it

    # ---- connections (one per thread) -------------------------------------------------------------
    def _client(self) -> RemoteClient:
        c = getattr(self._tls, "client", None)
        if c is None:
            c = RemoteClient(self.host, self.port, self.timeout_ms)
            self._tls.client = c
        return c

    def _drop_client(self):
        c = getattr(self._tls, "client", None)
        if c is not None:
            c.close()
            self._tls.client = None

    # ---- LowerTier ----------------------------------------------------------------------------------
    def _usable(self) -> bool:
        return time.monotonic() >= self._down_until

    def _failed(self, what: str, err):
        self.errors += 1
        self._down_until = time.monotonic() + self.retry_s
        self._drop_client()
        logger.warning("b200kv remote tier %s:%d: %s failed (%s); local tier only for %.0f s",
                       self.host, self.port, what, err, self.retry_s)

    def _prefix(self, keys) -> int:
        return self._client().exists(keys)

    def _get(self, key: int) -> int:
        rc = self._client().get(self.pool, key, self.owner)
        if rc == EIO:
            self._drop_client()
            raise B200KVError(rc, "b200kv_remote_get")
        return rc

    def _put(self, key: int) -> int:
        return self._client().put(self.pool, key, self.owner)

    def stats(self) -> dict:
        return {"fetched_chunks": self.fetched_chunks, "pushed_chunks": self.pushed_chunks,
                "push_skipped": self.push_skipped + self.push_present, "errors": self.errors}
