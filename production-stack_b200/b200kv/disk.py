"""Local-disk chunk tier: `LMCACHE_LOCAL_DISK` + `LMCACHE_MAX_LOCAL_DISK_SIZE`
(helm/templates/deployment-vllm-multi.yaml:334-337, operator/internal/controller/vllmruntime_controller.go:558-569).

* `DiskFile` — one handle on the tier's file and its shm index (ctypes over the C ABI `b200kv_disk_*`,
  csrc/b200kv_disk.cpp); every process of a box that opens the same directory shares both.
* `DiskTier` — what the connector uses, a `LowerTier` (b200kv/lower_tier.py):
    - worker role: `push(keys)` writes what the worker stored through to disk after its D2H commit, from a
      bounded queue: when the disk cannot keep up the chunk is skipped and counted, the store path never waits;
    - scheduler role: `prefetch_state(req_id, tokens)` reads the chunks the disk holds beyond the pool's prefix
      into pool slots, several reads in flight, while the connector answers vLLM "ask me again".  After that a
      disk hit is an ordinary pool chunk in its stored format.
No byte of a chunk passes through Python: disk <-> pool slots inside the library.  Nothing on the data path raises:
an I/O error disables the tier with one warning, a chunk that fails its check is a miss.
"""
from __future__ import annotations

import ctypes as C
import errno
import logging
import os
import queue
import struct

import numpy as np

from . import _lib
from ._lib import B200KVError, DiskStats, check, lib
from .engine import KVPool, xxh64
from .lower_tier import LowerTier

logger = logging.getLogger("b200kv")

PUSH_QUEUE = 64    # chunks waiting for the disk: 2 GiB of Llama-3-8B RAW chunks, about a second of NVMe writes
PUSHERS = 2        # one thread hashes a chunk while the other writes one (tools/bench_disk.py)


def file_path(directory: str, chunk_bytes: int) -> str:
    """The tier's file for chunks of chunk_bytes (b200kv_disk_open names it so)."""
    return os.path.join(directory, f"b200kv-disk-{chunk_bytes:x}.slots")


def index_name(directory: str, chunk_bytes: int) -> str:
    """The shm index of that file, named after the file's device, inode and chunk size as b200kv_disk_open names
    it; it outlives the processes on purpose (a restart attaches to it) and can be removed once none is open."""
    st = os.stat(file_path(directory, chunk_bytes))
    return "/b200kv-disk-%016x" % xxh64(struct.pack("<QQQ", st.st_dev, st.st_ino, chunk_bytes), 0)


class DiskFile:
    """The tier's file in `directory` for chunks of `chunk_bytes`, sized to `disk_bytes` when it is created."""

    def __init__(self, directory: str, disk_bytes: int, chunk_bytes: int):
        h = C.c_void_p()
        check(lib().b200kv_disk_open(directory.encode(), disk_bytes, chunk_bytes, C.byref(h)),
              f"b200kv_disk_open({directory})")
        self._h = h

    @property
    def handle(self) -> C.c_void_p:
        if self._h is None:
            raise RuntimeError("disk tier is closed")
        return self._h

    def put(self, pool: KVPool, key: int, owner: int = 0) -> int:
        return lib().b200kv_disk_put(self.handle, pool.handle, C.c_uint64(int(key)), owner)

    def get(self, pool: KVPool, key: int) -> int:
        return lib().b200kv_disk_get(self.handle, pool.handle, C.c_uint64(int(key)))

    def lookup(self, keys) -> int:
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        n = C.c_int32(0)
        check(lib().b200kv_disk_lookup(self.handle, keys.ctypes.data_as(C.POINTER(C.c_uint64)), len(keys),
                                       C.byref(n)), "b200kv_disk_lookup")
        return n.value

    def stats(self) -> dict:
        st = DiskStats()
        check(lib().b200kv_disk_get_stats(self.handle, C.byref(st)), "b200kv_disk_get_stats")
        return st.as_dict()

    def clear(self) -> bool:
        rc = lib().b200kv_disk_clear(self.handle)
        if rc == _lib.EBUSY:
            return False
        check(rc, "b200kv_disk_clear")
        return True

    def close(self):
        if self._h is not None:
            lib().b200kv_disk_close(self._h)
            self._h = None


class DiskTier(LowerTier):
    name = "disk"

    def __init__(self, pool: KVPool, directory: str, disk_bytes: int, chunk: int, key_seed, owner: int = 0,
                 include_partial: bool = True, wait_s: float = 2.0, io_lanes: int = 4, push_queue: int = PUSH_QUEUE,
                 pushers: int = PUSHERS, prefix_lease_ms: int = 30000):
        """Raises B200KVError when the directory cannot hold the tier (missing, not writable, no room for the
        preallocation): the caller runs without it."""
        self.directory = directory
        self.file = DiskFile(directory, disk_bytes, pool.stats()["slot_bytes"])
        super().__init__(pool, chunk, key_seed, owner, include_partial, wait_s=wait_s, io_lanes=io_lanes,
                         push_queue=push_queue, pushers=pushers, prefix_lease_ms=prefix_lease_ms)
        self._disabled = False

    # ---- LowerTier ----------------------------------------------------------------------------------
    def _usable(self) -> bool:
        return not self._disabled

    def _failed(self, what: str, err):
        with self._inflight_mu:           # several pushers and prefetch lanes may fail at once: one warning
            self.errors += 1
            first = not (self._disabled or self._closed)
            self._disabled = True
        if first:
                logger.warning("b200kv disk tier %s: %s failed (%s); the disk tier is off from now on", self.directory,
                           what, err)

    def _io_error(self, rc: int, where: str):
        e = self.file.stats()["last_errno"]
        raise B200KVError(rc, f"{where} ({errno.errorcode.get(e, e)})")

    def _prefix(self, keys) -> int:
        return self.file.lookup(keys)

    def _get(self, key: int) -> int:
        rc = self.file.get(self.pool, key)
        if rc == _lib.EIO:
            self._io_error(rc, "b200kv_disk_get")
        return rc

    def _put(self, key: int) -> int:
        rc = self.file.put(self.pool, key, self.owner)
        if rc == _lib.EIO:
            self._io_error(rc, "b200kv_disk_put")
        return rc

    # ---- connector surface --------------------------------------------------------------------------
    def clear(self) -> bool:
        """reset_cache: empty the index and retire every chunk on disk."""
        try:
            return self.file.clear()
        except Exception as e:
            self._failed("clear", e)
            return False

    def stats(self) -> dict:
        fs = self.file.stats() if self.file._h is not None else {}
        return {"fetched_chunks": self.fetched_chunks, "written_chunks": self.pushed_chunks,
                "skipped_chunks": self.push_skipped, "present_chunks": self.push_present,
                "corrupt_chunks": fs.get("n_corrupt", 0),
                "usage_bytes": fs.get("n_used", 0) * fs.get("slot_bytes", 0),
                "capacity_bytes": fs.get("n_slots", 0) * fs.get("slot_bytes", 0),
                "direct_io": bool(fs.get("direct_io", 0)), "errors": self.errors, "enabled": not self._disabled}

    def close(self):
        self._closed = True
        while True:                        # what is still queued is not written
            try:
                item = self._push_q.get_nowait()
            except queue.Empty:
                break
            if item is not None:
                self._settled("push_skipped")
        pushers = self._pushers
        super().close()
        self._exec.shutdown(wait=True, cancel_futures=True)
        self._io.shutdown(wait=True, cancel_futures=True)
        if not any(t.is_alive() for t in pushers):
            self.file.close()              # else a write is stuck in the kernel: keep the handle it uses
