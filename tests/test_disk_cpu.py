"""Local-disk chunk tier (CPU): LMCACHE_LOCAL_DISK + LMCACHE_MAX_LOCAL_DISK_SIZE
(helm/templates/deployment-vllm-multi.yaml:334-337).  Chunks travel pool slot <-> file slot inside libb200kv.so;
bytes, format tag, token count and owner must survive the round trip exactly, a damaged slot must never be
loaded, and the tier must survive a restart of every process that uses it."""
import importlib.util
import logging
import os
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np
import pytest

from b200kv import KVPool, _lib
from b200kv.config import B200KVConfig, default_disk_dir
from b200kv.disk import DiskFile, DiskTier, file_path, index_name
from b200kv.engine import chunk_keys
from b200kv.lower_tier import LowerTier

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SLOT = 64 * 1024 + 256          # a pool slot that is not a whole number of 4 KiB blocks: the tail is bounced
STRIDE = 4096 + 68 * 1024       # one disk slot of it: header + chunk rounded up to 4 KiB


def disk_bytes(n_slots, stride=STRIDE):
    return 4096 + n_slots * stride


def mk_pool(n_slots=8, slot=SLOT):
    return KVPool(None, n_slots * slot, slot, _lib.POOL_CREATE)


def put_local(pool, key, n_tok=256, seed=0, fmt=0, owner=0):
    slot = pool.reserve(int(key), n_tok, fmt, owner)
    view = pool.slot_view(slot)
    data = np.random.default_rng(seed).integers(0, 256, len(view), dtype=np.uint8)
    view[:] = data
    pool.commit(int(key))
    return data


def read_local(pool, key):
    slot, n_tok, fmt = pool.acquire(int(key))
    out = pool.slot_view(slot).copy()
    pool.release(int(key))
    return out, n_tok, fmt


def slot_of(directory, chunk_bytes, key):
    """File slot of a key, read from the shared index."""
    idx = KVPool(index_name(directory, chunk_bytes), 0, 16, _lib.POOL_ATTACH)
    try:
        slot = idx.acquire(int(key))[0]
        idx.release(int(key))
        return slot
    finally:
        idx.close()


@pytest.fixture
def ddir(tmp_path):
    """A tier directory; the shm indices of the files made in it are removed afterwards."""
    d = tmp_path / "disk"
    d.mkdir()
    yield str(d)
    for f in os.listdir(d):
        if f.endswith(".slots"):
            KVPool.unlink(index_name(str(d), int(f[len("b200kv-disk-"):-len(".slots")], 16)))


@pytest.mark.parametrize("slot", [SLOT, 64 * 1024])    # bounced tail / every byte direct
def test_roundtrip_into_another_pool_is_bit_exact(ddir, slot):
    a, b = mk_pool(8, slot), mk_pool(8, slot)
    d = DiskFile(ddir, disk_bytes(4, 4096 + (slot + 4095) // 4096 * 4096), slot)
    want = {}
    for i, (key, n_tok, fmt, owner) in enumerate([(101, 256, 0, 7), (102, 256, 1 | 1 << 8 | 1 << 24, 8),
                                                  (103, 40, 2 | 1 << 16, 9)]):
        want[key] = (put_local(a, key, n_tok, i, fmt, owner), n_tok, fmt, owner)
        assert d.put(a, key, owner) == 0
    assert d.put(a, 101, 7) == _lib.EEXIST            # on disk already: nothing written
    assert d.put(a, 999, 7) == _lib.ENOENT            # not in the local pool
    assert d.lookup(np.array([101, 102, 103, 104], np.uint64)) == 3
    assert d.lookup(np.array([104, 101], np.uint64)) == 0
    for key, (data, n_tok, fmt, owner) in want.items():
        assert d.get(b, key) == 0
        got, n2, f2 = read_local(b, key)
        assert np.array_equal(got, data) and (n2, f2) == (n_tok, fmt)
        assert list(b.lookup_owner(np.array([key], np.uint64))[1]) == [owner]
    assert d.get(b, 101) == 0                         # already local: fine
    assert d.get(b, 555) == _lib.ENOENT
    st = d.stats()
    assert (st["n_put"], st["n_get"], st["n_get_miss"], st["n_used"]) == (3, 3, 1, 3)
    assert st["bytes_written"] == st["bytes_read"] == 3 * slot and st["direct_io"] == 1
    assert os.path.getsize(file_path(ddir, slot)) <= disk_bytes(4, 4096 + (slot + 4095) // 4096 * 4096)
    d.close()


def test_lru_at_capacity_and_pins_block_eviction(ddir):
    a = mk_pool(16)
    d = DiskFile(ddir, disk_bytes(4), SLOT)
    for k in range(1, 5):
        put_local(a, k, seed=k)
        assert d.put(a, k) == 0
    assert d.get(mk_pool(2), 1) == 0                  # a read makes chunk 1 the most recent
    for k in (5, 6):
        put_local(a, k, seed=k)
        assert d.put(a, k) == 0
    present = [k for k in range(1, 7) if d.lookup(np.array([k], np.uint64))]
    assert present == [1, 4, 5, 6] and d.stats()["n_evicted"] == 2
    # a chunk being read is pinned: every other chunk is evicted before it, and with all pinned nothing is
    idx = KVPool(index_name(ddir, SLOT), 0, 16, _lib.POOL_ATTACH)
    for k in (1, 4, 5):
        idx.acquire(k)
    put_local(a, 7, seed=7)
    assert d.put(a, 7) == 0
    assert [k for k in range(1, 8) if d.lookup(np.array([k], np.uint64))] == [1, 4, 5, 7]
    idx.acquire(7)
    put_local(a, 8, seed=8)
    assert d.put(a, 8) == _lib.ENOSPC and d.stats()["n_dropped"] == 1
    for k in (1, 4, 5, 7):
        idx.release(k)
    assert d.put(a, 8) == 0
    assert idx.check()
    idx.close()
    d.close()


_WRITER = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1])
from b200kv import KVPool
from b200kv.disk import DiskFile
directory, first, n, slot, n_disk = sys.argv[2], int(sys.argv[3]), int(sys.argv[4]), int(sys.argv[5]), int(sys.argv[6])
pool = KVPool(None, 4 * slot, slot, 1)
d = DiskFile(directory, n_disk, slot)
for k in range(first, first + n):
    s = pool.reserve(k, 256, 0, first)
    pool.slot_view(s)[:] = np.random.default_rng(k).integers(0, 256, slot, dtype=np.uint8)
    pool.commit(k)
    assert d.put(pool, k, first) == 0
d.close()
"""


def _run_writers(ddir, ranges, n_disk):
    pkg = os.path.join(ROOT, "production-stack_b200")
    procs = [subprocess.Popen([sys.executable, "-c", _WRITER, pkg, ddir, str(first), str(n), str(SLOT), str(n_disk)])
             for first, n in ranges]
    assert [p.wait(timeout=120) for p in procs] == [0] * len(procs)


def test_two_processes_write_one_directory_then_the_index_checks(ddir):
    _run_writers(ddir, [(1000, 24), (2000, 24)], disk_bytes(64))
    idx = KVPool(index_name(ddir, SLOT), 0, 16, _lib.POOL_ATTACH)
    assert idx.check() and idx.stats()["n_used"] == 48
    idx.close()
    d, b = DiskFile(ddir, disk_bytes(64), SLOT), mk_pool(64)
    for k in list(range(1000, 1024)) + list(range(2000, 2024)):
        assert d.get(b, k) == 0
        got, _, _ = read_local(b, k)
        assert np.array_equal(got, np.random.default_rng(k).integers(0, 256, SLOT, dtype=np.uint8))
        assert list(b.lookup_owner(np.array([k], np.uint64))[1]) == [k // 1000 * 1000]
    d.close()


def test_restart_rebuilds_the_index_from_the_file(ddir):
    _run_writers(ddir, [(1, 10)], disk_bytes(16))
    d = DiskFile(ddir, disk_bytes(16), SLOT)          # the index in shm survived: attached, nothing to rebuild
    assert d.stats()["n_restored"] == 0 and d.lookup(np.arange(1, 11, dtype=np.uint64)) == 10
    d.close()
    KVPool.unlink(index_name(ddir, SLOT))             # as after a reboot or a new pod: no index in shm
    d = DiskFile(ddir, disk_bytes(32), SLOT)          # the file keeps the size it was created with
    st = d.stats()
    assert st["n_restored"] == 10 and st["n_slots"] == 16 and st["n_corrupt"] == 0
    b = mk_pool(16)
    for k in range(1, 11):
        assert d.get(b, k) == 0
        assert np.array_equal(read_local(b, k)[0], np.random.default_rng(k).integers(0, 256, SLOT, dtype=np.uint8))
    # LRU order survives too: the oldest write goes first
    a = mk_pool(16)
    for k in range(11, 18):
        put_local(a, k, seed=k)
        assert d.put(a, k) == 0
    assert d.lookup(np.array([1], np.uint64)) == 0 and d.stats()["n_used"] == 16
    d.close()


def test_torn_slot_and_garbage_header_are_rejected_and_counted(ddir):
    a, b = mk_pool(8), mk_pool(8)
    d = DiskFile(ddir, disk_bytes(8), SLOT)
    for k in (1, 2, 3):
        put_local(a, k, seed=k)
        assert d.put(a, k) == 0
    path = file_path(ddir, SLOT)
    fd = os.open(path, os.O_RDWR)
    try:
        os.pwrite(fd, b"\xa5" * 4096, 4096 + slot_of(ddir, SLOT, 1) * STRIDE + 4096 + 8192)   # payload after header
        os.pwrite(fd, os.urandom(4096), 4096 + slot_of(ddir, SLOT, 2) * STRIDE)              # header
    finally:
        os.close(fd)
    for k in (1, 2):
        assert d.get(b, k) == _lib.ENOENT                       # never loaded ...
        assert b.lookup_owner(np.array([k], np.uint64))[0] == 0
        assert d.lookup(np.array([k], np.uint64)) == 0          # ... and gone from the index
    assert d.stats()["n_corrupt"] == 2 and b.stats()["n_used"] == 0 and b.check()
    assert d.get(b, 3) == 0
    d.close()
    # a restart trusts headers: a garbage one is counted and not indexed, a torn payload is caught on read
    d = DiskFile(ddir, disk_bytes(8), SLOT)
    assert d.put(a, 1) == 0                                     # stored again after its drop
    fd = os.open(path, os.O_RDWR)
    try:
        os.pwrite(fd, os.urandom(4096), 4096 + slot_of(ddir, SLOT, 3) * STRIDE)
    finally:
        os.close(fd)
    fd = os.open(path, os.O_RDWR)
    try:
        os.pwrite(fd, b"\x5a" * 4096, 4096 + slot_of(ddir, SLOT, 1) * STRIDE + 4096)
    finally:
        os.close(fd)
    d.close()
    KVPool.unlink(index_name(ddir, SLOT))
    d = DiskFile(ddir, disk_bytes(8), SLOT)
    st = d.stats()
    assert st["n_restored"] == 1 and st["n_corrupt"] == 1       # chunk 1; chunk 3's header is garbage
    c = mk_pool(8)
    assert d.get(c, 3) == _lib.ENOENT and d.get(c, 1) == _lib.ENOENT and d.stats()["n_corrupt"] == 2
    assert c.lookup_owner(np.array([1], np.uint64))[0] == 0
    d.close()


def test_unusable_directories_disable_the_tier_with_a_warning(ddir, tmp_path, monkeypatch, caplog):
    pool = mk_pool(4)
    with pytest.raises(_lib.B200KVError) as ei:
        DiskTier(pool, str(tmp_path / "missing"), disk_bytes(4), 16, 1)
    assert ei.value.code == _lib.ENOENT
    with pytest.raises(_lib.B200KVError) as ei:
        DiskTier(pool, ddir, disk_bytes(1 << 30), 16, 1)       # 77 TB: the preallocation does not fit
    assert ei.value.code == _lib.ENOSPC
    assert not os.path.exists(file_path(ddir, SLOT)) or os.path.getsize(file_path(ddir, SLOT)) == 0
    if os.geteuid() != 0:                                      # root writes into a 0555 directory anyway
        ro = tmp_path / "ro"
        ro.mkdir()
        ro.chmod(0o555)
        with pytest.raises(_lib.B200KVError) as ei:
            DiskTier(pool, str(ro), disk_bytes(4), 16, 1)
        assert ei.value.code in (-13, -30)                     # EACCES / EROFS
    # ENOSPC on a write: the tier switches itself off with one warning and the store path carries on
    monkeypatch.setenv("B200KV_DISK_TEST_WRITE_ERRNO", "28")
    tier = DiskTier(pool, ddir, disk_bytes(4), 16, 1)
    caplog.set_level(logging.WARNING, logger="b200kv")
    for k in (1, 2, 3):
        put_local(pool, k, seed=k)
    tier.push([1, 2, 3])
    assert tier.flush(10)
    st = tier.stats()
    assert st["written_chunks"] == 0 and not st["enabled"] and st["skipped_chunks"] + st["errors"] == 3
    warnings = [r for r in caplog.records if "disk tier" in r.getMessage()]
    assert len(warnings) == 1 and "ENOSPC" in warnings[0].getMessage()
    assert tier.prefetch_state("r", np.arange(64, dtype=np.int32)) == LowerTier.DONE
    tier.close()


def test_config_parsing(tmp_path, monkeypatch, caplog):
    monkeypatch.setattr(tempfile, "tempdir", str(tmp_path))
    c = B200KVConfig.from_env({"LMCACHE_LOCAL_DISK": "file:///kv-store-disk/", "LMCACHE_MAX_LOCAL_DISK_SIZE": "640"})
    assert c.disk_dir() == "/kv-store-disk/" and c.disk_bytes == 640 << 30 and c.disk_wait_ms == 2000
    assert B200KVConfig.from_env({"LMCACHE_LOCAL_DISK": "/nvme/kv", "LMCACHE_MAX_LOCAL_DISK_SIZE": "0.5"}).disk_dir() \
        == "/nvme/kv"
    for v in ("True", "1", "true"):                            # what the operator emits
        c = B200KVConfig.from_env({"LMCACHE_LOCAL_DISK": v, "LMCACHE_MAX_LOCAL_DISK_SIZE": "5",
                                   "B200KV_DISK_WAIT_MS": "300"})
        assert c.disk_dir() == default_disk_dir() == os.path.join(str(tmp_path), "b200kv-disk")
        assert c.disk_wait_ms == 300
    c = B200KVConfig.from_env({}).apply_extra({"lmcache.local_disk": "file:///x/", "lmcache.max_local_disk_size": 2})
    assert c.disk_dir() == "/x/" and c.disk_bytes == 2 << 30
    assert B200KVConfig.from_env({}).apply_extra({"lmcache.local_disk": True, "lmcache.max_local_disk_size": "1"}) \
        .disk_dir() == default_disk_dir()
    f = tmp_path / "lmcache.yaml"
    f.write_text("local_disk: file:///from-file/\nmax_local_disk_size: 3\n")
    assert B200KVConfig.from_env({"LMCACHE_CONFIG_FILE": str(f)}).disk_dir() == "/from-file/"
    caplog.set_level(logging.WARNING, logger="b200kv")
    c = B200KVConfig.from_env({"LMCACHE_MAX_LOCAL_DISK_SIZE": "640"})          # a size without a path
    assert c.disk_dir() is None
    assert any("LMCACHE_MAX_LOCAL_DISK_SIZE=640 is accepted for chart compatibility but has no effect" in r.getMessage()
               for r in caplog.records)
    for env in ({}, {"LMCACHE_LOCAL_DISK": "/d"}, {"LMCACHE_LOCAL_DISK": "False", "LMCACHE_MAX_LOCAL_DISK_SIZE": "4"},
                {"LMCACHE_LOCAL_DISK": "/d", "LMCACHE_MAX_LOCAL_DISK_SIZE": "0"}):
        assert B200KVConfig.from_env(env).disk_dir() is None
    with pytest.raises(ValueError):
        B200KVConfig.from_env({"LMCACHE_LOCAL_DISK": "s3://bucket", "LMCACHE_MAX_LOCAL_DISK_SIZE": "1"}).disk_dir()


def _wait_done(tier, req, toks, limit=10):
    t0 = time.time()
    while tier.prefetch_state(req, toks) == tier.PENDING:
        assert time.time() - t0 < limit
        time.sleep(0.002)


def test_tier_push_then_prefetch_into_another_pool(ddir):
    C_, seed = 16, 1234
    toks = np.arange(5 * C_ + 3, dtype=np.int32)
    keys = chunk_keys(toks, C_, seed, True)
    prod_pool, cons_pool = mk_pool(8), mk_pool(8)
    data = [put_local(prod_pool, k, min(C_, len(toks) - i * C_), i, owner=1) for i, k in enumerate(keys)]
    prod = DiskTier(prod_pool, ddir, disk_bytes(16), C_, seed, owner=1)
    prod.push(keys)
    assert prod.flush(10) and prod.stats()["written_chunks"] == len(keys)
    prod.push(keys[:2])                                   # stored again: already on disk
    assert prod.flush(10) and prod.stats()["present_chunks"] == 2 and prod.stats()["skipped_chunks"] == 0

    cons = DiskTier(cons_pool, ddir, disk_bytes(16), C_, seed, owner=2)
    put_local(cons_pool, keys[0], C_, 0)                  # first chunk already local: only the rest is read
    assert cons.prefetch_state("r1", toks) == LowerTier.PENDING
    _wait_done(cons, "r1", toks)
    assert cons.stats()["fetched_chunks"] == len(keys) - 1
    assert cons_pool.lookup_owner(keys)[0] == len(keys)
    for i, k in enumerate(keys):
        assert np.array_equal(read_local(cons_pool, k)[0], data[i])
    assert cons.prefetch_state("r1", toks) == LowerTier.DONE           # one prefetch per request
    assert cons.prefetch_state("r2", toks) == LowerTier.DONE           # everything local: no job
    cons_pool.clear()
    assert cons.prefetch_state("r1", toks) == LowerTier.DONE           # still answered: not asked twice
    cons.forget("r1")
    assert cons.prefetch_state("r1", toks) == LowerTier.PENDING        # a new request with the same id
    _wait_done(cons, "r1", toks)
    assert cons.stats()["fetched_chunks"] == 2 * len(keys) - 1
    prod.close()
    cons.close()


def test_prefetch_does_not_evict_the_prefix_it_extends(ddir):
    """A pool that holds one prompt but not two: the chunks read from disk must not push out the prompt's own
    leading chunks that were already local (the lookup afterwards needs the whole prefix)."""
    C_, seed = 16, 99
    toks = np.arange(6 * C_, dtype=np.int32)
    keys = chunk_keys(toks, C_, seed, True)
    src = mk_pool(8)
    for i, k in enumerate(keys):
        put_local(src, k, C_, i)
    writer = DiskTier(src, ddir, disk_bytes(16), C_, seed)
    writer.push(keys)
    assert writer.flush(10) and writer.stats()["written_chunks"] == 6
    pool = mk_pool(8)
    put_local(pool, keys[0], C_, 0)                     # the prompt's first two chunks are local and the oldest
    put_local(pool, keys[1], C_, 1)
    for k in range(5000, 5004):                         # then another prompt's
        put_local(pool, k, C_, k)
    tier = DiskTier(pool, ddir, disk_bytes(16), C_, seed, prefix_lease_ms=5000)
    assert tier.prefetch_state("r", toks) == LowerTier.PENDING
    _wait_done(tier, "r", toks)
    assert tier.stats()["fetched_chunks"] == 4 and pool.lookup_owner(keys)[0] == 6
    writer.close()
    tier.close()


def test_full_queue_skips_instead_of_waiting(ddir):
    pool = mk_pool(8)
    tier = DiskTier(pool, ddir, disk_bytes(8), 16, 1, push_queue=2, pushers=1)
    gate = threading.Event()
    real_put = tier._put
    tier._put = lambda key: (gate.wait(10), real_put(key))[1]         # a disk that does not keep up
    for k in range(1, 7):
        put_local(pool, k, seed=k)
    t0 = time.monotonic()
    tier.push([1])
    time.sleep(0.05)                                                   # the writer holds chunk 1
    tier.push([2, 3, 4, 5, 6])
    assert time.monotonic() - t0 < 1.0                                 # the store path never waited
    assert tier.stats()["skipped_chunks"] == 3                         # 2 and 3 queued, 4..6 skipped
    gate.set()
    assert tier.flush(10) and tier.stats()["written_chunks"] == 3
    tier.close()


# ---- connector ---------------------------------------------------------------------------------------------

vllm_needed = pytest.mark.skipif(importlib.util.find_spec("vllm") is None, reason="needs vllm")


def _connector(monkeypatch, env, role="SCHEDULER", kv_role="kv_both"):
    from vllm.distributed.kv_transfer.kv_connector.v1.base import KVConnectorRole

    from b200kv.connector import B200KVConnector
    from tests.test_connector_cpu import fake_vllm_config
    for k in ("LMCACHE_LOCAL_DISK", "LMCACHE_MAX_LOCAL_DISK_SIZE", "LMCACHE_REMOTE_URL", "B200KV_DISK_WAIT_MS",
              "B200KV_REMOTE_WAIT_MS", "LMCACHE_CONFIG_FILE"):
        monkeypatch.delenv(k, raising=False)
    for k, v in {"LMCACHE_MAX_LOCAL_CPU_SIZE": "0.05", "LMCACHE_CHUNK_SIZE": "64", "B200KV_ASYNC_LOAD": "0",
                 **env}.items():
        monkeypatch.setenv(k, v)
    cfg = fake_vllm_config(f"t{os.getpid()}d{os.urandom(3).hex()}", role=kv_role)
    return B200KVConnector(cfg, getattr(KVConnectorRole, role), None), cfg


def _seed(conn, cfg):
    from b200kv.connector import geometry_from_vllm
    return geometry_from_vllm(cfg, conn.cfg).key_seed("synth-llama", 1, 0)


def _ask_until_answered(conn, req, limit=10):
    t0 = time.time()
    while True:
        n, is_async = conn.get_num_new_matched_tokens(req, 0)
        if n is not None:
            return n, is_async, time.time() - t0
        assert time.time() - t0 < limit
        time.sleep(0.005)


@vllm_needed
def test_unset_variables_open_nothing_and_start_nothing(monkeypatch, tmp_path):
    from types import SimpleNamespace as NS
    monkeypatch.setattr(tempfile, "tempdir", str(tmp_path))
    before = {t.name for t in threading.enumerate()}
    conn, _ = _connector(monkeypatch, {"LMCACHE_MAX_LOCAL_DISK_SIZE": "1"})     # a size alone: today's warning only
    try:
        assert conn._disk is None
        prompt = list(range(200))
        assert conn.get_num_new_matched_tokens(NS(request_id="r", prompt_token_ids=prompt, num_tokens=200,
                                                  all_token_ids=prompt), 0) == (0, False)
        fds = [os.readlink(f"/proc/self/fd/{f}") for f in os.listdir("/proc/self/fd")
               if os.path.exists(f"/proc/self/fd/{f}")]
        assert not [f for f in fds if "b200kv-disk" in f] and not os.path.exists(default_disk_dir())
        assert not [t for t in {t.name for t in threading.enumerate()} - before if "disk" in t]
        assert conn.reset_cache() is True
    finally:
        conn.shutdown()
        KVPool.unlink(conn._pool_name)


@vllm_needed
def test_scheduler_prefetches_from_disk_then_hits_and_reset_clears_it(monkeypatch, tmp_path):
    from types import SimpleNamespace as NS
    monkeypatch.setattr(tempfile, "tempdir", str(tmp_path))
    conn, cfg = _connector(monkeypatch, {"LMCACHE_LOCAL_DISK": "True", "LMCACHE_MAX_LOCAL_DISK_SIZE": "0.01"})
    try:
        assert conn._disk is not None and conn._disk.directory == os.path.join(str(tmp_path), "b200kv-disk")
        cb = conn._pool.stats()["slot_bytes"]
        prompt = list(range(200))
        keys = chunk_keys(np.asarray(prompt, np.int32), 64, _seed(conn, cfg))
        other = KVPool(None, 8 * cb, cb, _lib.POOL_CREATE)            # another replica wrote chunks 0..2
        d = DiskFile(conn._disk.directory, conn.cfg.disk_bytes, cb)
        for i, k in enumerate(keys[:3]):
            slot = other.reserve(int(k), 64, 0, 5)
            other.slot_view(slot)[:] = i + 1
            other.commit(int(k))
            assert d.put(other, int(k), 5) == 0
        req = NS(request_id="r1", prompt_token_ids=prompt, num_tokens=200, all_token_ids=prompt)
        assert conn.get_num_new_matched_tokens(req, 0) == (None, False)
        n, is_async, _ = _ask_until_answered(conn, req)
        assert (n, is_async) == (192, False)
        slot, n_tok, fmt = conn._pool.acquire(int(keys[1]))
        assert n_tok == 64 and int(conn._pool.slot_view(slot)[0]) == 2
        conn._pool.release(int(keys[1]))
        meta = conn.build_connector_meta(NS(scheduled_new_reqs=[], scheduled_cached_reqs=NS(
            req_ids=[], new_block_ids=[], resumed_req_ids=set(), all_token_ids={}), num_scheduled_tokens={},
            finished_req_ids=set()))
        assert meta.disk_counters == (3, 0)
        assert conn.request_finished(req, []) == (False, None)
        assert conn.reset_cache() is True                              # pool and disk
        assert d.lookup(np.asarray(keys[:3], np.uint64)) == 0 and conn._pool.stats()["n_used"] == 0
        d.close()
        other.close()
    finally:
        conn.shutdown()
        KVPool.unlink(conn._pool_name)
        KVPool.unlink(index_name(os.path.join(str(tmp_path), "b200kv-disk"), cb))


@vllm_needed
def test_disk_before_server_within_the_two_budgets(monkeypatch, ddir):
    """The disk is asked first; the cache server only for what the disk did not have; a request never waits longer
    than B200KV_DISK_WAIT_MS + B200KV_REMOTE_WAIT_MS, however slow both are."""
    from types import SimpleNamespace as NS

    from b200kv.remote import RemoteServer
    srv = RemoteServer("127.0.0.1", 0, 64 << 20)
    conn, cfg = _connector(monkeypatch, {"LMCACHE_LOCAL_DISK": f"file://{ddir}", "LMCACHE_MAX_LOCAL_DISK_SIZE": "0.01",
                                         "LMCACHE_REMOTE_URL": f"lm://127.0.0.1:{srv.port}",
                                         "B200KV_DISK_WAIT_MS": "300", "B200KV_REMOTE_WAIT_MS": "400"})
    order = []
    try:
        for name, tier in (("disk", conn._disk), ("remote", conn._remote)):
            real = tier._fetch

            def fetch(missing, name=name, real=real):
                order.append((name, [len(m) for m in missing]))
                return real(missing)
            tier._fetch = fetch
        cb = conn._pool.stats()["slot_bytes"]
        prompt = list(range(256))
        keys = chunk_keys(np.asarray(prompt, np.int32), 64, _seed(conn, cfg))
        other = KVPool(None, 8 * cb, cb, _lib.POOL_CREATE)
        d = DiskFile(ddir, conn.cfg.disk_bytes, cb)
        for k in keys[:2]:
            slot = other.reserve(int(k), 64, 0, 5)
            other.slot_view(slot)[:] = 1
            other.commit(int(k))
            assert d.put(other, int(k), 5) == 0
        req = NS(request_id="r1", prompt_token_ids=prompt, num_tokens=256, all_token_ids=prompt)
        n, _, _ = _ask_until_answered(conn, req)
        assert n == 128 and order == [("disk", [4]), ("remote", [2])]    # the server is asked for chunks 2..3 only
        # both tiers stall: the answer comes within the two budgets added together
        gate = threading.Event()
        for tier in (conn._disk, conn._remote):
            tier._fetch = lambda missing: gate.wait(10)
        req2 = NS(request_id="r2", prompt_token_ids=prompt[::-1], num_tokens=256, all_token_ids=prompt[::-1])
        n, _, dt = _ask_until_answered(conn, req2)
        assert n == 0 and 0.6 < dt < 0.7 + 0.5
        gate.set()
        d.close()
        other.close()
    finally:
        conn.shutdown()
        KVPool.unlink(conn._pool_name)
        srv.stop()


@vllm_needed
def test_unusable_directory_leaves_the_connector_serving(monkeypatch, tmp_path, caplog):
    caplog.set_level(logging.WARNING, logger="b200kv")
    conn, _ = _connector(monkeypatch, {"LMCACHE_LOCAL_DISK": str(tmp_path / "missing"),
                                       "LMCACHE_MAX_LOCAL_DISK_SIZE": "1"})
    try:
        assert conn._disk is None
        assert [r for r in caplog.records if "disk tier" in r.getMessage() and "unavailable" in r.getMessage()]
    finally:
        conn.shutdown()
        KVPool.unlink(conn._pool_name)


@vllm_needed
def test_disk_series_only_when_the_tier_is_configured(monkeypatch, tmp_path):
    from prometheus_client import CollectorRegistry, Counter, Gauge, Histogram, generate_latest

    from b200kv.connector import B200KVConnector
    from b200kv.metrics import B200KVStats
    from tests.test_connector_cpu import fake_vllm_config
    for k in ("LMCACHE_LOCAL_DISK", "LMCACHE_MAX_LOCAL_DISK_SIZE", "LMCACHE_CONFIG_FILE"):
        monkeypatch.delenv(k, raising=False)

    def series(extra):
        reg = CollectorRegistry()

        def bind(cls):
            return lambda **kw: cls(registry=reg, **{k: v for k, v in kw.items() if k != "multiprocess_mode"})
        pm = B200KVConnector.build_prom_metrics(fake_vllm_config("prom", extra), {Gauge: bind(Gauge), Counter: bind(Counter),
                                                Histogram: bind(Histogram)}, ["model_name", "engine"], {0: ["synth", "0"]})
        a = B200KVStats({"num_stored_tokens": 256, "disk_written_chunks": 3, "disk_skipped_chunks": 1,
                         "disk_usage_bytes": 3 << 25})
        agg = a.aggregate(B200KVStats({"disk_fetched_chunks": 2, "disk_corrupt_chunks": 1, "disk_written_chunks": 1}))
        assert agg.reduce()["disk_written_chunks"] == 4
        pm.observe(agg.data, 0)
        return generate_latest(reg).decode()

    assert "b200kv:disk" not in series({})
    text = series({"lmcache.local_disk": str(tmp_path), "lmcache.max_local_disk_size": 1})
    for name, v in (("fetched", 2), ("written", 4), ("skipped", 1), ("corrupt", 1)):
        assert f'b200kv:disk_{name}_chunks_total{{engine="0",model_name="synth"}} {v}.0' in text, name
    assert 'b200kv:disk_usage{engine="0",model_name="synth"} 1.00663296e+08' in text
