"""Local-disk chunk tier with the real CUDA engine (run on an H100 with -m gpu).  An engine stores a prompt, the
worker's write-through puts its chunks on disk, and the pinned pool is emptied, so only the disk holds them.  The
scheduler-side prefetch reads them back into the pool, and a second engine loads them, chunk-wise or layer-wise, into
other pages: those must equal the oracle's pages bit for bit (RAW) / code for code (FP8, Q4).  K/V RAW, FP8 and Q4
on NHD and HND tiles, MLA FP8, DeepSeek-V3.2 with indexer planes, and a geometry with a draft layer.  Then a second
process with a fresh pool and no index in shm loads what the first wrote from the same directory."""
import os
import subprocess
import sys
import time
from unittest import mock

import numpy as np
import pytest

from oracle import kv_oracle as ko
from tests import test_gpu_spec_decode as sd

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from b200kv import FMT_FP8, FMT_Q4, FMT_RAW, KVEngine, KVPool  # noqa: E402
from b200kv.disk import DiskTier, index_name  # noqa: E402
from b200kv.engine import chunk_keys  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CASES = {   # name: (kind, L, D, fmt)
    "raw-nhd": ("nhd", 3, 0, FMT_RAW),
    "fp8-nhd": ("nhd", 3, 0, FMT_FP8),
    "q4-nhd": ("nhd", 3, 0, FMT_Q4),
    "raw-hnd": ("hnd", 3, 0, FMT_RAW),
    "fp8-hnd": ("hnd", 3, 0, FMT_FP8),
    "q4-hnd": ("hnd", 3, 0, FMT_Q4),
    "mla-fp8": ("mla", 3, 0, FMT_FP8),
    "v32-raw": ("idx", 3, 0, FMT_RAW),
    "v32-fp8": ("idx", 3, 0, FMT_FP8),
    "draft-nhd": ("nhd", 4, 1, FMT_RAW),
}


class Case(sd.Case):
    """The speculative-decoding test's case (host pages, device caches, oracle pages) for any of CASES."""

    def __init__(self, name, rng, NB, bs, C=256):
        with mock.patch.dict(sd.CASES, {name: CASES[name]}):
            super().__init__(name, rng, NB, bs, C)

    def expect(self, sm, dm, before=None):
        if self.kind in ("nhd", "hnd") and self.fmt == FMT_Q4:
            want = [np.zeros_like(h) for h in self.host]
            oe = ko.OracleEngine(self.C, "q4")
            toks = np.arange(len(sm), dtype=np.int32)
            oe.store(toks, np.ones(len(sm), bool), self.host, sm)
            oe.retrieve(toks, np.ones(len(sm), bool), want, dm)
            return want
        return super().expect(sm, dm, before)


def disk_bytes(chunk_bytes, n_slots):
    return 4096 + n_slots * (4096 + (chunk_bytes + 4095) // 4096 * 4096)


def wait_prefetch(tier, req, toks):
    t0 = time.time()
    while tier.prefetch_state(req, toks) == tier.PENDING:
        assert time.time() - t0 < 60
        time.sleep(0.002)


def store_then_empty_pool(case, pool, directory, toks, sm):
    """Engine A stores, the worker's disk tier writes the chunks through, and the pool forgets them."""
    g = case.geom
    eng = KVEngine(g, pool, 0, staging_bytes=4 * g.chunk_bytes)
    eng.register_kv_caches(case.registered(case.device()))
    writer = DiskTier(pool, directory, disk_bytes(g.chunk_bytes, 8), case.C, eng.key_seed, owner=3)
    try:
        eng.wait(eng.store(toks, None, sm))
        keys = eng._keys(toks)
        writer.push(keys)                           # what WorkerState.on_stored hands over after a store
        assert writer.flush(60)
        assert writer.stats()["written_chunks"] == len(keys) and writer.stats()["skipped_chunks"] == 0
        assert pool.clear() and eng.lookup(toks) == 0
        return eng.key_seed
    finally:
        writer.close()
        eng.close()


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("mode", ["chunk", "layer"])
def test_disk_only_chunks_prefetch_and_load_bit_exact(name, mode, tmp_path):
    sd.need_gpu()
    rng = np.random.default_rng(sum(map(ord, name + mode)))
    case = Case(name, rng, 64, 64 if case_is_mla(name) else 16)
    g, C, n = case.geom, case.C, 2 * 256 + 70
    pool = KVPool(None, 8 * g.chunk_bytes, g.chunk_bytes, 1)
    toks = (np.arange(n, dtype=np.int32) * 7 + len(name)) % 9000
    sm, dm = sd.slots(rng, case.NB, case.bs, n), sd.slots(rng, case.NB, case.bs, n)
    reader = None
    try:
        seed = store_then_empty_pool(case, pool, str(tmp_path), toks, sm)
        reader = DiskTier(pool, str(tmp_path), disk_bytes(g.chunk_bytes, 8), C, seed)    # the scheduler's tier
        assert reader.prefetch_state("req", toks) == reader.PENDING
        wait_prefetch(reader, "req", toks)
        assert reader.stats()["fetched_chunks"] == 3 and reader.stats()["corrupt_chunks"] == 0
        assert list(pool.lookup_owner(chunk_keys(toks, C, seed, True))[1]) == [3, 3, 3]
        dst = case.device(zero=True)
        eng = KVEngine(g, pool, 0, staging_bytes=4 * g.chunk_bytes)
        eng.register_kv_caches(case.registered(dst))
        assert eng.lookup(toks) == n
        if mode == "chunk":
            assert eng.retrieve(toks, None, dm).all()
        else:
            s = torch.cuda.Stream()
            ret, ticket = eng.retrieve(toks, None, dm, stream=s, return_ticket=True, layers_per_group=2)
            assert ret.all() and ticket
            eng.wait(ticket)
        torch.cuda.synchronize()
        sd.assert_pages(case, dst, case.expect(sm, dm), f"{name} {mode} from disk")
        eng.close()
    finally:
        if reader is not None:
            reader.close()
        KVPool.unlink(index_name(str(tmp_path), g.chunk_bytes))
        pool.close()


def case_is_mla(name):
    return CASES[name][0] in ("mla", "idx")


_SECOND = r"""
import sys
import numpy as np
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[2])
import torch
from b200kv import KVEngine, KVPool
from b200kv.disk import DiskTier
from tests.test_gpu_disk import Case, disk_bytes, wait_prefetch
directory, out = sys.argv[3], sys.argv[4]
case = Case("raw-nhd", np.random.default_rng(11), 64, 16)
g, n = case.geom, 2 * 256 + 70
toks = (np.arange(n, dtype=np.int32) * 7 + 7) % 9000
dm = np.load(out + ".dm.npy")
pool = KVPool(None, 8 * g.chunk_bytes, g.chunk_bytes, 1)
eng = KVEngine(g, pool, 0, staging_bytes=4 * g.chunk_bytes)
dst = case.device(zero=True)
eng.register_kv_caches(case.registered(dst))
tier = DiskTier(pool, directory, disk_bytes(g.chunk_bytes, 8), case.C, eng.key_seed)
assert tier.file.stats()["n_restored"] == 3
wait_prefetch(tier, "again", toks)
assert tier.stats()["fetched_chunks"] == 3, tier.stats()
assert eng.retrieve(toks, None, dm).all()
torch.cuda.synchronize()
np.savez(out, *case.pages(dst))
tier.close(); eng.close(); pool.close()
"""


def test_a_second_process_loads_what_the_first_wrote(tmp_path):
    sd.need_gpu()
    rng = np.random.default_rng(11)
    case = Case("raw-nhd", rng, 64, 16)
    g, n = case.geom, 2 * 256 + 70
    toks = (np.arange(n, dtype=np.int32) * 7 + 7) % 9000
    sm, dm = sd.slots(rng, case.NB, case.bs, n), sd.slots(rng, case.NB, case.bs, n)
    pool = KVPool(None, 8 * g.chunk_bytes, g.chunk_bytes, 1)
    directory = str(tmp_path / "disk")
    os.mkdir(directory)
    store_then_empty_pool(case, pool, directory, toks, sm)
    pool.close()
    KVPool.unlink(index_name(directory, g.chunk_bytes))     # a restarted box: no index in shm
    out = str(tmp_path / "pages")
    np.save(out + ".dm.npy", dm)
    try:
        subprocess.run([sys.executable, "-c", _SECOND, os.path.join(ROOT, "production-stack_b200"), ROOT, directory,
                        out], check=True, timeout=600)
    finally:
        KVPool.unlink(index_name(directory, g.chunk_bytes))
    got = np.load(out + ".npz")
    want = case.expect(sm, dm)
    assert len(got.files) == len(want)
    for i, w in enumerate(want):
        assert np.array_equal(got[f"arr_{i}"], w), f"plane {i}"
