"""Q4 chunks of an fp8 (e4m3) KV cache, on one GPU: prints one JSON line.

Llama-3-8B geometry (32 layers, 8 KV heads x 128, vLLM block 16, LMCache chunk 256) with 1-byte e4m3 pages, as
vLLM allocates them under --kv-cache-dtype fp8; 32 768 tokens per step, their blocks scattered over the pages.

* q4_store / q4_load: the Q4 kernels of fp8 pages through the device-resident gather / scatter (b200kv_gather /
  b200kv_scatter), kernel time from the engine's CUDA events;
* raw_store / raw_load: the RAW gather / scatter of the same pages.  A Q4 engine and a RAW engine run ALTERNATELY in
  this one process (step i: Q4 leg, then RAW leg), so clock and thermal drift hit both alike;
* pool_store / pool_retrieve: KVEngine.store / retrieve of the 32 768 tokens through the pinned host pool in Q4,
  host wall time from the call to the end of its ticket.

Algorithmic bytes (DESIGN §3): a store reads the pages and writes the chunk format, a load the reverse.  Per token:
Q4 64 * 1024 B of pages + 64 * 576 B of records (R 65 536 + W 36 864), RAW 2 * 64 * 1024 B; GB/s = those bytes over
the median kernel time.  Every leg is checked bit for bit on a sample: the Q4 records of the first chunk for two
layers against tests/fp8_cache_oracle.py, the decoded pages of those tokens, the RAW pages, and the pool round trip.
The card's name, power limit and max SM clock are read in the same run.

    python tools/bench_fp8_cache.py [--steps 10] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "production-stack_b200")]

import numpy as np  # noqa: E402

from tools.bench_mla import card  # noqa: E402

N_TOK = 32768
KV = dict(L=32, H=8, D=128, BS=16, C=256)
SAMPLE_LAYERS = (0, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import torch

    from b200kv import FMT_Q4, FMT_RAW, KVEngine, KVGeometry, KVPool, _lib
    from oracle import kv_oracle as ko
    from tests import fp8_cache_oracle as fo
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8_cache.py needs a GPU: there is no CPU path to measure")
    dev = torch.device("cuda:0")
    L, H, D, BS, C = KV["L"], KV["H"], KV["D"], KV["BS"], KV["C"]
    legs, checks = {}, {}

    def timed_pair(engines, which, fns):
        """Alternate the legs of the two engines; median / min / max kernel ms of each."""
        for _ in range(a.warmup):
            for f in fns:
                f()
        torch.cuda.synchronize()
        ms = [[], []]
        for _ in range(a.steps):
            for i, (e, f) in enumerate(zip(engines, fns)):
                f()
                torch.cuda.synchronize()
                ms[i].append(e.last_kernel_ms(which))
        return [(float(np.median(m)), float(min(m)), float(max(m))) for m in ms]

    def record(name, t, gb, per_token_ns=True):
        legs[name] = {"ms_median": t[0], "ms_min": t[1], "ms_max": t[2], "GBps": gb / (t[0] / 1e3)}
        if per_token_ns:
            legs[name]["ns_per_token"] = t[0] * 1e6 / N_TOK

    rng = np.random.default_rng(0)
    nb_need = N_TOK // BS
    NB = 2 * nb_need + 8
    perm = rng.permutation(NB)
    sm = ko.slot_mapping_from_blocks(perm[:nb_need], BS, N_TOK)
    dm = ko.slot_mapping_from_blocks(perm[nb_need:2 * nb_need], BS, N_TOK)
    smi, dmi = torch.from_numpy(sm).to(dev), torch.from_numpy(dm).to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    pages = [torch.randn((2, NB, BS, H, D), generator=g, device=dev).to(torch.float8_e4m3fn).view(torch.uint8)
             for _ in range(L)]

    def sample(pg, idx):   # (2 layers, 2, C, H, D) codes of the first C tokens of a mapping
        return np.stack([pg[l].view(2, -1, H, D)[:, idx[:C]].cpu().numpy() for l in SAMPLE_LAYERS])

    engines, bufs = [], []
    for fmt in (FMT_Q4, FMT_RAW):
        geom = KVGeometry(L, H, D, NB, BS, C, 1, 0, fmt, _lib.LAYOUT_NHD, fp8_dtype=_lib.DTYPE_E4M3)
        e = KVEngine(geom, None, 0, staging_bytes=0)
        e.register_kv_caches(pages)
        engines.append(e)
        bufs.append(torch.zeros((N_TOK // C) * geom.chunk_bytes, dtype=torch.uint8, device=dev))
    gq = engines[0].geom
    rec = H * D // 2 + H * (D // 32) * 2
    q4_gb = (gq.planes * H * D + gq.planes * rec) * N_TOK / 1e9
    raw_gb = 2 * gq.planes * H * D * N_TOK / 1e9
    src = sample(pages, smi)
    st = timed_pair(engines, 0, [lambda e=e, b=b: e.gather(sm, b.data_ptr()) for e, b in zip(engines, bufs)])
    # the chunks are what the pages held: check them before the loads overwrite the destination blocks
    codes, sc = fo.q4_pack_chunk(src, "e4m3")
    r = bufs[0][:gq.planes * C * rec].view(L, 2, C, rec)[list(SAMPLE_LAYERS)].cpu().numpy()
    checks["q4_store"] = bool(np.array_equal(r[..., :H * D // 2], codes.reshape(2, 2, C, -1)) and
                              np.array_equal(r[..., H * D // 2:].copy().view(np.uint16), sc.reshape(2, 2, C, -1)))
    raw = bufs[1][:engines[1].geom.chunk_bytes].view(L, 2, C, H, D)[list(SAMPLE_LAYERS)].cpu().numpy()
    checks["raw_store"] = bool(np.array_equal(raw, src))
    # loads alternate too; the Q4 leg's pages are checked after the RAW leg rewrote them, so reload once at the end
    ld = timed_pair(engines, 1, [lambda e=e, b=b: e.scatter(dm, b.data_ptr()) for e, b in zip(engines, bufs)])
    checks["raw_load"] = bool(np.array_equal(sample(pages, dmi), src))
    engines[0].scatter(dm, bufs[0].data_ptr())
    torch.cuda.synchronize()
    checks["q4_load"] = bool(np.array_equal(sample(pages, dmi), fo.q4_unpack_chunk(codes, sc, "e4m3")))
    record("q4_store", st[0], q4_gb)
    record("q4_load", ld[0], q4_gb)
    record("raw_store", st[1], raw_gb)
    record("raw_load", ld[1], raw_gb)
    for e in engines:
        e.close()
    del bufs

    # ---- the pinned pool: store, then retrieve into the other blocks --------------------------------------------
    pool = KVPool(None, (N_TOK // C + 4) * gq.chunk_bytes, gq.chunk_bytes, 1)
    eng = KVEngine(gq, pool, 0, staging_bytes=8 * gq.chunk_bytes)
    eng.register_kv_caches(pages)
    st_ms, rt_ms = [], []
    for i in range(a.warmup + a.steps):
        toks = rng.integers(0, 128256, N_TOK).astype(np.int32)    # fresh keys: every step stores every chunk
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        eng.wait(eng.store(toks, None, sm))
        t1 = time.perf_counter()
        ret, ticket = eng.retrieve(toks, None, dm, return_ticket=True)
        if ticket:
            eng.wait(ticket)
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        if i >= a.warmup:
            st_ms.append((t1 - t0) * 1e3)
            rt_ms.append((t2 - t1) * 1e3)
    checks["pool_hit"] = bool(ret.all())
    checks["pool_round_trip"] = bool(np.array_equal(sample(pages, dmi), fo.q4_unpack_chunk(codes, sc, "e4m3")))
    pool_gb = gq.planes * rec * N_TOK / 1e9      # bytes over PCIe each way
    record("pool_store", (float(np.median(st_ms)), min(st_ms), max(st_ms)), pool_gb)
    record("pool_retrieve", (float(np.median(rt_ms)), min(rt_ms), max(rt_ms)), pool_gb)
    eng.close()
    pool.close()

    result = {"tokens": N_TOK, "kv_geometry": KV, "cache_dtype": "fp8 (e4m3)",
              "bytes_per_token": {"q4_store_read": gq.planes * H * D, "q4_store_write": gq.planes * rec,
                                  "raw_each_way": gq.planes * H * D},
              "legs": legs, "q4_over_raw_time": {"store": st[0][0] / st[1][0], "load": ld[0][0] / ld[1][0]},
              "bit_exact": checks, "all_bit_exact": all(checks.values()),
              "card": card(), "steps": a.steps, "warmup": a.warmup}
    print(json.dumps(result), flush=True)
    return 0 if result["all_bit_exact"] else 1


if __name__ == "__main__":
    sys.exit(main())
