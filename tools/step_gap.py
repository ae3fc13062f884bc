#!/usr/bin/env python
"""Where the device-resident step of bench.py spends its time.  Prints one JSON line.

Runs bench.py's device-resident (`value`) leg as bench.py runs it: the same geometry, seeds, slot maps,
engine and staging set-up, and `last_kernel_ms` read after every step.  Reports

  ms_per_step        CUDA events around the timed steps, as bench.py measures it
  gather/scatter_ms  the library's kernel-only events of each step (kv_bulk_copy_kernel<store> / <load>)
  gap_ms             ms_per_step - (gather_ms + scatter_ms): the time in a step when neither kernel runs
  host_*_us          perf_counter around each eng.gather / eng.scatter call (the enqueue: run table built,
                     uploaded, kernel launched) and around the last_kernel_ms reads (which wait for the step)

then a measured HBM copy ceiling for the same step: two device-to-device copies of 4 GiB each (what a step
moves, 4 GiB out of the pages and 4 GiB back), CUDA events, reported as a time per step and in bench.py's
`value` units.  The card's name, power limit and maximum SM clock are read with nvidia-smi in the same run.

  python tools/step_gap.py [--steps 20] [--warmup 3] [--lib path/to/libb200kv.so]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "production-stack_b200"))

import bench  # noqa: E402  (geometry, seeds and slot maps of the benchmark)

GiB = 1 << 30


def card(index: int) -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", f"--query-gpu={q}", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = (f.strip() for f in out.split(","))
        return {"name": name, "power_limit": power, "clocks_max_sm": clock}
    except Exception as e:
        return {"error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--lib", default=None, help="libb200kv.so to load instead of the in-tree one")
    ap.add_argument("--copy-reps", type=int, default=5)
    args = ap.parse_args()

    import torch

    from b200kv import _lib
    if args.lib:
        _lib.LIB_PATH = os.path.abspath(args.lib)
    from b200kv import FMT_RAW, KVEngine, KVGeometry, KVPool

    if not torch.cuda.is_available():
        raise SystemExit("step_gap.py needs an H100")
    local = 0
    torch.cuda.set_device(local)
    dev = torch.device(f"cuda:{local}")
    L, H, D, NB, BS, C = bench.L, bench.H, bench.D, bench.NB, bench.BS, bench.C
    SESSIONS, CTX = bench.SESSIONS, bench.CTX

    # ---- engine, caches and maps exactly as bench.run_ours sets them up (rank 0) ----------------
    rank = 0
    geom = KVGeometry(L, H, D, NB, BS, C, 2, 0, FMT_RAW)
    g = torch.Generator(device=dev).manual_seed(rank)
    caches = [torch.randn((2, NB, BS, H, D), generator=g, device=dev, dtype=torch.float32).bfloat16()
              for _ in range(L)]
    n_chunks_step = SESSIONS * CTX // C
    pool = KVPool(None, (n_chunks_step + n_chunks_step // 2) * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, local, staging_bytes=2 * n_chunks_step * geom.chunk_bytes, owner=rank)
    eng.register_kv_caches(caches)
    perm = torch.randperm(NB, generator=torch.Generator().manual_seed(1234)).numpy()
    dperm = torch.randperm(NB, generator=torch.Generator().manual_seed(4321)).numpy()
    nblk = CTX // BS
    all_src = np.concatenate([bench.slot_map(perm[s * nblk:(s + 1) * nblk], CTX) for s in range(SESSIONS)])
    all_dst = np.concatenate([bench.slot_map(dperm[s * nblk:(s + 1) * nblk], CTX) for s in range(SESSIONS)])
    stream = torch.cuda.current_stream()
    dbuf = torch.empty(n_chunks_step * geom.chunk_bytes, dtype=torch.uint8, device=dev)

    # ---- the device-resident step, timed as bench.py times it, plus host clocks ---------------------
    for _ in range(args.warmup):
        eng.gather(all_src, dbuf.data_ptr(), stream)
        eng.scatter(all_dst, dbuf.data_ptr(), stream)
    torch.cuda.synchronize()
    host_g, host_s, host_read, kern = [], [], [], []
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    ev0.record(stream)
    for _ in range(args.steps):
        t0 = time.perf_counter()
        eng.gather(all_src, dbuf.data_ptr(), stream)
        t1 = time.perf_counter()
        eng.scatter(all_dst, dbuf.data_ptr(), stream)
        t2 = time.perf_counter()
        kern.append((eng.last_kernel_ms(0), eng.last_kernel_ms(1)))
        t3 = time.perf_counter()
        host_g.append((t1 - t0) * 1e6)
        host_s.append((t2 - t1) * 1e6)
        host_read.append((t3 - t2) * 1e6)
    ev1.record(stream)
    torch.cuda.synchronize()
    ms_per_step = ev0.elapsed_time(ev1) / args.steps
    g_ms = float(np.mean([a for a, _ in kern]))
    s_ms = float(np.mean([b for _, b in kern]))
    payload = 2 * SESSIONS * CTX * bench.TOKEN_BYTES_ALL

    eng.close()
    pool.close()
    del caches, dbuf
    torch.cuda.empty_cache()

    # ---- measured HBM copy ceiling: 2 x 4 GiB device-to-device, CUDA events -------------------------
    a = torch.empty(payload // 2, dtype=torch.uint8, device=dev)
    b = torch.empty_like(a)
    a.fill_(1)
    b.copy_(a)
    a.copy_(b)
    torch.cuda.synchronize()
    ev0.record(stream)
    for _ in range(args.copy_reps):
        b.copy_(a)
        a.copy_(b)
    ev1.record(stream)
    torch.cuda.synchronize()
    copy_ms = ev0.elapsed_time(ev1) / args.copy_reps
    del a, b

    def stats(x):
        return {"median": float(np.median(x)), "min": float(np.min(x)), "max": float(np.max(x))}

    out = {
        "lib": _lib.LIB_PATH,
        "card": card(local),
        "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_per_step,
        "value_GBps": payload / (ms_per_step * 1e-3) / 1e9,
        "gather_ms": g_ms, "scatter_ms": s_ms,
        "gap_ms": ms_per_step - g_ms - s_ms,
        "host_gather_us": stats(host_g), "host_scatter_us": stats(host_s),
        "host_last_kernel_ms_us": stats(host_read),
        "copy_ceiling": {"ms_per_step": copy_ms, "value_GBps": payload / (copy_ms * 1e-3) / 1e9,
                         "hbm_GBps": 2 * payload / (copy_ms * 1e-3) / 1e9,
                         "how": f"2 x 4 GiB torch device-to-device copy, CUDA events, mean of {args.copy_reps} "
                                "(measured on this card in this run)"},
    }
    out["step_over_copy_ceiling"] = copy_ms / ms_per_step
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
