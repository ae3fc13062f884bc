"""Sparse-attention MLA offload at DeepSeek-V3.2 geometry on one GPU: prints one JSON line.

Geometry: 61 layers; per (token, layer) one 576-element bf16 latent (1152 bytes) and one indexer key of 128 e4m3
values + one fp32 scale (132 bytes, 10.3 % of the bytes); vLLM block size 64, LMCache chunk 256; 16 sessions x 2048
tokens = 32 768 tokens per step, their blocks scattered over the pages.  The same step runs on an engine with
indexer planes and on a plain MLA engine over the same latent pages, so the cost of the indexer planes is the
difference.  Legs (RAW):

* gather / scatter: device-resident copy kernels (b200kv_gather / b200kv_scatter), algorithmic bytes 2 x payload
  per token (read + write) over kernel time (CUDA events around the op's kernels: latent and indexer together);
* indexer_kernel: kv_indexer_copy_kernel's own time in the indexed gather and scatter (torch.profiler);
* e2e: store every session into the pinned host pool and retrieve it into other pages (store_batch + wait, then
  retrieve_batch + wait), payload bytes moved each way over wall time.

Every leg's output is checked bit for bit against the pages themselves.  The card's name and power limit are read
in the same run.

    python tools/bench_mla_sparse.py [--steps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "production-stack_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402

from bench_mla import card  # noqa: E402

L, D, BS, C, IDX = 61, 576, 64, 256, 132
SESSIONS, SESSION_TOKENS = 16, 2048
N_TOK = SESSIONS * SESSION_TOKENS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()

    import torch

    from b200kv import FMT_RAW, KVEngine, KVGeometry, KVPool, _lib
    from oracle import kv_oracle as ko
    if not torch.cuda.is_available():
        raise SystemExit("bench_mla_sparse.py needs a GPU: there is no CPU path to measure")

    dev = torch.device("cuda:0")
    nb_need = N_TOK // BS
    NB = nb_need * 2 + 8
    g = torch.Generator(device=dev).manual_seed(0)
    latent = [torch.randn((NB, BS, D), generator=g, device=dev).bfloat16() for _ in range(L)]
    indexer = [torch.randint(0, 256, (NB, BS, IDX), generator=g, device=dev, dtype=torch.uint8) for _ in range(L)]
    caches = {}
    for l in range(L):
        caches[f"model.layers.{l}.self_attn.attn"] = latent[l]
        caches[f"model.layers.{l}.self_attn.indexer.k_cache"] = indexer[l]
    rng = np.random.default_rng(0)
    perm = rng.permutation(NB)
    src_blocks, dst_blocks = perm[:nb_need], perm[nb_need:2 * nb_need]
    sm = ko.slot_mapping_from_blocks(src_blocks, BS, N_TOK)
    dm = ko.slot_mapping_from_blocks(dst_blocks, BS, N_TOK)
    sb, db = torch.from_numpy(src_blocks).to(dev), torch.from_numpy(dst_blocks).to(dev)
    want_lat = [p[sb].clone() for p in latent]
    want_idx = [p[sb].clone() for p in indexer]
    n_chunks = N_TOK // C
    checks, legs = {}, {}

    def clear_dst():
        for p in latent + indexer:
            p[db] = 0

    def dst_ok(with_idx):
        ok = all(torch.equal(p[db].view(torch.int16), w.view(torch.int16)) for p, w in zip(latent, want_lat))
        return ok and (not with_idx or all(torch.equal(p[db], w) for p, w in zip(indexer, want_idx)))

    def kernel_leg(eng, which, fn):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        ms = []
        for _ in range(a.steps):
            fn()
            torch.cuda.synchronize()
            ms.append(eng.last_kernel_ms(which))
        return float(np.median(ms)), float(min(ms)), float(max(ms))

    for name, idx in (("plain", False), ("indexed", True)):
        geom = KVGeometry(L, 1, D, NB, BS, C, 2, 0, FMT_RAW, _lib.LAYOUT_MLA,
                          idx_value_bytes=128 if idx else 0, idx_scale_bytes=4 if idx else 0)
        eng = KVEngine(geom, None, 0, staging_bytes=0)
        eng.register_kv_caches(caches if idx else latent)
        buf = torch.zeros(n_chunks * geom.chunk_bytes, dtype=torch.uint8, device=dev)
        g_ms = kernel_leg(eng, 0, lambda: eng.gather(sm, buf.data_ptr()))
        clear_dst()
        s_ms = kernel_leg(eng, 1, lambda: eng.scatter(dm, buf.data_ptr()))
        checks[f"{name}_gather_scatter"] = dst_ok(idx)
        gb = 2 * geom.payload_bytes_per_token * N_TOK / 1e9
        for leg, ms in (("gather", g_ms), ("scatter", s_ms)):
            legs[f"{name}_{leg}"] = {"kernel_ms_median": ms[0], "kernel_ms_min": ms[1], "kernel_ms_max": ms[2],
                                     "GBps": gb / (ms[0] / 1e3)}
        if idx:
            from torch.profiler import ProfilerActivity, profile
            own = {"gather": [], "scatter": []}
            for _ in range(a.steps):
                for leg, fn in (("gather", lambda: eng.gather(sm, buf.data_ptr())),
                                ("scatter", lambda: eng.scatter(dm, buf.data_ptr()))):
                    torch.cuda.synchronize()
                    with profile(activities=[ProfilerActivity.CUDA]) as prof:
                        fn()
                        torch.cuda.synchronize()
                    us = sum(e.device_time_total for e in prof.key_averages() if "kv_indexer_copy_kernel" in e.key)
                    own[leg].append(us / 1e3)
            ib = 2 * L * IDX * N_TOK / 1e9
            for leg in ("gather", "scatter"):
                ms = float(np.median(own[leg]))
                legs[f"indexer_kernel_{leg}"] = {"kernel_ms_median": ms, "GBps": ib / (ms / 1e3) if ms else None}
        eng.close()
        del buf

        pool = KVPool(None, (n_chunks + 2) * geom.chunk_bytes, geom.chunk_bytes, 1)
        eng = KVEngine(geom, pool, 0, staging_bytes=16 * geom.chunk_bytes)
        eng.register_kv_caches(caches if idx else latent)
        toks = [((np.arange(SESSION_TOKENS, dtype=np.int64) + 7919 * s) % 100003).astype(np.int32)
                for s in range(SESSIONS)]
        reqs = [(toks[s], sm[s * SESSION_TOKENS:(s + 1) * SESSION_TOKENS], 0) for s in range(SESSIONS)]
        dreqs = [(toks[s], dm[s * SESSION_TOKENS:(s + 1) * SESSION_TOKENS], 0) for s in range(SESSIONS)]
        times, ok = [], True
        for step in range(a.warmup + a.steps):
            pool.clear()
            clear_dst()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            eng.wait(eng.store_batch(reqs))
            t1 = time.perf_counter()
            loaded, ticket = eng.retrieve_batch(dreqs)
            eng.wait(ticket)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            ok = ok and int(np.sum(loaded)) == N_TOK
            if step >= a.warmup:
                times.append((t1 - t0, t2 - t1))
        checks[f"{name}_e2e"] = bool(ok and dst_ok(idx))
        st, ld = float(np.median([t[0] for t in times])), float(np.median([t[1] for t in times]))
        payload = geom.payload_bytes_per_token * N_TOK
        legs[f"{name}_e2e"] = {"store_ms": st * 1e3, "retrieve_ms": ld * 1e3, "payload_bytes": payload,
                               "store_GBps": payload / st / 1e9, "retrieve_GBps": payload / ld / 1e9,
                               "chunk_bytes": geom.chunk_bytes}
        eng.close()
        pool.close()

    share = IDX / (D * 2 + IDX)
    added = {leg: float(legs[f"indexed_{leg}"]["kernel_ms_median"] / legs[f"plain_{leg}"]["kernel_ms_median"] - 1)
             for leg in ("gather", "scatter")}
    added.update({f"e2e_{k}": float(legs["indexed_e2e"][f"{k}_ms"] / legs["plain_e2e"][f"{k}_ms"] - 1)
                  for k in ("store", "retrieve")})
    result = {"geometry": {"layers": L, "latent_dim": D, "indexer_bytes": IDX, "block_tokens": BS, "chunk_tokens": C,
                           "tokens": N_TOK},
              "legs": legs, "indexer_byte_share": share, "indexer_added_time": added,
              "within_byte_share": {k: v <= share / (1 - share) for k, v in added.items()},
              "bit_exact": checks, "all_bit_exact": all(checks.values()), "card": card(),
              "steps": a.steps, "warmup": a.warmup}
    print(json.dumps(result), flush=True)
    return 0 if result["all_bit_exact"] else 1


if __name__ == "__main__":
    sys.exit(main())
