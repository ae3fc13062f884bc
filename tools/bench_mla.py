"""MLA offload at DeepSeek-V3 geometry on one GPU: prints one JSON line.

Geometry: 61 layers, one 576-element bf16 latent per (token, layer) = 70 272 bytes of KV per token, vLLM block
size 64 (FlashMLA), LMCache chunk 256; 16 sessions x 2048 tokens = 32 768 tokens per step, their blocks
scattered over the pages.  Legs:

* raw_gather / raw_scatter: device-resident RAW copy kernels (b200kv_gather / b200kv_scatter), algorithmic
  bytes 2 x 70 272 per token (read + write) over kernel time (CUDA events around the kernels);
* fp8_store / fp8_load: the FP8 latent-record kernels, (1152 + 656) bytes per (token, layer);
* e2e_raw / e2e_fp8: store every session into the pinned host pool and retrieve it into other pages
  (store_batch + wait, then retrieve_batch + wait), payload bytes moved each way over wall time.

Each leg's output is checked bit for bit: RAW against the pages themselves, FP8 records against
tests/mla_oracle.py on a sample, and what the e2e legs load against what the device-resident legs produced.
The card's name and power limit are read in the same run.

    python tools/bench_mla.py [--steps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "production-stack_b200")]

import numpy as np  # noqa: E402

L, D, BS, C = 61, 576, 64, 256
SESSIONS, SESSION_TOKENS = 16, 2048
N_TOK = SESSIONS * SESSION_TOKENS


def card() -> dict:
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, pw, clk = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit_w": float(pw), "max_sm_mhz": float(clk)}
    except Exception as e:  # the numbers below still stand; the card is named by torch
        import torch
        return {"name": torch.cuda.get_device_name(0), "power_limit_w": None, "error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()

    import torch

    from b200kv import FMT_FP8, FMT_RAW, KVEngine, KVGeometry, KVPool, _lib
    from oracle import kv_oracle as ko
    from tests import mla_oracle as mo
    if not torch.cuda.is_available():
        raise SystemExit("bench_mla.py needs a GPU: there is no CPU path to measure")

    dev = torch.device("cuda:0")
    nb_need = N_TOK // BS
    NB = nb_need * 2 + 8                     # room for a second, disjoint set of destination blocks
    g = torch.Generator(device=dev).manual_seed(0)
    pages = [torch.randn((NB, BS, D), generator=g, device=dev).bfloat16() for _ in range(L)]
    rng = np.random.default_rng(0)
    perm = rng.permutation(NB)
    src_blocks, dst_blocks = perm[:nb_need], perm[nb_need:2 * nb_need]
    sm = ko.slot_mapping_from_blocks(src_blocks, BS, N_TOK)
    dm = ko.slot_mapping_from_blocks(dst_blocks, BS, N_TOK)
    smi, dmi = torch.from_numpy(sm).to(dev), torch.from_numpy(dm).to(dev)
    src_snapshot = [p.view(-1, D)[smi].clone() for p in pages]       # what every load must bring back
    n_chunks = N_TOK // C
    result = {"geometry": {"layers": L, "head_dim": D, "block_tokens": BS, "chunk_tokens": C,
                           "sessions": SESSIONS, "session_tokens": SESSION_TOKENS,
                           "kv_bytes_per_token_bf16": L * D * 2}}
    checks = {}

    def clear_dst():
        for p in pages:
            p.view(-1, D)[dmi] = 0

    def dst_equals(want):
        return all(torch.equal(p.view(-1, D)[dmi].view(torch.int16), w.view(torch.int16)) for p, w in zip(pages, want))

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

    legs = {}
    fp8_pages = None
    for fmt, name in ((FMT_RAW, "raw"), (FMT_FP8, "fp8")):
        geom = KVGeometry(L, 1, D, NB, BS, C, 2, 0, fmt, _lib.LAYOUT_MLA)
        eng = KVEngine(geom, None, 0, staging_bytes=0)
        eng.register_kv_caches(pages)
        buf = torch.zeros(n_chunks * geom.chunk_bytes, dtype=torch.uint8, device=dev)
        g_ms = kernel_leg(eng, 0, lambda: eng.gather(sm, buf.data_ptr()))
        clear_dst()
        s_ms = kernel_leg(eng, 1, lambda: eng.scatter(dm, buf.data_ptr()))
        per_tok = 2 * L * D * 2 if fmt == FMT_RAW else L * (D * 2 + mo.MLA_RECORD)
        gb = per_tok * N_TOK / 1e9
        legs[f"{name}_gather" if fmt == FMT_RAW else "fp8_store"] = {
            "kernel_ms_median": g_ms[0], "kernel_ms_min": g_ms[1], "kernel_ms_max": g_ms[2], "GBps": gb / (g_ms[0] / 1e3)}
        legs[f"{name}_scatter" if fmt == FMT_RAW else "fp8_load"] = {
            "kernel_ms_median": s_ms[0], "kernel_ms_min": s_ms[1], "kernel_ms_max": s_ms[2], "GBps": gb / (s_ms[0] / 1e3)}
        if fmt == FMT_RAW:
            chunks = buf.view(n_chunks, L, C, D * 2)
            want = torch.stack([s.view(n_chunks, C, D) for s in src_snapshot], 1).view(torch.uint8)
            checks["raw_gather"] = bool(torch.equal(chunks, want.view(n_chunks, L, C, D * 2)))
            checks["raw_scatter"] = dst_equals(src_snapshot)
        else:
            # records of the first chunk, three layers, against the specification; decoded pages of those tokens
            rec = buf[:L * C * mo.MLA_RECORD].view(L, C, mo.MLA_RECORD)[[0, 30, 60]].cpu().numpy()
            host = np.stack([p.view(-1, D)[smi[:C]].cpu().view(torch.int16).numpy().view(np.uint16)
                             for p in (pages[0], pages[30], pages[60])])
            want = mo.fp8_pack_chunk(host.reshape(3, 1, C, 1, D))
            checks["fp8_store_sample"] = bool(np.array_equal(rec, want))
            dec = mo.fp8_unpack_chunk(rec).reshape(3, C, D)
            got = np.stack([p.view(-1, D)[dmi[:C]].cpu().view(torch.int16).numpy().view(np.uint16)
                            for p in (pages[0], pages[30], pages[60])])
            checks["fp8_load_sample"] = bool(np.array_equal(got, dec))
            fp8_pages = [p.view(-1, D)[dmi].clone() for p in pages]
        eng.close()
        del buf

        # ---- e2e through the pinned pool ------------------------------------------------------------------
        pool = KVPool(None, (n_chunks + 2) * geom.chunk_bytes, geom.chunk_bytes, 1)
        eng = KVEngine(geom, pool, 0, staging_bytes=16 * geom.chunk_bytes)
        eng.register_kv_caches(pages)
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
        ok = ok and dst_equals(src_snapshot if fmt == FMT_RAW else fp8_pages)
        checks[f"e2e_{name}"] = bool(ok)
        st, ld = np.median([t[0] for t in times]), np.median([t[1] for t in times])
        payload = geom.payload_bytes_per_token * N_TOK
        legs[f"e2e_{name}"] = {"store_ms": st * 1e3, "retrieve_ms": ld * 1e3, "payload_bytes": payload,
                               "store_GBps": payload / st / 1e9, "retrieve_GBps": payload / ld / 1e9,
                               "chunk_bytes": geom.chunk_bytes}
        eng.close()
        pool.close()

    result.update({"legs": legs, "bit_exact": checks, "all_bit_exact": all(checks.values()), "card": card(),
                   "steps": a.steps, "warmup": a.warmup})
    print(json.dumps(result), flush=True)
    return 0 if result["all_bit_exact"] else 1


if __name__ == "__main__":
    sys.exit(main())
