"""Peer pull between replicas of different tensor-parallel sizes, at Llama-3-70B KV geometry: prints one JSON line.

Geometry: 80 layers, 8 KV heads, head_dim 128, block size 16, bf16; 16 sessions x 2048 tokens = 32 768 tokens per
pull, their blocks scattered over the pages on both sides.  Legs, each in NHD and HND tile order:

* tp2to4: decode rank 0 of TP=4 (2 heads) pulls heads [0, 2) of prefill rank 0 of TP=2 (4 heads): one sliced pull,
  512-byte NHD rows;
* tp2to1: the TP=1 decoder (8 heads) pulls heads [0, 4) from prefill rank 0 and [4, 8) from rank 1: two sliced
  pulls into one page set;
* same2 / same8: a same-TP pull of the same bytes (2 heads, 8 heads per token) through the unsliced path.

Time is the pull kernels' (b200kv_last_kernel_ms, CUDA events on the launching stream), median over the steps;
bytes are the payload read once, n_tokens * 2 planes * L * heads moved * D * 2.  `ratio` is each sliced leg's
bytes/s over that of the same-TP leg of equal bytes; the target is 0.8.  Every leg's pages are checked bit for bit
against torch indexing of the source pages on the first and last layer.  With two GPUs the producer also sits on
device 1 and the NHD legs are repeated over NVLink.  The card's name and power limit are read in the same run.

    python tools/bench_pd_hetero.py [--steps 10] [--warmup 2]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "production-stack_b200")]

import numpy as np  # noqa: E402

L, T, D, BS = 80, 8, 128, 16
SESSIONS, SESSION_TOKENS = 16, 2048
N_TOK = SESSIONS * SESSION_TOKENS
NB = N_TOK // BS + 64
TARGET = 0.8


def card(dev: int = 0) -> dict:
    try:
        out = subprocess.run(["nvidia-smi", f"--id={dev}", "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30).stdout
        name, pw, clk = [x.strip() for x in out.strip().split(",")]
        return {"name": name, "power_limit_w": float(pw), "max_sm_mhz": float(clk)}
    except Exception as e:  # the numbers below still stand; the card is named by torch
        import torch
        return {"name": torch.cuda.get_device_name(dev), "power_limit_w": None, "error": repr(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()

    import torch

    from b200kv import FMT_RAW, KVEngine, KVGeometry, _lib, pd
    if not torch.cuda.is_available():
        raise SystemExit("bench_pd_hetero needs a CUDA device")

    def pages(H, dev, seed):
        """One cache per layer, (2, NB, BS*H*D) int16 (bf16 bits): the same bytes serve both tile orders."""
        g = torch.Generator(device=dev).manual_seed(seed)
        return [torch.randint(-32768, 32767, (2, NB, BS * H * D), generator=g, device=dev, dtype=torch.int16)
                for _ in range(L)]

    def as_tokens(x, H, hnd):
        """(2, NB, BS*H*D) of one tile order -> (2, NB*BS, H, D)."""
        v = x.view(2, NB, H, BS, D).permute(0, 1, 3, 2, 4) if hnd else x.view(2, NB, BS, H, D)
        return v.reshape(2, NB * BS, H, D)

    def engine(H, caches, hnd, dev):
        g = KVGeometry(L, H, D, NB, BS, 256, 2, 0, FMT_RAW, _lib.LAYOUT_HND if hnd else _lib.LAYOUT_NHD)
        e = KVEngine(g, None, dev, staging_bytes=0)
        e.register_kv_ptrs([c[0].data_ptr() for c in caches], [c[1].data_ptr() for c in caches])
        return e

    rng = np.random.default_rng(0)
    src = pd.slots_of(rng.permutation(NB)[: N_TOK // BS], BS, N_TOK)
    dst = pd.slots_of(rng.permutation(NB)[: N_TOK // BS], BS, N_TOK)

    def run(eng, sources, dev):
        """median kernel ms of pulling every source, after warm-up"""
        torch.cuda.set_device(dev)
        times = []
        for step in range(a.warmup + a.steps):
            ms = 0.0
            for pid in sources:
                eng.wait(eng.peer_pull(pid, src, dst))
                ms += eng.last_kernel_ms(2)
            if step >= a.warmup:
                times.append(ms)
        return float(np.median(times))

    def check(local, H, hnd, parts):
        """parts: [(peer caches, peer heads, src_head0, dst_head0, n_heads)]: layers 0 and L-1 bit-exact."""
        si, di = torch.from_numpy(src).to(local[0].device), torch.from_numpy(dst).to(local[0].device)
        for l in (0, L - 1):
            got = as_tokens(local[l], H, hnd)[:, di]
            for peer, hp, s0, d0, n in parts:
                want = as_tokens(peer[l], hp, hnd)[:, si][:, :, s0:s0 + n].to(got.device)
                if not torch.equal(got[:, :, d0:d0 + n], want):
                    return False
        return True

    def legs(prod_dev, layouts):
        out, exact = {}, True
        pdev = f"cuda:{prod_dev}"
        p0, p1 = pages(4, pdev, 1), pages(4, pdev, 2)                 # prefill ranks 0 and 1 of TP=2
        same2, same8 = pages(2, pdev, 3), pages(8, pdev, 4)           # same-TP producers
        loc2, loc8 = pages(2, "cuda:0", 5), pages(8, "cuda:0", 6)
        stride4 = BS * 4 * D * 2
        for hnd in layouts:
            lay = "hnd" if hnd else "nhd"
            e2, e8 = engine(2, loc2, hnd, 0), engine(8, loc8, hnd, 0)
            ptrs = lambda c: ([x[0].data_ptr() for x in c], [x[1].data_ptr() for x in c])   # noqa: E731
            e2.import_peer_ptrs(0, prod_dev, *ptrs(p0), peer_block_stride=stride4, head_slice=(4, 0, 0, 2))
            e2.import_peer_ptrs(1, prod_dev, *ptrs(same2))
            e8.import_peer_ptrs(0, prod_dev, *ptrs(p0), peer_block_stride=stride4, head_slice=(4, 0, 0, 4))
            e8.import_peer_ptrs(1, prod_dev, *ptrs(p1), peer_block_stride=stride4, head_slice=(4, 0, 4, 4))
            e8.import_peer_ptrs(2, prod_dev, *ptrs(same8))
            for name, eng, srcs, heads, parts, H, local in (
                    ("tp2to4", e2, [0], 2, [(p0, 4, 0, 0, 2)], 2, loc2),
                    ("same2", e2, [1], 2, [(same2, 2, 0, 0, 2)], 2, loc2),
                    ("tp2to1", e8, [0, 1], 8, [(p0, 4, 0, 0, 4), (p1, 4, 0, 4, 4)], 8, loc8),
                    ("same8", e8, [2], 8, [(same8, 8, 0, 0, 8)], 8, loc8)):
                ms = run(eng, srcs, 0)
                nbytes = N_TOK * 2 * L * heads * D * 2
                ok = check(local, H, hnd, parts)
                exact &= ok
                out[f"{name}_{lay}"] = {"ms": round(ms, 4), "bytes": nbytes, "GBps": round(nbytes / ms / 1e6, 1),
                                        "bit_exact": ok}
            e2.close()
            e8.close()
            out[f"ratio_tp2to4_{lay}"] = round(out[f"tp2to4_{lay}"]["GBps"] / out[f"same2_{lay}"]["GBps"], 3)
            out[f"ratio_tp2to1_{lay}"] = round(out[f"tp2to1_{lay}"]["GBps"] / out[f"same8_{lay}"]["GBps"], 3)
        del p0, p1, same2, same8, loc2, loc8
        torch.cuda.empty_cache()
        return out, exact

    one, exact = legs(0, (False, True))
    ratios = {k: v for k, v in one.items() if k.startswith("ratio")}
    res = {"bench": "pd_hetero", "card": card(0), "geometry": {"layers": L, "kv_heads": T, "head_dim": D,
           "block_tokens": BS, "dtype": "bf16", "tokens": N_TOK}, "steps": a.steps, "warmup": a.warmup,
           "one_device": one, "target_ratio": TARGET, "target_met": all(r >= TARGET for r in ratios.values()),
           "bit_exact": exact}
    if torch.cuda.device_count() > 1:
        cross, ok = legs(1, (False,))
        res["cross_device"] = cross
        res["bit_exact"] = exact and ok
    else:
        res["cross_device"] = "one GPU visible: not measured"
    print(json.dumps(res))


if __name__ == "__main__":
    main()
