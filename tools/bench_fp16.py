"""FP8 and Q4 kernels on bf16 vs fp16 KV caches, on one GPU: prints one JSON line.

K/V legs at Llama-3-8B geometry (32 layers, 8 KV heads x 128, vLLM block 16, LMCache chunk 256), MLA legs at
DeepSeek-V3 geometry (61 layers, 576-element latent, block 64); 32 768 tokens per step, their blocks scattered over
the pages.  For each format a bf16 engine and an fp16 engine run ALTERNATELY in this one process (step i: bf16 leg,
then fp16 leg), so clock and thermal drift hit both alike:

* fp8_store / fp8_load, q4_store / q4_load: device-resident gather / scatter (b200kv_gather / b200kv_scatter, the
  block-structured mapping takes the persistent FP8 store), kernel time from the engine's CUDA events;
* mla_fp8_store / mla_fp8_load: the FP8 latent-record kernels.

Algorithmic bytes (DESIGN §3): a store reads the 16-bit pages and writes the chunk format, a load the reverse, so
bytes per token = planes * H * D * 2 + format bytes per token (KVGeometry.payload_bytes_per_token); GB/s = those
bytes over the median kernel time.  Every leg is checked against the oracle (tests/fp16_oracle.py
with the engine's dtype) on a sample: the chunk bytes of the first chunk for two layers, and
the decoded pages of those tokens.  The card's name, power limit and max SM clock are read in the same run.

    python tools/bench_fp16.py [--steps 10] [--warmup 3]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "production-stack_b200")]

import numpy as np  # noqa: E402

from tools.bench_mla import card  # noqa: E402

N_TOK = 32768
KV = dict(L=32, H=8, D=128, BS=16, C=256)
MLA = dict(L=61, D=576, BS=64, C=256)
SAMPLE_LAYERS = (0, 1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()

    import torch

    from b200kv import DTYPE_BF16, DTYPE_FP16, FMT_FP8, FMT_Q4, KVEngine, KVGeometry, _lib
    from oracle import kv_oracle as ko
    from tests import fp16_oracle as fo
    from tests import mla_oracle as mo
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp16.py needs a GPU: there is no CPU path to measure")
    dev = torch.device("cuda:0")
    tdt = {DTYPE_BF16: torch.bfloat16, DTYPE_FP16: torch.float16}
    dname = {DTYPE_BF16: "bf16", DTYPE_FP16: "fp16"}
    legs, checks = {}, {}

    def bits(t):
        return t.cpu().view(torch.int16).numpy().view(np.uint16)

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

    def record(name, dt, t, gb):
        legs[f"{name}_{dname[dt]}"] = {"kernel_ms_median": t[0], "kernel_ms_min": t[1], "kernel_ms_max": t[2],
                                      "GBps": gb / (t[0] / 1e3)}

    rng = np.random.default_rng(0)

    # ---- K/V: FP8 and Q4 ---------------------------------------------------------------------------------------
    L, H, D, BS, C = KV["L"], KV["H"], KV["D"], KV["BS"], KV["C"]
    nb_need = N_TOK // BS
    NB = 2 * nb_need + 8
    perm = rng.permutation(NB)
    sm = ko.slot_mapping_from_blocks(perm[:nb_need], BS, N_TOK)
    dm = ko.slot_mapping_from_blocks(perm[nb_need:2 * nb_need], BS, N_TOK)
    smi, dmi = torch.from_numpy(sm).to(dev), torch.from_numpy(dm).to(dev)
    g = torch.Generator(device=dev).manual_seed(0)
    src32 = [torch.randn((2, NB, BS, H, D), generator=g, device=dev) for _ in range(L)]
    pages = {dt: [x.to(tdt[dt]) for x in src32] for dt in (DTYPE_BF16, DTYPE_FP16)}
    del src32
    for fmt, name in ((FMT_FP8, "fp8"), (FMT_Q4, "q4")):
        engines, bufs = [], []
        for dt in (DTYPE_BF16, DTYPE_FP16):
            geom = KVGeometry(L, H, D, NB, BS, C, 2, 0, fmt, _lib.LAYOUT_NHD, dt)
            e = KVEngine(geom, None, 0, staging_bytes=0)
            e.register_kv_caches(pages[dt])
            engines.append(e)
            bufs.append(torch.zeros((N_TOK // C) * geom.chunk_bytes, dtype=torch.uint8, device=dev))
        geom = engines[0].geom
        gb = (geom.planes * H * D * 2 + geom.payload_bytes_per_token) * N_TOK / 1e9
        st = timed_pair(engines, 0, [lambda e=e, b=b: e.gather(sm, b.data_ptr()) for e, b in zip(engines, bufs)])
        ld = timed_pair(engines, 1, [lambda e=e, b=b: e.scatter(dm, b.data_ptr()) for e, b in zip(engines, bufs)])
        for i, dt in enumerate((DTYPE_BF16, DTYPE_FP16)):
            record(f"{name}_store", dt, st[i], gb)
            record(f"{name}_load", dt, ld[i], gb)
            # sample: the first chunk of two layers against the oracle with this engine's dtype
            o = "bf16" if dt == DTYPE_BF16 else "fp16"
            host = np.stack([bits(pages[dt][l].view(2, -1, H, D)[:, smi[:C]]) for l in SAMPLE_LAYERS])   # (2,2,C,H,D)
            chunk = bufs[i][:geom.chunk_bytes].cpu().numpy()
            if fmt == FMT_FP8:
                codes, scales = fo.fp8_pack_chunk(host, o)
                so = geom.planes * C * H * D
                got_s = chunk[so:so + geom.planes * H * 4].copy().view(np.float32).reshape(L, 2, H)[list(SAMPLE_LAYERS)]
                got_c = chunk[:so].reshape(L, 2, C, H, D)[list(SAMPLE_LAYERS)]
                ok_store = np.array_equal(got_c, codes) and np.array_equal(got_s, scales)
                dec = fo.fp8_unpack_chunk(codes, scales, o)
            else:
                codes, sc = fo.q4_pack_chunk(host, o)
                rec = H * D // 2 + H * (D // 32) * 2
                r = chunk[:geom.planes * C * rec].reshape(L, 2, C, rec)[list(SAMPLE_LAYERS)]
                ok_store = np.array_equal(r[..., :H * D // 2], codes.reshape(2, 2, C, -1)) and \
                    np.array_equal(r[..., H * D // 2:].copy().view(np.uint16), sc.reshape(2, 2, C, -1))
                dec = fo.q4_unpack_chunk(codes, sc, o)
            got = np.stack([bits(pages[dt][l].view(2, -1, H, D)[:, dmi[:C]]) for l in SAMPLE_LAYERS])
            checks[f"{name}_store_{dname[dt]}"] = bool(ok_store)
            checks[f"{name}_load_{dname[dt]}"] = bool(np.array_equal(got, dec))
        for e in engines:
            e.close()
        del bufs
    del pages
    torch.cuda.empty_cache()

    # ---- MLA FP8 latent records ------------------------------------------------------------------------------
    L, D, BS, C = MLA["L"], MLA["D"], MLA["BS"], MLA["C"]
    nb_need = N_TOK // BS
    NB = 2 * nb_need + 8
    perm = rng.permutation(NB)
    sm = ko.slot_mapping_from_blocks(perm[:nb_need], BS, N_TOK)
    dm = ko.slot_mapping_from_blocks(perm[nb_need:2 * nb_need], BS, N_TOK)
    smi, dmi = torch.from_numpy(sm).to(dev), torch.from_numpy(dm).to(dev)
    engines, bufs, mpages = [], [], {}
    for dt in (DTYPE_BF16, DTYPE_FP16):
        mpages[dt] = [torch.randn((NB, BS, D), generator=g, device=dev).to(tdt[dt]) for _ in range(L)]
        geom = KVGeometry(L, 1, D, NB, BS, C, 2, 0, FMT_FP8, _lib.LAYOUT_MLA, dt)
        e = KVEngine(geom, None, 0, staging_bytes=0)
        e.register_kv_caches(mpages[dt])
        engines.append(e)
        bufs.append(torch.zeros((N_TOK // C) * geom.chunk_bytes, dtype=torch.uint8, device=dev))
    gb = L * (D * 2 + mo.MLA_RECORD) * N_TOK / 1e9
    st = timed_pair(engines, 0, [lambda e=e, b=b: e.gather(sm, b.data_ptr()) for e, b in zip(engines, bufs)])
    ld = timed_pair(engines, 1, [lambda e=e, b=b: e.scatter(dm, b.data_ptr()) for e, b in zip(engines, bufs)])
    for i, dt in enumerate((DTYPE_BF16, DTYPE_FP16)):
        record("mla_fp8_store", dt, st[i], gb)
        record("mla_fp8_load", dt, ld[i], gb)
        o = "bf16" if dt == DTYPE_BF16 else "fp16"
        rec = bufs[i][:L * C * mo.MLA_RECORD].view(L, C, mo.MLA_RECORD)[list(SAMPLE_LAYERS)].cpu().numpy()
        host = np.stack([bits(mpages[dt][l].view(-1, D)[smi[:C]]) for l in SAMPLE_LAYERS])
        want = fo.mla_fp8_pack_chunk(host.reshape(len(SAMPLE_LAYERS), 1, C, 1, D), o)
        checks[f"mla_fp8_store_{dname[dt]}"] = bool(np.array_equal(rec, want))
        dec = fo.mla_fp8_unpack_chunk(rec, o).reshape(len(SAMPLE_LAYERS), C, D)
        got = np.stack([bits(mpages[dt][l].view(-1, D)[dmi[:C]]) for l in SAMPLE_LAYERS])
        checks[f"mla_fp8_load_{dname[dt]}"] = bool(np.array_equal(got, dec))
    for e in engines:
        e.close()

    ratio = {k[:-5]: legs[k[:-5] + "_fp16"]["kernel_ms_median"] / legs[k]["kernel_ms_median"]
             for k in legs if k.endswith("_bf16")}
    result = {"tokens": N_TOK, "kv_geometry": KV, "mla_geometry": MLA, "legs": legs,
              "fp16_over_bf16_time": ratio, "bit_exact": checks, "all_bit_exact": all(checks.values()),
              "card": card(), "steps": a.steps, "warmup": a.warmup}
    print(json.dumps(result), flush=True)
    return 0 if result["all_bit_exact"] else 1


if __name__ == "__main__":
    sys.exit(main())
