"""The local-disk chunk tier on the bench.py wave (16 requests x 2 048 tokens of Llama-3-8B: 128 chunks) in RAW and
FP8, against the disk's own ceiling measured in the same run.  Prints one JSON line:

* ceiling: O_DIRECT sequential write and read of the same bytes to the same directory, one chunk per call, from 1
  and from 4 threads (the tier writes from one thread and reads on 4 lanes);
* write_GBps: write-through of the stored wave, pool -> disk (push of every chunk until the queue is drained);
* prefetch_GBps: disk -> pool for the wave's 16 requests, the pool emptied first (what the scheduler does while vLLM
  is told to ask again);
* disk_to_hbm_ms vs pool_to_hbm_ms: the wave's pages from disk-only chunks (prefetch + load) and from the pool (load);
* hash_share / copy_share: the part of the tier's own time spent in XXH64 of the payload and in bounce copies;
* the GPU name and power limit, and the filesystem and device behind the directory.
The directory is a fresh one under --dir (default $TMPDIR); everything written there is removed at exit.

    python tools/bench_disk.py [--dir /nvme] [--requests 16] [--tokens 2048]
"""
import argparse
import json
import mmap
import os
import shutil
import subprocess
import sys
import tempfile
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "production-stack_b200"))
from b200kv import FMT_FP8, FMT_RAW, KVEngine, KVGeometry, KVPool  # noqa: E402
from b200kv.disk import DiskTier, file_path, index_name  # noqa: E402

L, H, D, BS, C = 32, 8, 128, 16, 256      # Llama-3-8B, vLLM block 16, LMCache chunk 256


def where(directory: str) -> dict:
    """Filesystem, mount source and block device model behind a directory (from /proc and /sys, read only)."""
    best = ("", {})
    try:
        with open("/proc/self/mountinfo") as f:
            for line in f:
                a, b = line.split(" - ")
                parts, rest = a.split(), b.split()
                mnt = parts[4]
                if (directory + "/").startswith(mnt.rstrip("/") + "/") and len(mnt) >= len(best[0]):
                    best = (mnt, {"mount": mnt, "fstype": rest[0], "source": rest[1], "dev": parts[2]})
    except OSError:
        pass
    info = best[1]
    dev = info.get("dev")
    if dev:
        for rel in ("device/model", "../device/model"):
            try:
                with open(f"/sys/dev/block/{dev}/{rel}") as f:
                    info["model"] = f.read().strip()
                    break
            except OSError:
                continue
        try:
            st = os.statvfs(directory)
            info["free_GB"] = round(st.f_bavail * st.f_frsize / 1e9, 1)
        except OSError:
            pass
    return info


def gpu_info() -> dict:
    import torch
    out = {"gpu": torch.cuda.get_device_name(0)}
    try:
        r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        out["power_limit"], out["max_sm_clock"] = [x.strip() for x in r.stdout.strip().split(",")]
    except Exception as e:       # the numbers stand without it, but say so
        out["power_limit"] = f"unknown ({e})"
    return out


def ceiling(directory: str, n: int, chunk: int) -> dict:
    """O_DIRECT sequential write then read of n chunks of `chunk` bytes (4 KiB-rounded), one chunk per call."""
    chunk = (chunk + 4095) // 4096 * 4096
    path = os.path.join(directory, "ceiling.bin")
    buf = mmap.mmap(-1, chunk)                 # page-aligned, as O_DIRECT needs
    buf.write(np.random.default_rng(0).integers(0, 256, chunk, dtype=np.uint8).tobytes())
    out = {}
    fd = os.open(path, os.O_RDWR | os.O_CREAT | os.O_DIRECT, 0o600)
    try:
        os.posix_fallocate(fd, 0, n * chunk)
        for threads in (1, 4):
            for op in ("write", "read"):
                def work(i, op=op, threads=threads):
                    mine = mmap.mmap(-1, chunk)
                    mine.write(bytes(buf))
                    for c in range(i, n, threads):
                        if op == "write":
                            os.pwritev(fd, [mine], c * chunk)
                        else:
                            os.preadv(fd, [mine], c * chunk)
                ts = [threading.Thread(target=work, args=(i,)) for i in range(threads)]
                t0 = time.perf_counter()
                [t.start() for t in ts]
                [t.join() for t in ts]
                out[f"{op}_GBps_{threads}t"] = round(n * chunk / (time.perf_counter() - t0) / 1e9, 3)
    finally:
        os.close(fd)
        os.unlink(path)
    out["write_GBps"] = max(v for k, v in out.items() if k.startswith("write"))
    out["read_GBps"] = max(v for k, v in out.items() if k.startswith("read"))
    return out


def leg(directory: str, fmt: int, requests: int, tokens: int, reps: int = 5) -> dict:
    import torch
    n_tok = requests * tokens
    nb = n_tok // BS + 16
    geom = KVGeometry(L, H, D, nb, BS, C, 2, 0, fmt)
    cb, n_chunks = geom.chunk_bytes, requests * ((tokens + C - 1) // C)
    gen = torch.Generator(device="cuda:0").manual_seed(fmt)
    src = [torch.randn((2, nb, BS, H, D), generator=gen, device="cuda:0").bfloat16() for _ in range(L)]
    dst = [torch.zeros_like(t) for t in src]
    pool = KVPool(None, (n_chunks + 4) * cb, cb, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=2 * 16 * cb)
    eng.register_kv_caches(src)
    eng_d = KVEngine(geom, pool, 0, staging_bytes=2 * 16 * cb)
    eng_d.register_kv_caches(dst)
    rng = np.random.default_rng(fmt)
    perm = rng.permutation(n_tok // BS)
    reqs = []
    for r in range(requests):
        toks = (np.arange(tokens, dtype=np.int32) + 100_000 * r + 7 * fmt) % 128_000
        blocks = perm[r * tokens // BS:(r + 1) * tokens // BS]
        sm = (blocks[:, None] * BS + np.arange(BS)[None, :]).reshape(-1)[:tokens].astype(np.int64)
        reqs.append((toks, sm, 0))
    eng.wait(eng.store_batch(reqs))

    def load():
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        loaded, ticket = eng_d.retrieve_batch(reqs)
        eng_d.wait(ticket)
        torch.cuda.synchronize()
        assert sum(loaded) == n_tok, loaded
        return time.perf_counter() - t0

    load()                                             # warm-up
    pool_ms = sorted(load() for _ in range(reps))[reps // 2] * 1e3
    want = [int(t.view(torch.int16).sum(dtype=torch.int64)) for t in dst]

    disk_bytes = 4096 + (n_chunks + 4) * (4096 + (cb + 4095) // 4096 * 4096)
    writer = DiskTier(pool, directory, disk_bytes, C, eng.key_seed, push_queue=n_chunks)
    index = index_name(directory, cb)              # the shm index outlives the tier on purpose: removed here
    try:
        return disk_legs(writer, directory, disk_bytes, cb, n_chunks, n_tok, reqs, pool, eng, dst, load, want, pool_ms)
    finally:
        KVPool.unlink(index)
        eng.close()
        eng_d.close()
        pool.close()


def disk_legs(writer, directory, disk_bytes, cb, n_chunks, n_tok, reqs, pool, eng, dst, load, want, pool_ms):
    import torch
    keys = [int(k) for t, _, _ in reqs for k in eng._keys(t)]
    t0 = time.perf_counter()
    writer.push(keys)
    assert writer.flush(600)
    t_write = time.perf_counter() - t0
    ws, wf = writer.stats(), writer.file.stats()
    assert ws["written_chunks"] == n_chunks, ws
    writer.close()

    assert pool.clear() and eng.lookup(reqs[0][0]) == 0
    for t in dst:
        t.zero_()
    reader = DiskTier(pool, directory, disk_bytes, C, eng.key_seed, wait_s=600.0)
    t0 = time.perf_counter()
    pending = {f"r{i}": t for i, (t, _, _) in enumerate(reqs)}
    while pending:
        for rid in [r for r, t in pending.items() if reader.prefetch_state(r, t) == reader.DONE]:
            pending.pop(rid)
        time.sleep(0.0005)
    t_prefetch = time.perf_counter() - t0
    rs, rf = reader.stats(), reader.file.stats()
    assert rs["fetched_chunks"] == n_chunks and rs["corrupt_chunks"] == 0, rs
    t_load = load()
    got = [int(t.view(torch.int16).sum(dtype=torch.int64)) for t in dst]
    assert got == want, "pages loaded from disk differ from pages loaded from the pool"
    reader.close()
    os.unlink(file_path(directory, cb))               # the next leg's file takes the space

    def share(st, key):
        busy = st["hash_ns"] + st["copy_ns"] + st["io_ns"]
        return round(st[key] / busy, 4) if busy else None

    total = n_chunks * cb
    return {"chunk_bytes": cb, "chunks": n_chunks, "bytes": total, "direct_io": rs["direct_io"],
            "write_GBps": round(total / t_write / 1e9, 3), "prefetch_GBps": round(total / t_prefetch / 1e9, 3),
            "pool_to_hbm_ms": round(pool_ms, 2), "disk_to_hbm_ms": round((t_prefetch + t_load) * 1e3, 2),
            "prefetch_ms": round(t_prefetch * 1e3, 2), "load_after_prefetch_ms": round(t_load * 1e3, 2),
            "write_hash_share": share(wf, "hash_ns"), "write_copy_share": share(wf, "copy_ns"),
            "read_hash_share": share(rf, "hash_ns"), "read_copy_share": share(rf, "copy_ns"),
            "write_hash_share_of_wall": round(wf["hash_ns"] / 1e9 / t_write, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default=None, help="where to put the tier (a fresh directory is made inside)")
    ap.add_argument("--requests", type=int, default=16)
    ap.add_argument("--tokens", type=int, default=2048)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_disk.py measures disk -> HBM and needs a GPU")
    directory = tempfile.mkdtemp(prefix="b200kv-bench-disk-", dir=args.dir)
    out = {"workload": f"{args.requests} x {args.tokens} tokens, Llama-3-8B (L=32, H=8, D=128), chunk {C}",
           "dir": directory, "host_cores": len(os.sched_getaffinity(0)), **gpu_info(), "filesystem": where(directory)}
    try:
        raw_chunk = KVGeometry(L, H, D, 1, BS, C, 2, 0, FMT_RAW).chunk_bytes
        out["ceiling"] = ceiling(directory, args.requests * ((args.tokens + C - 1) // C), raw_chunk)
        for name, fmt in (("raw", FMT_RAW), ("fp8", FMT_FP8)):
            r = leg(directory, fmt, args.requests, args.tokens)
            r["write_of_ceiling"] = round(r["write_GBps"] / out["ceiling"]["write_GBps"], 3)
            r["prefetch_of_ceiling"] = round(r["prefetch_GBps"] / out["ceiling"]["read_GBps"], 3)
            out[name] = r
    finally:
        shutil.rmtree(directory, ignore_errors=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
