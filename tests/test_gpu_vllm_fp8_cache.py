"""The connector under a REAL vLLM engine with an fp8 KV cache (tiny bf16 Llama, real random weights, see
tests/vllm_fp8_cache_driver.py): pass 2 must be served from the pinned pool and match pass 1.

* RAW : identical greedy tokens, logprobs within the FP8 tolerance of tests/test_gpu_vllm_connector.py.  The chunks
        are the pages' bytes (tests/test_gpu_fp8_cache.py), but vLLM's fp8 attention quantises the query as well, so
        its full prefill (pass 1) and its prefill of the last token over the loaded cache (pass 2) differ by more than
        the bf16 RAW tolerance allows (measured: 0.12 nats on an H100 80GB HBM3 at 700 W);
* FP8 : the connector logs that the fp8 pages are stored RAW (the driver captures its logger), and pass 2 matches
        as RAW does;
* Q4  : the chosen token's logprob within Q4_LOGPROB_TOL of the recomputed one on the first 4 decode steps, for
        e4m3 (--kv-cache-dtype fp8) and e5m2 caches.
"""
import glob
import json
import os
import subprocess
import sys

import pytest

from tests.test_gpu_vllm_connector import FP8_LOGPROB_TOL, _check_hits, _compare

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "production-stack_b200")
DRIVER = os.path.join(ROOT, "tests", "vllm_fp8_cache_driver.py")
# nats, on the chosen token of each of the first 4 decode steps: Q4 keeps 4 bits of every fp8 code, half a step of
# the group's scale is up to 1/14 of its largest value
Q4_LOGPROB_TOL = 1.0


def _run(fmt: str, kv_cache_dtype: str, tmp_path):
    pytest.importorskip("vllm")
    pool = f"/b200kv-vllmfp8kv-{os.getpid()}-{fmt}-{kv_cache_dtype}"
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([PKG, env.get("PYTHONPATH", "")])
    env.update(LMCACHE_LOCAL_CPU="True", LMCACHE_MAX_LOCAL_CPU_SIZE="2", LMCACHE_CHUNK_SIZE="256",
               B200KV_FORMAT=fmt, B200KV_POOL_NAME=pool, B200KV_STAGING_MB="512", VLLM_LOGGING_LEVEL="WARNING",
               CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
    out_file = str(tmp_path / "result.json")
    from b200kv import KVPool
    try:
        p = subprocess.run([sys.executable, DRIVER, "--out", out_file, "--kv-cache-dtype", kv_cache_dtype], env=env,
                           capture_output=True, text=True, timeout=900)
        assert p.returncode == 0 and os.path.exists(out_file), \
            f"vLLM driver failed (rc={p.returncode})\n--- stdout\n{p.stdout[-3000:]}\n--- stderr\n{p.stderr[-6000:]}"
        res = json.load(open(out_file))
        segs = glob.glob("/dev/shm" + pool + "*")
        assert segs, "the engine never created its pool segment"
        kp = KVPool("/" + os.path.basename(segs[0]), 0, 0, 2)
        res["pool"] = kp.stats()
        kp.close()
        return res
    finally:
        for f in glob.glob("/dev/shm" + pool + "*"):
            KVPool.unlink("/" + os.path.basename(f))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["raw", "fp8"])
def test_vllm_fp8_cache_greedy_identical_with_kv_hit_raw(fmt, tmp_path):
    res = _run(fmt, "fp8", tmp_path)
    assert res["cache_dtype"] == "fp8", res["cache_dtype"]
    assert res["chunk_format"] == 0, res["chunk_format"]                 # RAW either way
    if fmt == "fp8":
        assert any("already holds fp8 codes" in m and "stored RAW" in m for m in res["connector_log"]), res["connector_log"]
    _check_hits(res)
    same, worst = _compare(res, 12, FP8_LOGPROB_TOL)
    print(f"fp8 cache, B200KV_FORMAT={fmt}: {same}/6 prompts identical, max |dlogprob| {worst:.5f}")
    assert same == 6, [(a["tokens"], b["tokens"]) for a, b in zip(res["first"], res["second"])]
    assert worst <= FP8_LOGPROB_TOL


@pytest.mark.gpu
@pytest.mark.parametrize("kv_cache_dtype", ["fp8", "fp8_e5m2"])
def test_vllm_fp8_cache_q4_hit_within_tolerance(kv_cache_dtype, tmp_path):
    res = _run("q4", kv_cache_dtype, tmp_path)
    assert res["cache_dtype"] == kv_cache_dtype, res["cache_dtype"]
    assert res["chunk_format"] == 2, res["chunk_format"]
    _check_hits(res)
    same, worst = _compare(res, 4, Q4_LOGPROB_TOL)
    print(f"{kv_cache_dtype} cache, q4: {same}/6 prompts agree on 4 steps (near-ties excepted), "
          f"max |dlogprob| {worst:.4f}")
    assert same == 6
    assert worst <= Q4_LOGPROB_TOL
