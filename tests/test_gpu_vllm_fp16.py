"""The connector under a REAL vLLM engine serving a model whose config says float16 (tiny Llama, real random
weights, see tests/vllm_fp16_driver.py) with dtype="auto": vLLM allocates an fp16 KV cache, and pass 2 must be
served from the pinned pool and match pass 1.

* RAW : identical greedy tokens, logprobs within the RAW tolerance of tests/test_gpu_vllm_connector.py;
* FP8 : the chosen token's logprob within FP8_LOGPROB_TOL of the recomputed one on the first 4 decode steps.
"""
import glob
import json
import os
import subprocess
import sys

import pytest

from tests.test_gpu_vllm_connector import FP8_LOGPROB_TOL, RAW_LOGPROB_TOL, _check_hits, _compare

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "production-stack_b200")
DRIVER = os.path.join(ROOT, "tests", "vllm_fp16_driver.py")


def _run(fmt: str, tmp_path):
    pytest.importorskip("vllm")
    pool = f"/b200kv-vllmfp16-{os.getpid()}-{fmt}"
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([PKG, env.get("PYTHONPATH", "")])
    env.update(LMCACHE_LOCAL_CPU="True", LMCACHE_MAX_LOCAL_CPU_SIZE="2", LMCACHE_CHUNK_SIZE="256",
               B200KV_FORMAT=fmt, B200KV_POOL_NAME=pool, B200KV_STAGING_MB="512", VLLM_LOGGING_LEVEL="WARNING",
               CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
    out_file = str(tmp_path / "result.json")
    from b200kv import KVPool
    try:
        p = subprocess.run([sys.executable, DRIVER, "--out", out_file], env=env, capture_output=True, text=True,
                           timeout=900)
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
def test_vllm_fp16_greedy_identical_with_kv_hit_raw(tmp_path):
    res = _run("raw", tmp_path)
    assert res["model_dtype"] == "torch.float16", res["model_dtype"]
    _check_hits(res)
    same, worst = _compare(res, 12, RAW_LOGPROB_TOL)
    print(f"fp16 raw: {same}/6 prompts identical, max |dlogprob| {worst:.5f}")
    assert same == 6, [(a["tokens"], b["tokens"]) for a, b in zip(res["first"], res["second"])]
    assert worst <= RAW_LOGPROB_TOL


@pytest.mark.gpu
def test_vllm_fp16_fp8_hit_within_tolerance(tmp_path):
    res = _run("fp8", tmp_path)
    assert res["model_dtype"] == "torch.float16", res["model_dtype"]
    _check_hits(res)
    same, worst = _compare(res, 4, FP8_LOGPROB_TOL)
    print(f"fp16 fp8: {same}/6 prompts agree on 4 steps (near-ties excepted), max |dlogprob| {worst:.4f}")
    assert same == 6
    assert worst <= FP8_LOGPROB_TOL
