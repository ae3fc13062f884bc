"""The connector under a REAL vLLM engine with speculative decoding (see tests/vllm_spec_decode_driver.py): a tiny
DeepSeek-V3 with its MTP layer, and a tiny Llama with a one-layer EAGLE-3 drafter.  vLLM registers the target's
layers and the drafter's in one group; before draft layers were supported the engine failed in register_kv_caches.

Each model runs its prompts twice, with RAW and FP8 chunks, chunk-wise and layer-wise (one layer per group, so the
draft layer's group is its own and must be waited for in the last target layer's hook).  Required:

* the engine starts, and pass 2 is served from the pool (_check_hits);
* pass 2's greedy tokens agree with pass 1's under the rule of the existing vLLM tests (_compare): RAW over 12 steps,
  FP8 over the first 4 within the FP8 logprob bound;
* with RAW, the draft layer's pages at positions [0, n-1) of every prompt are bit-identical in both passes: pass 2
  loaded them.  Position n-1 is recomputed, because its draft KV depends on the token after it."""
import glob
import json
import os
import subprocess
import sys

import pytest

from tests.test_gpu_vllm_connector import FP8_LOGPROB_TOL, RAW_LOGPROB_TOL, _check_hits, _compare

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "production-stack_b200")
DRIVER = os.path.join(ROOT, "tests", "vllm_spec_decode_driver.py")


def _run(model, fmt, layerwise, tmp_path):
    pytest.importorskip("vllm")
    pool = f"/b200kv-vllmspec-{os.getpid()}-{model}-{fmt}-{layerwise}"
    snap = tmp_path / "snap"
    snap.mkdir()
    env = dict(os.environ)
    # the driver's connector subclass is loaded by module path (tests.vllm_spec_decode_driver) in vLLM's workers
    env["PYTHONPATH"] = os.pathsep.join([PKG, ROOT, env.get("PYTHONPATH", "")])
    env.update(LMCACHE_LOCAL_CPU="True", LMCACHE_MAX_LOCAL_CPU_SIZE="2", LMCACHE_CHUNK_SIZE="256",
               B200KV_FORMAT=fmt, B200KV_POOL_NAME=pool, B200KV_STAGING_MB="512", VLLM_LOGGING_LEVEL="WARNING",
               B200KV_LAYERWISE=layerwise, B200KV_LAYER_GROUP="1", B200KV_TEST_SNAPSHOT_DIR=str(snap),
               CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
    out_file = str(tmp_path / "result.json")
    from b200kv import KVPool
    try:
        p = subprocess.run([sys.executable, DRIVER, "--model", model, "--out", out_file], env=env,
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
@pytest.mark.parametrize("layerwise", ["0", "1"], ids=["chunkwise", "layerwise"])
@pytest.mark.parametrize("fmt", ["raw", "fp8"])
@pytest.mark.parametrize("model", ["deepseek-mtp", "llama-eagle3"])
def test_vllm_spec_decode_hit(model, fmt, layerwise, tmp_path):
    res = _run(model, fmt, layerwise, tmp_path)
    print(f"{model} {fmt} layer-wise {layerwise}: backend {res['backend']}, block size {res['block_size']}, "
          f"draft pages {res['draft_pages']}")
    _check_hits(res)
    if fmt == "raw":
        same, worst = _compare(res, 12, RAW_LOGPROB_TOL)
        assert same == 6, [(a["tokens"], b["tokens"]) for a, b in zip(res["first"], res["second"])]
        assert worst <= RAW_LOGPROB_TOL
        for n, d in zip(res["prompt_lens"], res["draft_pages"]):
            assert d is not None and d["n"] == n and d["nonzero"], d
            assert d["same_prefix"] >= n - 1, (n, d)
    else:
        same, worst = _compare(res, 4, FP8_LOGPROB_TOL)
        assert same == 6 and worst <= FP8_LOGPROB_TOL
        assert all(d is not None for d in res["draft_pages"])
