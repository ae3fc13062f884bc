"""Disaggregated prefill under REAL vLLM engines of different tensor-parallel sizes (tests/vllm_pd_hetero_driver.py):
a tiny Llama with 4 KV heads prefilled at TP=1 and decoded at TP=2, then the reverse.  The decoder's greedy output
matches a run without P/D within the RAW logprob tolerance of tests/test_gpu_vllm_connector.py, it pulled tokens, and
no pull failed.  Needs 2 GPUs (a TP=2 engine)."""
import json
import os
import subprocess
import sys

import pytest

from tests.test_gpu_vllm_connector import RAW_LOGPROB_TOL, _compare

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "production-stack_b200")
DRIVER = os.path.join(ROOT, "tests", "vllm_pd_hetero_driver.py")


@pytest.mark.gpu
@pytest.mark.parametrize("prefill_tp,decode_tp", [(1, 2), (2, 1)])
def test_vllm_pd_across_tensor_parallel_sizes(prefill_tp, decode_tp, tmp_path):
    pytest.importorskip("vllm")
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("a TP=2 engine needs 2 GPUs")
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([PKG, env.get("PYTHONPATH", "")])
    trace = str(tmp_path / "pd_trace.jsonl")
    env.update(LMCACHE_LOCAL_CPU="True", LMCACHE_MAX_LOCAL_CPU_SIZE="1", LMCACHE_CHUNK_SIZE="256",
               B200KV_SHM_DIR=str(tmp_path), B200KV_PD_TRACE=trace, VLLM_LOGGING_LEVEL="WARNING")
    out_file = str(tmp_path / "result.json")
    p = subprocess.run([sys.executable, DRIVER, "--prefill-tp", str(prefill_tp), "--decode-tp", str(decode_tp),
                        "--out", out_file], env=env, capture_output=True, text=True, timeout=1800)
    assert p.returncode == 0 and os.path.exists(out_file), \
        f"vLLM driver failed (rc={p.returncode})\n--- stdout\n{p.stdout[-3000:]}\n--- stderr\n{p.stderr[-6000:]}"
    res = json.load(open(out_file))
    events = [json.loads(l) for l in open(trace)] if os.path.exists(trace) else []
    pulled = sum(e.get("tokens", 0) for e in events if e["event"] == "pull_issued")
    failed = [e for e in events if e["event"] in ("pull_failed", "pull_invalidated")]
    assert pulled > 0 and not failed, (pulled, failed)
    same, worst = _compare(res, 12, RAW_LOGPROB_TOL)
    assert same == len(res["prompt_lens"]), [(a["tokens"], b["tokens"]) for a, b in zip(res["first"], res["second"])]
    assert worst <= RAW_LOGPROB_TOL
