"""The connector under a REAL vLLM engine serving a sparse-attention MLA model (tiny DeepSeek-V3.2 with random
weights, see tests/vllm_mla_sparse_driver.py): vLLM registers a latent and an indexer cache per layer, pass 2 must
be served from the pinned pool and match pass 1 with RAW chunks: the same greedy tokens on every prompt (a step whose
top-2 margin is a near-tie at the bound may differ, as in tests/test_gpu_vllm_connector.py), and logprobs within
SPARSE_RAW_LOGPROB_TOL.  Prompts are longer than index_topk, so a wrong or late indexer
key changes which tokens the sparse attention reads.

The logprob bound is wider than the dense models' RAW_LOGPROB_TOL (0.08).  Pass 2 recomputes only each prompt's tail,
through vLLM's prefill-with-cached-context kernels, so its hidden states differ from pass 1's in the last bits, as for
every model.  Here those bits also feed the indexer, whose top-k over 512 of up to 3 329 tokens is a step function: a
near-tie at the 512th score can swap one attended token.  Measured on an H100 with layer-wise loads of one layer per
group: 6/6 prompts agree over 12 steps, max |dlogprob| 0.125.

Two load schedules: chunk-wise, and layer-wise with one layer per group (the default schedule, at its finest), where
vLLM runs each layer's indexer before the layer's attention hook: the connector must have waited for that layer's
group (both planes) before the indexer reads its keys."""
import os

import pytest

from tests.test_gpu_vllm_connector import _check_hits, _compare
from tests import test_gpu_vllm_mla as base

DRIVER = os.path.join(base.ROOT, "tests", "vllm_mla_sparse_driver.py")
SPARSE_RAW_LOGPROB_TOL = 0.25   # nats; see the module docstring


@pytest.mark.gpu
@pytest.mark.parametrize("layerwise", ["0", "1"])
def test_vllm_deepseek_v32_greedy_identical_with_kv_hit_raw(layerwise, tmp_path, monkeypatch):
    monkeypatch.setattr(base, "DRIVER", DRIVER)
    monkeypatch.setenv("B200KV_LAYERWISE", layerwise)
    monkeypatch.setenv("B200KV_LAYER_GROUP", "1")
    res = base._run("raw", tmp_path)
    print(f"sparse MLA backend {res['backend']}, block size {res['block_size']}, layer-wise {layerwise}")
    _check_hits(res)
    same, worst = _compare(res, 12, SPARSE_RAW_LOGPROB_TOL)
    print(f"v3.2 raw: {same}/6 prompts identical, max |dlogprob| {worst:.5f}")
    assert same == 6, [(a["tokens"], b["tokens"]) for a, b in zip(res["first"], res["second"])]
    assert worst <= SPARSE_RAW_LOGPROB_TOL
