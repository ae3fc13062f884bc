"""Boot a real vLLM engine on a tiny DeepSeek-V3.2 (multi-head latent attention with DeepSeek Sparse Attention: a
lightning indexer per layer and top-k sparse MLA; random weights, no tokenizer) with B200KVConnector in the plugin
slot and run the same prompts twice, as tests/vllm_mla_driver.py does for DeepSeek-V2.  The model is one config.json
(model_type deepseek_v32, vLLM's DeepseekV32ForCausalLM); vLLM's dummy loader fills the weights and spread_weights
redraws them.  Prints one JSON line with both passes' greedy tokens and logprobs, the attention backend and the block
size.  Started as a subprocess by tests/test_gpu_vllm_mla_sparse.py (never imported by the product)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time


def make_config(path: str, layers: int, vocab: int) -> None:
    os.makedirs(path, exist_ok=True)
    cfg = {"architectures": ["DeepseekV32ForCausalLM"], "model_type": "deepseek_v32", "vocab_size": vocab,
           "hidden_size": 1024, "intermediate_size": 2816, "moe_intermediate_size": 256, "num_hidden_layers": layers,
           "num_attention_heads": 16, "num_key_value_heads": 16, "kv_lora_rank": 512, "q_lora_rank": 384,
           "qk_rope_head_dim": 64, "qk_nope_head_dim": 128, "v_head_dim": 128, "first_k_dense_replace": layers,
           "n_routed_experts": 4, "num_experts_per_tok": 2, "n_shared_experts": 1, "n_group": 1, "topk_group": 1,
           "routed_scaling_factor": 1.0, "norm_topk_prob": True, "scoring_func": "sigmoid", "topk_method": "noaux_tc",
           "max_position_embeddings": 4096, "rms_norm_eps": 1e-6, "rope_theta": 10000.0,
           "tie_word_embeddings": False, "bos_token_id": 1, "eos_token_id": 2, "initializer_range": 0.02,
           "torch_dtype": "bfloat16", "hidden_act": "silu",
           # DeepSeek Sparse Attention: what makes vLLM build the indexer (deepseek_v2.py: hasattr index_topk)
           "index_topk": 512, "index_head_dim": 128, "index_n_heads": 64}
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(cfg, f)


def spread_weights(model) -> int:
    """vLLM's dummy weights (uniform +-1e-3, norms included) give near-uniform logits, so pass 1 and pass 2 would
    agree whatever attention read.  Redraw them: norms 1, every other weight N(0, 0.05), seeded."""
    import torch
    g = torch.Generator(device="cuda").manual_seed(0)
    for name, p in model.named_parameters():
        if not p.dtype.is_floating_point or p.dtype.itemsize < 2:
            continue
        if "norm" in name:
            p.data.fill_(1.0)
        else:
            p.data.normal_(0.0, 0.05, generator=g)
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--vocab", type=int, default=4096)
    ap.add_argument("--model-dir", default="/tmp/b200kv-tiny-deepseek-v32")
    ap.add_argument("--max-tokens", type=int, default=12)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    make_config(a.model_dir, a.layers, a.vocab)

    os.environ.setdefault("VLLM_ALLOW_INSECURE_SERIALIZATION", "1")   # apply_model ships spread_weights
    import numpy as np
    from vllm import LLM, SamplingParams
    from vllm.config import KVTransferConfig

    ktc = KVTransferConfig(kv_connector="B200KVConnector", kv_connector_module_path="b200kv.connector",
                           kv_role="kv_both", kv_load_failure_policy="recompute")
    llm = LLM(model=a.model_dir, skip_tokenizer_init=True, dtype="bfloat16", seed=0, max_model_len=4096,
              gpu_memory_utilization=0.25, enable_prefix_caching=False, enforce_eager=True, load_format="dummy",
              kv_transfer_config=ktc)
    llm.apply_model(spread_weights)
    backend, block_size = None, None
    try:
        vc = llm.llm_engine.vllm_config
        block_size = vc.cache_config.block_size
        backend = str(getattr(vc.attention_config, "backend", None))
    except Exception as e:
        backend = f"unknown ({e!r})"

    # prompts longer than index_topk, so the indexer's top-k selection decides what attention sees
    rng = np.random.default_rng(1234)
    shared = rng.integers(3, a.vocab, 512).tolist()
    prompts = []
    for i, n in enumerate((300, 700, 1029, 1536, 2100, 2817)):
        body = rng.integers(3, a.vocab, n).tolist()
        prompts.append((shared + body) if i % 2 else body)
    sp = SamplingParams(temperature=0.0, max_tokens=a.max_tokens, logprobs=5, detokenize=False, ignore_eos=True)

    def run():
        outs = llm.generate([{"prompt_token_ids": p} for p in prompts], sp, use_tqdm=False)
        res = []
        for o in outs:
            c = o.outputs[0]
            steps = []
            for t, step in zip(c.token_ids, c.logprobs or []):
                top = sorted((float(v.logprob) for v in step.values()), reverse=True)
                steps.append({"lp": float(step[t].logprob), "margin": top[0] - top[1] if len(top) > 1 else 99.0})
            res.append({"tokens": [int(t) for t in c.token_ids], "steps": steps})
        return res

    first = run()
    time.sleep(1.0)
    second = run()
    out = {"format": os.environ.get("B200KV_FORMAT", "raw"), "layerwise": os.environ.get("B200KV_LAYERWISE", "0"),
           "prompt_lens": [len(p) for p in prompts], "backend": backend, "block_size": block_size,
           "first": first, "second": second}
    line = json.dumps(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line)
    print("RESULT " + line, flush=True)


if __name__ == "__main__":
    sys.exit(main())
