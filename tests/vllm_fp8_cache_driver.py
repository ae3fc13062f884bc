"""Boot a real vLLM engine on a tiny bf16 Llama with an fp8 KV cache (--kv-cache-dtype fp8 / fp8_e5m2), with
B200KVConnector in the plugin slot, and run the same prompts twice.  Prints one JSON line with both passes' greedy
tokens and logprobs and the cache dtype vLLM chose.  Started as a subprocess by tests/test_gpu_vllm_fp8_cache.py
(never imported by the product)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time


def make_model(path: str, layers: int, vocab: int, seed: int = 0) -> None:
    """Llama-3-8B's per-layer KV geometry (8 KV heads x 128), real N(0, 0.02) weights, saved as bf16."""
    import torch
    from transformers import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2816, num_hidden_layers=layers, num_attention_heads=8,
                      num_key_value_heads=8, head_dim=128, vocab_size=vocab, max_position_embeddings=4096,
                      rms_norm_eps=1e-5, rope_theta=500000.0, tie_word_embeddings=False, bos_token_id=1,
                      eos_token_id=2, initializer_range=0.04, torch_dtype="bfloat16")
    m = LlamaForCausalLM(cfg).to(torch.bfloat16)
    m.save_pretrained(path, safe_serialization=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--vocab", type=int, default=4096)
    ap.add_argument("--model-dir", default="/tmp/b200kv-tiny-llama-bf16-fp8kv")
    ap.add_argument("--kv-cache-dtype", default="fp8")
    ap.add_argument("--max-tokens", type=int, default=12)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not os.path.exists(os.path.join(a.model_dir, "config.json")):
        make_model(a.model_dir, a.layers, a.vocab)

    import numpy as np
    from vllm import LLM, SamplingParams
    from vllm.config import KVTransferConfig

    ktc = KVTransferConfig(kv_connector="B200KVConnector", kv_connector_module_path="b200kv.connector",
                           kv_role="kv_both", kv_load_failure_policy="recompute")
    llm = LLM(model=a.model_dir, skip_tokenizer_init=True, dtype="auto", kv_cache_dtype=a.kv_cache_dtype, seed=0,
              max_model_len=4096, gpu_memory_utilization=0.25, enable_prefix_caching=False, enforce_eager=True,
              kv_transfer_config=ktc)
    vc = llm.llm_engine.vllm_config
    cache_dtype = str(vc.cache_config.cache_dtype)
    # the connector's geometry for this config, and what it logs deciding it (its "b200kv" logger has no handler in
    # vLLM's processes, so the driver asks again here with one)
    import logging

    from b200kv import connector
    from b200kv.config import B200KVConfig
    records = []
    handler = logging.Handler()
    handler.emit = records.append
    log = logging.getLogger("b200kv")
    log.addHandler(handler)
    log.setLevel(logging.INFO)
    connector._LOGGED.clear()
    chunk_format = connector.geometry_from_vllm(vc, B200KVConfig.from_env()).fmt
    log.removeHandler(handler)

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
    out = {"format": os.environ.get("B200KV_FORMAT", "raw"), "prompt_lens": [len(p) for p in prompts],
           "cache_dtype": cache_dtype, "chunk_format": chunk_format, "connector_log": [r.getMessage() for r in records],
           "first": first, "second": second}
    line = json.dumps(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line)
    print("RESULT " + line, flush=True)


if __name__ == "__main__":
    sys.exit(main())
