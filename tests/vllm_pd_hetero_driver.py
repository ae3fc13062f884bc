"""Disaggregated prefill between real vLLM engines of different tensor-parallel sizes: a tiny random-weight Llama with
4 KV heads, prefilled by a `kv_producer` at TP=--prefill-tp and decoded by a `kv_consumer` at TP=--decode-tp, both
with B200KVConnector, plus a reference engine without P/D.  The kv_transfer_params the producer returns are handed to
the consumer as the router does.  Prints one JSON line with both runs' greedy tokens and logprobs; the hand-off
events (tokens pulled, failed pulls) go to the file B200KV_PD_TRACE names.  Started as a subprocess by
tests/test_gpu_vllm_pd_hetero.py (never imported by the product).

    python tests/vllm_pd_hetero_driver.py --prefill-tp 1 --decode-tp 2 --out result.json
"""
from __future__ import annotations

import argparse
import json
import multiprocessing as mp
import os
import sys


def make_model(path: str, layers: int, vocab: int, seed: int = 0) -> None:
    """4 KV heads x 128, 8 query heads, real N(0, 0.02) weights, bf16."""
    import torch
    from transformers import LlamaConfig, LlamaForCausalLM
    torch.manual_seed(seed)
    cfg = LlamaConfig(hidden_size=1024, intermediate_size=2816, num_hidden_layers=layers, num_attention_heads=8,
                      num_key_value_heads=4, head_dim=128, vocab_size=vocab, max_position_embeddings=4096,
                      rms_norm_eps=1e-5, rope_theta=500000.0, tie_word_embeddings=False, bos_token_id=1,
                      eos_token_id=2, initializer_range=0.04, torch_dtype="bfloat16")
    LlamaForCausalLM(cfg).to(torch.bfloat16).save_pretrained(path, safe_serialization=True)


def prompts(vocab: int):
    import numpy as np
    rng = np.random.default_rng(1234)
    return [rng.integers(3, vocab, n).tolist() for n in (300, 700, 1029, 1536)]


def llm(a, tp: int, role: str | None, engine_id: str):
    from vllm import LLM
    from vllm.config import KVTransferConfig
    ktc = None if role is None else KVTransferConfig(
        kv_connector="B200KVConnector", kv_connector_module_path="b200kv.connector", kv_role=role,
        engine_id=engine_id, kv_load_failure_policy="recompute")
    return LLM(model=a.model_dir, skip_tokenizer_init=True, dtype="bfloat16", seed=0, max_model_len=4096,
               tensor_parallel_size=tp, gpu_memory_utilization=0.2, enable_prefix_caching=False, enforce_eager=True,
               kv_transfer_config=ktc)


def generate(engine, ps, max_tokens, params=None):
    from vllm import SamplingParams
    sps = [SamplingParams(temperature=0.0, max_tokens=max_tokens, logprobs=5, detokenize=False, ignore_eos=True,
                          extra_args=None if params is None else {"kv_transfer_params": params[i]})
           for i in range(len(ps))]
    outs = engine.generate([{"prompt_token_ids": p} for p in ps], sps, use_tqdm=False)
    res = []
    for o in outs:
        c = o.outputs[0]
        steps = []
        for t, step in zip(c.token_ids, c.logprobs or []):
            top = sorted((float(v.logprob) for v in step.values()), reverse=True)
            steps.append({"lp": float(step[t].logprob), "margin": top[0] - top[1] if len(top) > 1 else 99.0})
        res.append({"tokens": [int(t) for t in c.token_ids], "steps": steps,
                    "kv_transfer_params": getattr(o, "kv_transfer_params", None)})
    return res


def producer(a, q_params, q_done):
    """Prefill every prompt (one token) with do_remote_decode, hand the params over, keep the blocks until told."""
    eng = llm(a, a.prefill_tp, "kv_producer", "pd-hetero-P")
    ps = prompts(a.vocab)
    req = {"do_remote_decode": True, "do_remote_prefill": False, "remote_engine_id": None, "remote_block_ids": None,
           "remote_host": None, "remote_port": None}
    outs = generate(eng, ps, 1, [dict(req) for _ in ps])
    q_params.put([o["kv_transfer_params"] for o in outs])
    q_done.get(timeout=900)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prefill-tp", type=int, default=1)
    ap.add_argument("--decode-tp", type=int, default=2)
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--vocab", type=int, default=4096)
    ap.add_argument("--model-dir", default="/tmp/b200kv-tiny-llama-kv4")
    ap.add_argument("--max-tokens", type=int, default=12)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    if not os.path.exists(os.path.join(a.model_dir, "config.json")):
        make_model(a.model_dir, a.layers, a.vocab)
    ps = prompts(a.vocab)
    ctx = mp.get_context("spawn")
    q_params, q_done = ctx.Queue(), ctx.Queue()
    prod = ctx.Process(target=producer, args=(a, q_params, q_done))
    prod.start()
    try:
        params = q_params.get(timeout=900)
        if any(not p for p in params):
            raise RuntimeError(f"the producer returned no kv_transfer_params: {params}")
        for p in params:
            p["remote_host"] = "127.0.0.1"
        cons = llm(a, a.decode_tp, "kv_consumer", "pd-hetero-D")
        got = generate(cons, ps, a.max_tokens, params)
    finally:
        q_done.put(True)
        prod.join(120)
    del cons
    ref = generate(llm(a, a.decode_tp, None, "pd-hetero-ref"), ps, a.max_tokens)
    out = {"prefill_tp": a.prefill_tp, "decode_tp": a.decode_tp, "prompt_lens": [len(p) for p in ps],
           "first": ref, "second": got}
    line = json.dumps(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line)
    print("RESULT " + line, flush=True)


if __name__ == "__main__":
    sys.exit(main())
