"""Boot a real vLLM engine with speculative decoding and B200KVConnector, and run the same prompts twice, as
tests/vllm_mla_driver.py does without a drafter.  Two models, each a config.json with vLLM's dummy weights redrawn
(spread_weights, on the target and on the drafter, which apply_model does not reach):

* `deepseek-mtp`: a tiny DeepSeek-V3 (MLA) with num_nextn_predict_layers 1, served with {"method": "mtp"};
* `llama-eagle3`: a tiny Llama (Llama-3-8B's per-layer KV geometry) with a one-layer EAGLE-3 draft model.

vLLM puts the draft layer into the target's KV-cache group, so the connector registers L + 1 layers.  The connector is
SnapshotConnector below, loaded by module path: at the end of each request's prefill step (wait_for_save, which vLLM
defers until the drafter has run) it writes the draft layer's pages at the request's prompt slots to
$B200KV_TEST_SNAPSHOT_DIR.  Random weights make acceptance rates meaningless; comparing pass 2's draft pages with pass
1's shows that the draft KV arrived.  Prints one JSON line with both passes' greedy tokens and logprobs, and per prompt
the positions whose draft pages pass 2 has bit-identical to pass 1.  Started as a subprocess by
tests/test_gpu_vllm_spec_decode.py (never imported by the product)."""
from __future__ import annotations

import argparse
import hashlib
import json
import os
import sys
import time

from b200kv.connector import B200KVConnector


class SnapshotConnector(B200KVConnector):
    """B200KVConnector that also saves the first draft layer's pages of every request whose prefill ends in a step."""

    def register_kv_caches(self, kv_caches):
        super().register_kv_caches(kv_caches)
        draft = [n for n, i in self._layer_index.items() if i == self._n_target]
        self._draft_cache = kv_caches[draft[0]] if draft else None

    def wait_for_save(self):
        super().wait_for_save()
        out = os.environ.get("B200KV_TEST_SNAPSHOT_DIR")
        t = getattr(self, "_draft_cache", None)
        if not out or t is None or self._worker is None:
            return
        for m in self._metas():
            if not m.is_last_prefill or not len(m.token_ids):
                continue
            sm = m.slot_mapping(self._block_size)
            import numpy as np
            import torch
            slots = torch.from_numpy(np.asarray(sm, dtype=np.int64)).to(t.device)
            if t.dim() == 3:                                       # MLA (NB, bs, D)
                pages = t.reshape(-1, t.shape[-1])[slots]
            else:                                                  # (2, NB, bs, H, D) or (NB, 2, bs, H, D)
                kv = t if t.shape[0] == 2 else t.transpose(0, 1)
                pages = kv.reshape(2, -1, kv.shape[-2] * kv.shape[-1])[:, slots]
            host = pages.contiguous().view(torch.uint8).cpu().numpy()
            key = hashlib.sha1(np.asarray(m.token_ids, dtype=np.int32).tobytes()).hexdigest()[:16]
            n = 1 if not os.path.exists(os.path.join(out, f"{key}.1.npy")) else 2
            np.save(os.path.join(out, f"{key}.{n}.npy"), host)


def make_configs(model: str, path: str, layers: int, vocab: int) -> str | None:
    """config.json of the target (and of the EAGLE-3 draft model); -> the draft model's directory or None."""
    os.makedirs(path, exist_ok=True)
    if model == "deepseek-mtp":
        cfg = {"architectures": ["DeepseekV3ForCausalLM"], "model_type": "deepseek_v3", "vocab_size": vocab,
               "hidden_size": 1024, "intermediate_size": 2816, "moe_intermediate_size": 256,
               "num_hidden_layers": layers, "num_attention_heads": 16, "num_key_value_heads": 16, "kv_lora_rank": 512,
               "q_lora_rank": 384, "qk_rope_head_dim": 64, "qk_nope_head_dim": 128, "v_head_dim": 128,
               "first_k_dense_replace": layers + 1, "n_routed_experts": 4, "num_experts_per_tok": 2,
               "n_shared_experts": 1, "n_group": 1, "topk_group": 1, "routed_scaling_factor": 1.0,
               "norm_topk_prob": True, "scoring_func": "sigmoid", "topk_method": "noaux_tc",
               "max_position_embeddings": 4096, "rms_norm_eps": 1e-6, "rope_theta": 10000.0,
               "tie_word_embeddings": False, "bos_token_id": 1, "eos_token_id": 2, "initializer_range": 0.02,
               "torch_dtype": "bfloat16", "hidden_act": "silu", "num_nextn_predict_layers": 1}
        draft = None
    else:
        base = {"model_type": "llama", "hidden_size": 1024, "intermediate_size": 2816, "num_attention_heads": 8,
                "num_key_value_heads": 8, "head_dim": 128, "vocab_size": vocab, "max_position_embeddings": 4096,
                "rms_norm_eps": 1e-5, "rope_theta": 500000.0, "tie_word_embeddings": False, "bos_token_id": 1,
                "eos_token_id": 2, "torch_dtype": "bfloat16", "hidden_act": "silu"}
        cfg = {**base, "architectures": ["LlamaForCausalLM"], "num_hidden_layers": layers}
        draft = path + "-eagle3"
        os.makedirs(draft, exist_ok=True)
        with open(os.path.join(draft, "config.json"), "w") as f:
            # three target layers feed the drafter (vLLM's default picks (2, L/2, L-3), two distinct ones at L = 4)
            json.dump({**base, "architectures": ["LlamaForCausalLMEagle3"], "num_hidden_layers": 1,
                       "draft_vocab_size": vocab, "eagle_aux_hidden_state_layer_ids": [1, 2, 3]}, f)
    with open(os.path.join(path, "config.json"), "w") as f:
        json.dump(cfg, f)
    return draft


def spread_weights(model) -> int:
    """vLLM's dummy weights (uniform +-1e-3, norms included) give near-uniform logits, so pass 1 and pass 2 would
    agree whatever attention read.  Redraw them: norms 1, every other floating weight N(0, 0.05), seeded."""
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


def spread_drafter(worker) -> int:
    return spread_weights(worker.model_runner.drafter.model)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", choices=["deepseek-mtp", "llama-eagle3"], required=True)
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--vocab", type=int, default=4096)
    ap.add_argument("--max-tokens", type=int, default=12)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    model_dir = f"/tmp/b200kv-spec-{a.model}-{os.getpid()}"
    draft = make_configs(a.model, model_dir, a.layers, a.vocab)

    os.environ.setdefault("VLLM_ALLOW_INSECURE_SERIALIZATION", "1")   # apply_model / collective_rpc ship functions
    import numpy as np
    from vllm import LLM, SamplingParams
    from vllm.config import KVTransferConfig

    spec = {"method": "mtp", "num_speculative_tokens": 1} if draft is None else \
        {"method": "eagle3", "model": draft, "num_speculative_tokens": 1}
    ktc = KVTransferConfig(kv_connector="SnapshotConnector", kv_connector_module_path="tests.vllm_spec_decode_driver",
                           kv_role="kv_both", kv_load_failure_policy="recompute")
    llm = LLM(model=model_dir, skip_tokenizer_init=True, dtype="bfloat16", seed=0, max_model_len=4096,
              gpu_memory_utilization=0.25, enable_prefix_caching=False, enforce_eager=True, load_format="dummy",
              kv_transfer_config=ktc, speculative_config=spec)
    llm.apply_model(spread_weights)
    llm.collective_rpc(spread_drafter)
    backend, block_size = None, None
    try:
        vc = llm.llm_engine.vllm_config
        block_size = vc.cache_config.block_size
        backend = str(getattr(vc.attention_config, "backend", None))
    except Exception as e:
        backend = f"unknown ({e!r})"

    rng = np.random.default_rng(4321)
    prompts = [rng.integers(3, a.vocab, n).tolist() for n in (300, 700, 1029, 1536, 2100, 2817)]
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
    # draft pages: pass 2 loaded positions [0, n-1) (n-1 is recomputed, with the right next token)
    snap = os.environ.get("B200KV_TEST_SNAPSHOT_DIR", "")
    draft_pages = []
    for p in prompts:
        key = hashlib.sha1(np.asarray(p, dtype=np.int32).tobytes()).hexdigest()[:16]
        files = [os.path.join(snap, f"{key}.{i}.npy") for i in (1, 2)]
        if not snap or not all(os.path.exists(f) for f in files):
            draft_pages.append(None)
            continue
        p1, p2 = (np.load(f) for f in files)
        tok_axis = 0 if p1.ndim == 2 else 1              # MLA (n, bytes) or K/V (2, n, bytes)
        n = p1.shape[tok_axis]
        same = np.all((p1 == p2).reshape(p1.shape[:tok_axis + 1] + (-1,)), axis=-1)
        same = same if tok_axis == 0 else same.all(axis=0)
        draft_pages.append({"n": int(n), "same_prefix": int(np.argmin(same)) if not same.all() else int(n),
                            "nonzero": bool(np.any(p1[..., :] != 0))})
    out = {"model": a.model, "format": os.environ.get("B200KV_FORMAT", "raw"),
           "layerwise": os.environ.get("B200KV_LAYERWISE", "0"), "prompt_lens": [len(p) for p in prompts],
           "backend": backend, "block_size": block_size, "first": first, "second": second, "draft_pages": draft_pages}
    line = json.dumps(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line)
    print("RESULT " + line, flush=True)


if __name__ == "__main__":
    sys.exit(main())
