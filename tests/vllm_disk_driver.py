"""Boot a real vLLM engine (tiny Llama with real random weights, tests/vllm_inproc_driver.py's model) with
B200KVConnector and the local-disk tier, whose pinned pool is smaller than one pass's chunks, and run prompts one at a
time: with --passes 2 the first pass stores (and writes through to disk) and the second can only hit from disk; with
--passes 1 (a fresh process on the same directory: the warm restart) the only pass hits from disk.  The engine core
runs in this process, so the scheduler's disk tier is read directly.  Writes one JSON line with each pass's greedy
tokens and logprobs and the disk tier's counters.  Started as a subprocess by tests/test_gpu_vllm_disk.py (never
imported by the product)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from vllm_inproc_driver import make_model  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--passes", type=int, default=2)
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--vocab", type=int, default=4096)
    ap.add_argument("--model-dir", default="/tmp/b200kv-tiny-llama")
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
    llm = LLM(model=a.model_dir, skip_tokenizer_init=True, dtype="bfloat16", seed=0, max_model_len=4096,
              gpu_memory_utilization=0.25, enable_prefix_caching=False, enforce_eager=True, kv_transfer_config=ktc)
    conn = llm.llm_engine.engine_core.engine_core.scheduler.connector
    disk = conn._disk
    assert disk is not None, "the scheduler has no disk tier"
    at_start = disk.file.stats()["n_used"]      # what the first opener (the worker) found in the file

    rng = np.random.default_rng(1234)
    shared = rng.integers(3, a.vocab, 512).tolist()
    prompts = []
    for i, n in enumerate((300, 700, 1029, 1536, 2100, 2817)):
        body = rng.integers(3, a.vocab, n).tolist()
        prompts.append((shared + body) if i % 2 else body)       # odd ones share a 512-token (2-chunk) prefix
    sp = SamplingParams(temperature=0.0, max_tokens=a.max_tokens, logprobs=5, detokenize=False, ignore_eos=True)
    lease_s = int(os.environ.get("B200KV_LOOKUP_LEASE_MS", "30000")) / 1e3

    def run():
        res = []
        for p in prompts:        # one at a time: each prompt's chunks fit the small pool, all of a pass's do not
            o = llm.generate([{"prompt_token_ids": p}], sp, use_tqdm=False)[0]
            c = o.outputs[0]
            steps = []
            for t, step in zip(c.token_ids, c.logprobs or []):
                top = sorted((float(v.logprob) for v in step.values()), reverse=True)
                steps.append({"lp": float(step[t].logprob), "margin": top[0] - top[1] if len(top) > 1 else 99.0})
            res.append({"tokens": [int(t) for t in c.token_ids], "steps": steps,
                        "num_cached_tokens": getattr(o, "num_cached_tokens", None)})
            time.sleep(lease_s + 0.1)    # the lookup's lease on this prompt's chunks runs out: the pool may evict them
        return res

    def settle():
        """Until the write-through has drained: the index stops growing."""
        last, t0 = -1, time.time()
        while time.time() - t0 < 60:
            n = disk.file.stats()["n_used"]
            if n == last:
                return n
            last = n
            time.sleep(1.0)
        return last

    passes, fetched0, hits0 = [], 0, 0
    for i in range(a.passes):
        if i == a.passes - 1:
            fetched0, hits0 = disk.stats()["fetched_chunks"], conn._pool.stats()["n_hit_tokens"]
        passes.append(run())
        if i == 0:
            on_disk = settle()
    st = disk.stats()
    out = {"prompt_lens": [len(p) for p in prompts], "passes": passes, "on_disk": on_disk, "at_start": at_start,
           "fetched_last_pass": st["fetched_chunks"] - fetched0,
           "hit_tokens_last_pass": conn._pool.stats()["n_hit_tokens"] - hits0, "disk": st,
           "pool_slots": conn._pool.stats()["n_slots"]}
    line = json.dumps(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line)
    print("RESULT " + line, flush=True)


if __name__ == "__main__":
    sys.exit(main())
