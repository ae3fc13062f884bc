"""The local-disk tier under a REAL vLLM engine (tests/vllm_disk_driver.py): a tiny Llama, prompts run one at a time,
a pinned pool smaller than one pass's chunks, so pass 2 can only hit from disk.  Pass 2 must read chunks from disk,
hit (all but the recomputed last token of) every prompt, and produce the tokens of pass 1 with logprobs within the RAW
tolerance of tests/test_gpu_vllm_connector.py.  Then a fresh vLLM process, with a fresh pool and no disk index in shm,
runs the prompts once on the same directory: the warm restart, with the same checks against the first process's
pass 1."""
import json
import os
import subprocess
import sys

import pytest

from tests.test_gpu_vllm_connector import RAW_LOGPROB_TOL, _compare

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(ROOT, "production-stack_b200")
DRIVER = os.path.join(ROOT, "tests", "vllm_disk_driver.py")
CHUNK = 4 * 2 * 256 * 8 * 128 * 2          # the driver's model: 4 layers of Llama-3-8B's KV geometry, RAW


def _run(tmp_path, directory, pool, passes, tag):
    env = dict(os.environ)
    env["PYTHONPATH"] = os.pathsep.join([PKG, env.get("PYTHONPATH", "")])
    env.update(LMCACHE_LOCAL_CPU="True", LMCACHE_MAX_LOCAL_CPU_SIZE=str(20 * CHUNK / (1 << 30)),   # 20 chunk slots
               LMCACHE_CHUNK_SIZE="256", B200KV_FORMAT="raw", B200KV_POOL_NAME=pool, B200KV_STAGING_MB="512",
               LMCACHE_LOCAL_DISK=f"file://{directory}/", LMCACHE_MAX_LOCAL_DISK_SIZE="1",
               B200KV_LOOKUP_LEASE_MS="500", VLLM_ENABLE_V1_MULTIPROCESSING="0", VLLM_LOGGING_LEVEL="WARNING",
               CUDA_VISIBLE_DEVICES=os.environ.get("CUDA_VISIBLE_DEVICES", "0").split(",")[0])
    out_file = str(tmp_path / f"{tag}.json")
    p = subprocess.run([sys.executable, DRIVER, "--passes", str(passes), "--out", out_file], env=env,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0 and os.path.exists(out_file), \
        f"vLLM driver failed (rc={p.returncode})\n--- stdout\n{p.stdout[-3000:]}\n--- stderr\n{p.stderr[-6000:]}"
    return json.load(open(out_file))


def _check_disk_hits(res, what):
    lens = res["prompt_lens"]
    n_chunks = sum((n + 255) // 256 for n in lens) - 2 * 2           # the shared 2-chunk prefix is stored once
    assert n_chunks > res["pool_slots"], (n_chunks, res["pool_slots"])   # the pool cannot hold a pass
    assert res["fetched_last_pass"] > 0 and res["disk"]["corrupt_chunks"] == 0, (what, res["disk"])
    # the pass found (all but the recomputed last token of) every prompt: the pool's own hit counter
    assert res["hit_tokens_last_pass"] >= 0.95 * sum(lens), (what, res["hit_tokens_last_pass"], sum(lens))


@pytest.mark.gpu
def test_vllm_pass2_and_a_restarted_process_hit_from_disk(tmp_path):
    pytest.importorskip("vllm")
    from b200kv import KVPool
    from b200kv.disk import index_name
    directory = str(tmp_path / "disk")
    os.mkdir(directory)
    pools = [f"/b200kv-vllmdisk-{os.getpid()}-{i}" for i in (1, 2)]
    try:
        res = _run(tmp_path, directory, pools[0], 2, "first")
        assert res["on_disk"] >= sum((n + 255) // 256 for n in res["prompt_lens"]) - 2 * 2, res["on_disk"]
        _check_disk_hits(res, "pass 2")
        first = {"first": res["passes"][0], "second": res["passes"][1]}
        same, worst = _compare(first, 12, RAW_LOGPROB_TOL)
        print(f"disk pass 2: {same}/6 identical, max |dlogprob| {worst:.5f}, fetched {res['fetched_last_pass']}")
        assert same == 6 and worst <= RAW_LOGPROB_TOL

        KVPool.unlink(index_name(directory, CHUNK))                 # a restarted box: no index in shm
        again = _run(tmp_path, directory, pools[1], 1, "restart")
        assert again["at_start"] >= res["on_disk"], (again["at_start"], res["on_disk"])    # rebuilt from the file
        _check_disk_hits(again, "restart")
        same, worst = _compare({"first": res["passes"][0], "second": again["passes"][0]}, 12, RAW_LOGPROB_TOL)
        print(f"disk restart: {same}/6 identical, max |dlogprob| {worst:.5f}, fetched {again['fetched_last_pass']}")
        assert same == 6 and worst <= RAW_LOGPROB_TOL
    finally:
        import glob
        for pool in pools:
            for f in glob.glob("/dev/shm" + pool + "*"):
                KVPool.unlink("/" + os.path.basename(f))
        if os.path.exists(os.path.join(directory, f"b200kv-disk-{CHUNK:x}.slots")):
            KVPool.unlink(index_name(directory, CHUNK))
