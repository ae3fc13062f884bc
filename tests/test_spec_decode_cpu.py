"""Speculative decoding (MTP, EAGLE, EAGLE-3) on CPU: vLLM puts the drafter's attention layers into the target's
KV-cache group, so the connector moves L + D layers, the draft layers L..L+D-1 after the target's.

* geometry_from_vllm counts D from the speculative config; chunk sizes at C = 256 with one draft layer;
* a geometry without draft layers keeps its key seed bit for bit;
* register_kv_caches orders the caches by layer index and refuses a wrong draft count or non-contiguous indices;
* the last target layer's hook waits for every group holding a draft layer;
* the hit rule: one token less is reported, all hit tokens are loaded, and no loaded slot lies outside the blocks
  vLLM allocated; with D = 0 every decision is today's;
* the P/D document carries draft_layers; the lm:// tier moves a draft geometry's chunks like any other."""
import os
import random
from types import SimpleNamespace as NS

import numpy as np
import pytest

from b200kv import KVPool, _lib
from b200kv.adapter import SchedulerState
from b200kv.engine import DEFAULT_SEED, KVGeometry, chunk_keys, xxh64
from tests.test_mla_sparse_cpu import _RecordingWorker, _StubEngine

C = 256
V3 = dict(n_layers=61, n_kv_heads=1, head_dim=576, n_blocks=1, block_tokens=64, chunk_tokens=C, elem_bytes=2,
          layout=_lib.LAYOUT_MLA)


# ---------------------------------------------------------------------------------------------------------------
# geometry_from_vllm
# ---------------------------------------------------------------------------------------------------------------
def _vllm_config(model="deepseek-v3", spec=None, pp=1, sparse=False):
    import torch
    from vllm.config import KVTransferConfig
    ktc = KVTransferConfig(kv_connector="B200KVConnector", kv_connector_module_path="b200kv.connector",
                           kv_role="kv_both", engine_id="spec", kv_connector_extra_config={})
    if model.startswith("deepseek"):
        hf = NS(num_nextn_predict_layers=1, **(dict(index_topk=2048) if sparse else {}))
        mc = NS(model=model, dtype=torch.bfloat16, use_mla=True, get_num_layers=lambda pc: 61,
                get_num_kv_heads=lambda pc: 1, get_head_size=lambda: 576, hf_config=hf, hf_text_config=hf)
        bs = 64
    else:    # Llama-3-8B
        hf = NS()
        mc = NS(model=model, dtype=torch.bfloat16, use_mla=False, get_num_layers=lambda pc: 32,
                get_num_kv_heads=lambda pc: 8, get_head_size=lambda: 128, hf_config=hf, hf_text_config=hf)
        bs = 16
    return NS(kv_transfer_config=ktc, model_config=mc, speculative_config=spec,
              parallel_config=NS(tensor_parallel_size=1, pipeline_parallel_size=pp, rank=0),
              cache_config=NS(block_size=bs, cache_dtype="auto"))


MTP = NS(method="mtp", draft_model_config=NS(hf_config=NS(n_predict=1)), num_speculative_tokens=1)
EAGLE3 = NS(method="eagle3", draft_model_config=NS(hf_config=NS(num_hidden_layers=1)), num_speculative_tokens=3)


def _cfg(fmt=_lib.FMT_RAW):
    from b200kv.config import B200KVConfig
    cfg = B200KVConfig()
    cfg.fmt, cfg.chunk_size = fmt, C
    return cfg


@pytest.mark.parametrize("model,spec,sparse,fmt,want", [
    ("deepseek-v3", MTP, False, _lib.FMT_RAW, 18_284_544),
    ("deepseek-v3", MTP, False, _lib.FMT_FP8, 10_412_032),
    ("deepseek-v3.2", MTP, True, _lib.FMT_RAW, 20_379_648),
    ("llama-3-8b", EAGLE3, False, _lib.FMT_RAW, 34_603_008)])
def test_geometry_counts_the_draft_layers(model, spec, sparse, fmt, want):
    pytest.importorskip("vllm")
    from b200kv.connector import geometry_from_vllm
    L = 61 if model.startswith("deepseek") else 32
    g = geometry_from_vllm(_vllm_config(model, spec, sparse=sparse), _cfg(fmt))
    assert (g.n_layers, g.draft_layers, g.target_layers) == (L + 1, 1, L)
    assert g.indexed == sparse and g.chunk_bytes == want
    assert g.n_descs == (2 * (L + 1) if (sparse or not g.mla) else L + 1)
    plain = geometry_from_vllm(_vllm_config(model, None, sparse=sparse), _cfg(fmt))
    assert g.key_seed(model) != plain.key_seed(model)      # a replica with a drafter has its own namespace


@pytest.mark.parametrize("spec", [
    None,
    NS(method="ngram", draft_model_config=None, num_speculative_tokens=4),
    NS(method="suffix", draft_model_config=None, num_speculative_tokens=4),
    NS(method="draft_model", draft_model_config=NS(hf_config=NS(num_hidden_layers=2)), num_speculative_tokens=4),
    NS(method="medusa", draft_model_config=NS(hf_config=NS(num_hidden_layers=0)), num_speculative_tokens=4)])
def test_methods_without_draft_attention_leave_the_geometry_and_its_seed_unchanged(spec):
    pytest.importorskip("vllm")
    from b200kv.connector import geometry_from_vllm
    for model in ("deepseek-v3", "llama-3-8b"):
        vc = _vllm_config(model, spec)
        if spec is None:
            del vc.speculative_config          # configs of older vLLM builds have no such attribute at all
        g = geometry_from_vllm(vc, _cfg())
        assert g.draft_layers == 0 and g.n_layers == (61 if model == "deepseek-v3" else 32)
        # the seed as it was written before draft layers existed
        tag = (f"{model}|1|0|{g.n_layers}|{g.n_kv_heads}|{g.head_dim}|{g.elem_bytes}|{C}|{g.fmt}|{g.layout}")
        assert g.key_seed(model, 1, 0) == xxh64(tag.encode(), DEFAULT_SEED)


def test_key_seed_of_geometries_without_draft_layers_is_pinned():
    """The seeds of MLA, K/V, indexed and fp16 geometries as the code computed them before draft layers existed:
    chunks stored by a replica without a drafter stay reachable across the upgrade."""
    got = {"v3": KVGeometry(**V3).key_seed("deepseek-v3", 8, 3),
           "llama": KVGeometry(32, 8, 128, 1, 16, C).key_seed("llama", 2, 1),
           "v32": KVGeometry(**V3, idx_value_bytes=128, idx_scale_bytes=4).key_seed("deepseek-v3.2", 1, 0),
           "fp16": KVGeometry(32, 8, 128, 1, 16, C, dtype=_lib.DTYPE_FP16).key_seed("llama", 1, 0)}
    assert got == {"v3": 0xA59326E8282EE3E7, "llama": 0x61D9AB30456D5B91, "v32": 0xAC739E0CF39E7860,
                   "fp16": 0x2AAB04B86CC027D8}, {k: hex(v) for k, v in got.items()}


def test_mtp_layer_count_also_read_from_the_target_config():
    pytest.importorskip("vllm")
    from b200kv.connector import draft_layers_of
    vc = _vllm_config("deepseek-v3", NS(method="mtp", draft_model_config=NS(hf_config=NS())))
    vc.model_config.hf_text_config.num_nextn_predict_layers = 2
    assert draft_layers_of(vc) == 2
    vc.speculative_config = NS(method="deepseek_mtp", draft_model_config=NS(hf_config=NS(n_predict=1)))
    assert draft_layers_of(vc) == 1                              # an alias vLLM has not folded into "mtp"
    vc.speculative_config = NS(method="eagle", draft_model_config=NS(hf_config=NS(num_hidden_layers=1)))
    assert draft_layers_of(vc) == 1


def test_pipeline_parallelism_with_a_drafter_is_refused():
    pytest.importorskip("vllm")
    from b200kv.connector import geometry_from_vllm
    with pytest.raises(ValueError, match="pipeline parallelism"):
        geometry_from_vllm(_vllm_config("deepseek-v3", MTP, pp=2), _cfg())
    assert geometry_from_vllm(_vllm_config("deepseek-v3", None, pp=2), _cfg()).draft_layers == 0


def test_geometry_refuses_more_draft_layers_than_layers():
    with pytest.raises(ValueError):
        KVGeometry(**{**V3, "n_layers": 1}, draft_layers=1)
    with pytest.raises(ValueError):
        KVGeometry(**V3, draft_layers=-1)


# ---------------------------------------------------------------------------------------------------------------
# registration order and the layer hooks
# ---------------------------------------------------------------------------------------------------------------
def _worker(monkeypatch, L, G, spec=MTP, sparse=False, mla=True, names=None, shuffle=0):
    """A worker-role connector on a stand-in engine, with vLLM-named caches for L target layers and the draft
    layers `names` gives (default: L..L+D-1), in a shuffled dict order."""
    import torch
    from vllm.distributed.kv_transfer.kv_connector.v1.base import KVConnectorRole
    import b200kv.connector as bc
    monkeypatch.setattr(bc, "KVEngine", _StubEngine)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: None)
    monkeypatch.setenv("LMCACHE_MAX_LOCAL_CPU_SIZE", "0.01")
    monkeypatch.setenv("LMCACHE_CHUNK_SIZE", "64")
    monkeypatch.setenv("B200KV_LAYERWISE", "1")
    monkeypatch.setenv("B200KV_LAYER_GROUP", str(G))
    vc = _vllm_config("deepseek-v3" if mla else "llama", spec, sparse=sparse)
    vc.model_config.get_num_layers = lambda pc: L
    vc.cache_config.block_size = 16
    vc.scheduler_config = NS(disable_hybrid_kv_cache_manager=False)
    vc.kv_transfer_config.engine_id = f"spec-{os.getpid()}-{os.urandom(3).hex()}"
    w = bc.B200KVConnector(vc, KVConnectorRole.WORKER, None)
    D = bc.draft_layers_of(vc)
    layers = list(range(L)) + (list(range(L, L + D)) if names is None else names)
    items = []
    for l in layers:
        if mla:
            items.append((f"model.layers.{l}.self_attn.attn", torch.zeros((4, 16, 576), dtype=torch.bfloat16)))
        else:
            items.append((f"model.layers.{l}.self_attn.attn", torch.zeros((2, 4, 16, 8, 128), dtype=torch.bfloat16)))
        if sparse:
            items.append((f"model.layers.{l}.self_attn.indexer.k_cache", torch.zeros((4, 16, 132), dtype=torch.uint8)))
    if shuffle:
        random.Random(shuffle).shuffle(items)
    try:
        w.register_kv_caches(dict(items))
    except Exception:
        w.shutdown()
        raise
    return w, bc, dict(items)


@pytest.mark.parametrize("sparse", [False, True], ids=["mla", "v32"])
@pytest.mark.parametrize("seed", [1, 2, 3])
def test_registration_orders_caches_by_layer_index(monkeypatch, sparse, seed):
    pytest.importorskip("vllm")
    L = 5
    w, bc, caches = _worker(monkeypatch, L, 2, sparse=sparse, shuffle=seed)
    try:
        assert list(caches) != sorted(caches, key=bc._layer_index_of)       # the dict really is shuffled
        got = w._engine.kv_caches
        got = list(got.values()) if isinstance(got, dict) else list(got)
        lat = [caches[f"model.layers.{l}.self_attn.attn"] for l in range(L + 1)]
        want = lat + ([caches[f"model.layers.{l}.self_attn.indexer.k_cache"] for l in range(L + 1)] if sparse else [])
        if sparse:     # the engine gets the dict; split_indexer_caches separates the kinds, each in layer order
            from b200kv.engine import split_indexer_caches
            a, b = split_indexer_caches(w._engine.kv_caches)
            got = a + b
        assert len(got) == len(want) and all(x is y for x, y in zip(got, want))
        assert w._layer_index == {f"model.layers.{l}.self_attn.attn": l for l in range(L + 1)}
        assert (w._engine.geom.n_layers, w._engine.geom.draft_layers) == (L + 1, 1)
    finally:
        w.shutdown()


@pytest.mark.parametrize("names,why", [([], "0 at or above"), ([5, 6], "2 at or above"), ([6], r"\[6\]")],
                         ids=["missing", "two", "gap"])
def test_registration_refuses_a_wrong_draft_count_or_indices(monkeypatch, names, why):
    pytest.importorskip("vllm")
    with pytest.raises(ValueError, match=f"1 draft layer.*{why}"):
        _worker(monkeypatch, 5, 2, names=names)


def test_registration_refuses_non_contiguous_draft_indices(monkeypatch):
    pytest.importorskip("vllm")
    two = NS(method="mtp", draft_model_config=NS(hf_config=NS(n_predict=2)))
    with pytest.raises(ValueError, match=r"2 draft layer.*\[5, 7\]"):
        _worker(monkeypatch, 5, 2, spec=two, names=[5, 7])


def _run_step(w, bc, L, D, sparse, draft_hooks):
    """vLLM's order in one step: per target layer (the indexer first on V3.2) its attention with its hook, then the
    drafter's layers right after the last target layer, their hooks called or not (CUDA-graph replay)."""
    log = []
    w._worker = _RecordingWorker(log)
    w.bind_connector_metadata(bc.B200KVConnectorMetadata())
    w.start_load_kv(NS(cudagraph_runtime_mode=NS(name="NONE")))
    for l in range(L + D):
        if sparse:
            log.append(("indexer reads", l))
        if l < L or draft_hooks:
            w.wait_for_layer_load(f"model.layers.{l}.self_attn.attn")
        log.append(("attention", l))
    return log


@pytest.mark.parametrize("draft_hooks", [True, False], ids=["hooks", "no-draft-hooks"])
@pytest.mark.parametrize("sparse", [False, True], ids=["plain", "wait-ahead"])
@pytest.mark.parametrize("L,D,G", [(4, 1, 1), (4, 1, 2), (4, 1, 3), (4, 1, 4), (5, 1, 2), (3, 2, 1), (3, 2, 2),
                                   (3, 2, 4), (6, 3, 2)])
def test_last_target_hook_waits_for_the_draft_groups(monkeypatch, L, D, G, sparse, draft_hooks):
    pytest.importorskip("vllm")
    spec = NS(method="mtp", draft_model_config=NS(hf_config=NS(n_predict=D)))
    w, bc, _ = _worker(monkeypatch, L, G, spec=spec, sparse=sparse)
    try:
        log = _run_step(w, bc, L, D, sparse, draft_hooks)
        for l in range(L + D):
            for what in (("indexer reads", "attention") if sparse else ("attention",)):
                at = log.index((what, l))
                assert ("wait", l // G) in log[:at], (L, D, G, l, what, log)
        # every draft group is waited for by the last target layer's hook, before its attention runs
        last = log.index(("attention", L - 1))
        for l in range(L, L + D):
            assert ("wait", l // G) in log[:last]
        # a draft layer's own hook adds nothing; every group is waited for (once, unless the wait-ahead rule repeats
        # a target group's wait as it always has)
        waits = [e for e in log if e[0] == "wait"]
        assert sorted(set(waits)) == [("wait", g) for g in range((L + D + G - 1) // G)]
        assert sparse or len(waits) == len(set(waits))
        assert all(waits.count(("wait", l // G)) == 1 for l in range(L, L + D) if l % G == 0)
        assert all(e[0] != "wait" for e in log[last:])
        assert w._layer_hooks_seen == L
    finally:
        w._worker = None
        w.shutdown()


def test_without_a_drafter_hooks_are_unchanged(monkeypatch):
    pytest.importorskip("vllm")
    w, bc, _ = _worker(monkeypatch, 4, 2, spec=None)
    try:
        log = _run_step(w, bc, 4, 0, False, True)
        assert [e for e in log if e[0] != "attention"] == [("load", 2), ("wait", 0), ("wait", 1)]
    finally:
        w._worker = None
        w.shutdown()


# ---------------------------------------------------------------------------------------------------------------
# the hit rule
# ---------------------------------------------------------------------------------------------------------------
def _today(hit, nc, num_tokens, async_load):
    """The rule without draft layers, as it stood before they were added."""
    need = hit - nc
    if hit == num_tokens and not async_load:
        need -= 1
    return max(need, 0)


def _schedule(hit, nc, num_tokens, async_load, bs, D):
    """One request through SchedulerState as vLLM 0.22's scheduler drives it.  -> (reported, tokens loaded, slots
    allocated).  vLLM allocates blocks for nc + reported tokens on a detached load, and for at least one more token
    to compute otherwise (a prefill chunk of one token: the fewest blocks a synchronous load can get)."""
    prompt = list(range(1000, 1000 + num_tokens))
    st = SchedulerState(lambda toks: hit, bs, C, False, async_load=async_load, draft_layers=D)
    req = NS(request_id="r", prompt_token_ids=prompt, num_tokens=num_tokens)
    reported = st.num_new_matched_tokens("r", prompt, num_tokens, nc)
    detached = async_load and reported > 0
    n_alloc = nc + reported + (0 if detached else 1)
    blocks = list(range(100, 100 + -(-n_alloc // bs)))
    st.after_alloc(req, reported, (blocks,))
    if detached:
        metas = st.build_meta(NS(scheduled_new_reqs=[], scheduled_cached_reqs=NS(req_ids=[]),
                                 num_scheduled_tokens={}, finished_req_ids=set()))
    else:
        new = NS(req_id="r", prompt_token_ids=prompt, block_ids=(blocks,), num_computed_tokens=nc + reported)
        metas = st.build_meta(NS(scheduled_new_reqs=[new], scheduled_cached_reqs=NS(req_ids=[]),
                                 num_scheduled_tokens={"r": 1}, finished_req_ids=set()))
    loaded, slots = 0, len(blocks) * bs
    for m in metas:      # what WorkerState.start_load loads
        spec = m.load_spec
        if spec is not None and spec.can_load:
            loaded = min(spec.external_cached_tokens, len(m.token_ids))
            assert len(m.slot_mapping(bs)[:loaded]) == loaded      # every loaded token has a slot it owns
    return reported, loaded, slots


# (hit, num_computed, num_tokens, async, bs) -> (reported, loaded) with one draft layer, C = 256
TABLE = [
    ((512, 0, 600, False, 16), (511, 512)),
    ((512, 0, 512, False, 16), (511, 512)),     # full-prompt hit: subtracted once
    ((512, 0, 512, True, 16), (511, 512)),      # async full hit: the connector subtracts, vLLM does not again
    ((512, 0, 900, True, 16), (511, 512)),      # whole-chunk hit: hit-1 shares a block with hit-2
    ((529, 0, 529, False, 16), (528, 529)),     # partial chunk, synchronous: blocks cover hit-1
    ((529, 0, 529, True, 16), (511, 512)),      # partial chunk with hit = 1 (mod bs), async: trimmed to 512
    ((530, 0, 530, True, 16), (529, 530)),
    ((577, 0, 577, True, 64), (511, 512)),
    ((578, 0, 600, True, 64), (577, 578)),
    ((17, 0, 17, True, 16), (0, 0)),            # trimmed to nothing
    ((17, 0, 17, False, 16), (16, 17)),
    ((512, 256, 600, False, 16), (255, 512)),   # from vLLM's own prefix hit on
    ((512, 256, 600, True, 16), (255, 512)),
    ((257, 256, 300, False, 16), (0, 0)),       # nothing left to report: no load
    ((256, 256, 600, False, 16), (0, 0)),
    ((1, 0, 1, False, 16), (0, 0)),
    ((0, 0, 600, True, 16), (0, 0)),
]


@pytest.mark.parametrize("case,want", TABLE)
def test_hit_rule_table(case, want):
    hit, nc, n, async_load, bs = case
    reported, loaded, slots = _schedule(hit, nc, n, async_load, bs, D=1)
    assert (reported, loaded) == want
    assert loaded <= slots
    if reported:
        assert loaded == nc + reported + 1          # position hit-1 is loaded, and then recomputed


def _grid():
    for bs in (16, 64):
        for n in (1, 17, 255, 256, 257, 511, 512, 529, 577, 600, 768):
            for hit in sorted({0, 1, 16, 17, 256, 257, 511, 512, 513, 528, 529, 577, 578, 768} & set(range(n + 1))):
                for nc in sorted({0, 16, 64, 256, 512} & set(range(n))):
                    for a in (False, True):
                        yield hit, nc, n, a, bs


def test_hit_rule_invariants_over_a_grid():
    n_cases = 0
    for hit, nc, n, a, bs in _grid():
        r1, l1, s1 = _schedule(hit, nc, n, a, bs, D=1)
        r0, l0, s0 = _schedule(hit, nc, n, a, bs, D=0)
        assert l1 <= s1 and l0 <= s0, (hit, nc, n, a, bs)
        assert r0 == _today(hit, nc, n, a), (hit, nc, n, a, bs)       # D = 0: today's decision
        if r1:
            assert l1 == nc + r1 + 1 <= hit                            # all of the (maybe trimmed) hit is loaded
            assert l1 == hit or (a and (hit - 1) % bs == 0 and l1 % C == 0)
        assert r1 <= max(hit - nc - 1, 0)
        n_cases += 1
    assert n_cases > 500


def test_without_draft_layers_loads_are_todays():
    """D = 0 against the rule as it stood: reported tokens, and the tokens the worker loads."""
    for hit, nc, n, a, bs in _grid():
        r, loaded, _ = _schedule(hit, nc, n, a, bs, D=0)
        assert r == _today(hit, nc, n, a)
        assert loaded == (0 if r == 0 else hit)


# ---------------------------------------------------------------------------------------------------------------
# P/D and the lm:// tier
# ---------------------------------------------------------------------------------------------------------------
class _PdEngine:
    def __init__(self, n_layers, draft=None):
        self.geom = NS(n_blocks=64, stride=64 * 1152, n_layers=n_layers, n_kv_heads=1, head_dim=576, block_tokens=64,
                       elem_bytes=2, layout=_lib.LAYOUT_MLA, idx_token_bytes=0)
        if draft is not None:
            self.geom.draft_layers = draft

    def export_ipc(self):
        return b"\x07" * (72 * self.geom.n_layers)

    def import_peer(self, pid, device, descs, stride, n_blocks):
        self.imported = (pid, len(descs))


def test_pd_document_carries_the_draft_layers(tmp_path, monkeypatch):
    import json
    from b200kv import pd
    monkeypatch.setattr(pd, "SHM_DIR", str(tmp_path))
    path = pd.publish_ipc("P-mtp", _PdEngine(4, 1), device=0)
    assert json.load(open(path))["draft_layers"] == 1
    same = _PdEngine(4, 1)
    assert pd.PeerResolver(same).resolve("P-mtp") == 0 and same.imported == (0, 72 * 4)   # the draft planes too
    for consumer in (_PdEngine(3, 0), _PdEngine(4, 0), _PdEngine(3)):
        with pytest.raises(ValueError, match="draft layer.*speculative-decoding drafter"):
            pd.PeerResolver(consumer).resolve("P-mtp")
    # a document published before the field: no drafter
    pd.publish_ipc("P-old", _PdEngine(3, 0), device=0)
    doc = json.load(open(pd.ipc_path("P-old")))
    del doc["draft_layers"]
    json.dump(doc, open(pd.ipc_path("P-old"), "w"))
    assert pd.PeerResolver(_PdEngine(3)).resolve("P-old") == 0
    with pytest.raises(ValueError, match="with 0 draft layer"):
        pd.PeerResolver(_PdEngine(4, 1)).resolve("P-old")


def test_remote_tier_moves_draft_geometry_chunks_in_their_own_namespace():
    """The lm:// tier moves whole pool slots by key: a spec replica's chunks (chunk_bytes with the draft planes)
    round-trip bit-exact, and a plain replica's keys never find them."""
    from b200kv.remote import RemoteClient, RemoteServer
    spec = KVGeometry(n_layers=4, n_kv_heads=1, head_dim=576, n_blocks=1, block_tokens=16, chunk_tokens=64,
                      layout=_lib.LAYOUT_MLA, draft_layers=1)
    plain = KVGeometry(n_layers=3, n_kv_heads=1, head_dim=576, n_blocks=1, block_tokens=16, chunk_tokens=64,
                       layout=_lib.LAYOUT_MLA)
    assert spec.chunk_bytes == 4 * 64 * 576 * 2 and plain.chunk_bytes == 3 * 64 * 576 * 2
    slot = spec.chunk_bytes
    server = RemoteServer("127.0.0.1", 0, 8 * slot)
    a = KVPool(None, 4 * slot, slot, _lib.POOL_CREATE)
    b = KVPool(None, 4 * slot, slot, _lib.POOL_CREATE)
    try:
        toks = np.arange(3 * 64, dtype=np.int32)
        keys = chunk_keys(toks, 64, spec.key_seed("m"))
        rng = np.random.default_rng(0)
        c = RemoteClient("127.0.0.1", server.port)
        want = []
        for k in keys:
            s = a.reserve(int(k), 64, spec.fmt_tag, 1)
            want.append(rng.integers(0, 256, slot, dtype=np.uint8))
            a.slot_view(s)[:] = want[-1]
            a.commit(int(k))
            assert c.put(a, int(k), 1) == 0
        assert c.exists(keys) == 3
        assert c.exists(chunk_keys(toks, 64, plain.key_seed("m"))) == 0
        for k, data in zip(keys, want):
            assert c.get(b, int(k), 2) == 0
            s, n, fmt = b.acquire(int(k))
            assert np.array_equal(b.slot_view(s), data) and (n, fmt) == (64, spec.fmt_tag)
            b.release(int(k))
    finally:
        a.close()
        b.close()
        server.stop()
