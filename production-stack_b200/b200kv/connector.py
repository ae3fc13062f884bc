"""vLLM v1 KV-connector plugin: ``B200KVConnector``.

Loaded with
``--kv-transfer-config '{"kv_connector":"B200KVConnector","kv_connector_module_path":"b200kv.connector","kv_role":"kv_both"}'``
(vllm/distributed/kv_transfer/kv_connector/factory.py:96-128) — the slot production-stack fills
with ``LMCacheConnectorV1`` (helm/templates/deployment-vllm-multi.yaml:194-207,
operator/internal/controller/vllmruntime_controller.go:536-543).  Constructed twice by vLLM:
role SCHEDULER in the scheduler process (no CUDA) and role WORKER in each worker.

Lifecycle contract: KVConnectorBase_V1 (vllm/.../v1/base.py:171-674); the behaviour of every
method mirrors the LMCache adapter cited in b200kv/adapter.py.  The two roles share nothing but
the POSIX-shm pool index (b200kv_pool): no ZMQ lookup server, no PYTHONHASHSEED coupling.
"""
from __future__ import annotations

import logging
import os
from dataclasses import dataclass, field
from typing import TYPE_CHECKING, Any

import torch
from vllm.distributed.kv_transfer.kv_connector.v1.base import (KVConnectorBase_V1, KVConnectorMetadata,
                                                               KVConnectorRole, SupportsHMA)

from . import _lib
from .adapter import ReqMeta, SchedulerState, WorkerState, request_identity
from .config import B200KVConfig
from .engine import (FP8_CACHE_DTYPES, INDEXER_SCALE_BYTES, INDEXER_VALUE_BYTES, KVEngine, KVGeometry, KVPool,
                     dtype_code, paged_layout_of, split_indexer_caches, xxh64)
from .pd import PDMeta, PDScheduler, PDWorker, first_group, publish_ipc, unpublish_ipc

if TYPE_CHECKING:
    from vllm.config import VllmConfig
    from vllm.forward_context import ForwardContext
    from vllm.v1.core.kv_cache_manager import KVCacheBlocks
    from vllm.v1.core.sched.output import SchedulerOutput
    from vllm.v1.kv_cache_interface import KVCacheConfig
    from vllm.v1.request import Request

logger = logging.getLogger("b200kv")

_TRACE_PATH = os.environ.get("B200KV_TRACE")   # file to append per-call host timings to (debug only)


def _traced(fn):
    if not _TRACE_PATH:
        return fn
    import functools
    import time as _t

    @functools.wraps(fn)
    def wrap(self, *a, **kw):
        t0 = _t.perf_counter()
        try:
            return fn(self, *a, **kw)
        finally:
            dt = (_t.perf_counter() - t0) * 1e3
            if dt > 0.05:
                with open(_TRACE_PATH, "a") as f:
                    f.write(f"{_t.time():.6f} {self._role.name} {fn.__name__} {dt:.3f} ms\n")
    return wrap


@dataclass
class B200KVConnectorMetadata(KVConnectorMetadata):
    requests: list[ReqMeta] = field(default_factory=list)
    pd: PDMeta = field(default_factory=PDMeta)   # disaggregated-prefill pulls / held requests
    # this engine's cumulative (lookups, hit tokens, requested tokens): the worker reports them as the
    # lmcache:* series, so replicas sharing one pool each report their own traffic, not the box's
    sched_counters: tuple = (0, 0, 0)
    # this engine's scheduler's cumulative disk-tier (fetched, corrupt) chunks: the scheduler reads the disk
    disk_counters: tuple = (0, 0)


def geometry_from_vllm(vllm_config, cfg: B200KVConfig, n_blocks: int = 1) -> KVGeometry:
    """LMCache's kv_shape = (num_layer, 2, chunk, num_kv_head, head_size)
    (vllm_v1_adapter.py:471-477), derivable in both roles from the vLLM config alone.  An MLA model
    (model_config.use_mla) has one latent plane per layer: (num_layer, 1, chunk, 1, head_size)
    (vllm_v1_adapter.py:463-477).  The cache's element type: the model's with cache_dtype "auto",
    named by "float16" / "bfloat16".  Of a 1-byte cache, dtype stays bf16 and fp8_dtype says which fp8 type it holds:
    "fp8" and "fp8_e4m3" are e4m3 and "fp8_e5m2" is e5m2 (FP8_CACHE_DTYPES).  On
    those fp8 caches Q4 quantises the codes, and FP8 is stored RAW: the pages already are fp8.  Every other 1-byte
    cache dtype (fp8_per_token_head, fp8_inc) keeps the default type, which only RAW reads, and Q4 is refused.
    An MLA model with DeepSeek Sparse Attention (DeepSeek-V3.2: index_topk in the HF config, vLLM's test) also
    has an indexer key cache per layer, which the geometry's indexer planes describe.  With the fp8_ds_mla cache a
    latent token is already a 656-byte FP8 record, so the chunk stores it RAW, also when FP8 is asked for.
    With speculative decoding by a drafter that owns attention layers (draft_layers_of), those layers follow the
    target's: n_layers counts both."""
    mc, pc, cc = vllm_config.model_config, vllm_config.parallel_config, vllm_config.cache_config
    dt = str(cc.cache_dtype)
    dtype = _lib.DTYPE_BF16
    if dt in ("auto", "None"):
        elem = torch.empty((), dtype=mc.dtype).element_size()
        if mc.dtype == torch.float16:
            dtype = _lib.DTYPE_FP16
    else:
        elem = 1 if "fp8" in dt else 2
        if dt == "float16":
            dtype = _lib.DTYPE_FP16
    mla = bool(getattr(mc, "use_mla", False))
    head_dim, fmt = mc.get_head_size(), cfg.fmt
    if mla and dt == "fp8_ds_mla":
        head_dim = MLA_FP8_DS_BYTES
        if fmt == _lib.FMT_FP8:
            fmt = _lib.FMT_RAW
            _log_once("b200kv: the fp8_ds_mla cache already holds FP8 latent records: chunks are stored RAW")
    elif dt in FP8_CACHE_DTYPES and fmt == _lib.FMT_FP8:
        fmt = _lib.FMT_RAW
        _log_once(f"b200kv: the {dt} KV cache already holds fp8 codes, which the FP8 format would store as the same "
                  "bytes: chunks are stored RAW")
    elif elem == 1 and fmt == _lib.FMT_Q4 and dt not in FP8_CACHE_DTYPES:
        raise ValueError(f"B200KV_FORMAT=q4 cannot read --kv-cache-dtype {dt}: Q4 takes bf16, fp16, fp8 (fp8_e4m3) "
                         "and fp8_e5m2 caches; use B200KV_FORMAT=raw with this cache")
    hf = getattr(mc, "hf_text_config", None) or getattr(mc, "hf_config", None)
    sparse = mla and hasattr(hf, "index_topk")   # vLLM's own test for a V3.2 model (deepseek_v2.py, is_v32)
    draft = draft_layers_of(vllm_config)
    return KVGeometry(n_layers=mc.get_num_layers(pc) + draft, draft_layers=draft,
                      n_kv_heads=1 if mla else mc.get_num_kv_heads(pc),
                      head_dim=head_dim, n_blocks=n_blocks, block_tokens=cc.block_size,
                      chunk_tokens=cfg.chunk_size, elem_bytes=elem, block_stride_bytes=0, fmt=fmt,
                      layout=_lib.LAYOUT_MLA if mla else _lib.LAYOUT_NHD, dtype=dtype,
                      fp8_dtype=FP8_CACHE_DTYPES.get(dt, _lib.DTYPE_E4M3),
                      idx_value_bytes=INDEXER_VALUE_BYTES if sparse else 0,
                      idx_scale_bytes=INDEXER_SCALE_BYTES if sparse else 0)


MLA_FP8_DS_BYTES = 656   # one token of vLLM's fp8_ds_mla latent cache (uint8): the FP8 latent record
_LOGGED: set[str] = set()


def draft_layers_of(vllm_config) -> int:
    """Attention layers a speculative-decoding drafter adds to the target's KV-cache group.  vLLM puts them there
    (validate_same_kv_cache_group, v1/spec_decode/llm_base_proposer.py) and names them from num_hidden_layers
    upwards (DeepSeekMultiTokenPredictor.mtp_start_layer_idx; start_layer_id in llama_eagle.py / llama_eagle3.py).
    MTP ("mtp" and the per-model aliases vLLM folds into it): the model's num_nextn_predict_layers / n_predict.
    EAGLE and EAGLE-3: the draft model's layer count.  Every other method (ngram, suffix, ...) and no speculative
    config: 0."""
    sc = getattr(vllm_config, "speculative_config", None)
    method = str(getattr(sc, "method", None) or "")
    if sc is None or not (method == "mtp" or method.endswith("_mtp") or method in ("eagle", "eagle3")):
        return 0
    dmc = getattr(sc, "draft_model_config", None)
    hf = getattr(dmc, "hf_config", None)
    if method in ("eagle", "eagle3"):
        n = getattr(hf, "num_hidden_layers", None)
    else:
        n = getattr(hf, "n_predict", None) or getattr(hf, "num_nextn_predict_layers", None)
        if not n:
            mc = vllm_config.model_config
            thf = getattr(mc, "hf_text_config", None) or getattr(mc, "hf_config", None)
            n = getattr(thf, "num_nextn_predict_layers", None)
    if not n or int(n) < 0:
        raise ValueError(f"speculative method {method!r}: cannot tell how many attention layers the drafter has")
    if int(getattr(vllm_config.parallel_config, "pipeline_parallel_size", 1) or 1) > 1:
        # only the last stage holds the drafter, so the stages' caches would differ in more than their layer range
        raise ValueError(f"B200KVConnector does not support speculative decoding ({method!r}, {int(n)} draft "
                         "layers) with pipeline parallelism")
    return int(n)


def total_kv_heads_of(model_config) -> int:
    """The model's KV heads over all tensor-parallel ranks (ModelConfig.get_total_num_kv_heads); 0 for a config that
    cannot tell, with which P/D pairs replicas of the same tensor-parallel size only."""
    f = getattr(model_config, "get_total_num_kv_heads", None)
    return int(f()) if f else 0


def _log_once(msg: str):
    if msg not in _LOGGED:
        _LOGGED.add(msg)
        logger.info(msg)


def _layer_index_of(name: str) -> int:
    """vLLM's layer index of a KV-cache layer name ("model.layers.61.self_attn.attn" -> 61)."""
    from vllm.model_executor.models.utils import extract_layer_index
    try:
        return extract_layer_index(name)
    except (AssertionError, ValueError) as e:
        raise ValueError(f"KV cache {name}: no layer index in the name") from e


def hook_waits(layer: int, n_target: int, n_layers: int, layers_per_group: int, wait_ahead: bool) -> list[int]:
    """Layers whose load groups target layer `layer`'s wait_for_layer_load waits for (b200kv_wait_layer waits for
    the group holding the layer): its own group where it starts; with wait_ahead the next target layer's group where
    it starts; and in the last target layer's hook every group that starts at a draft layer.  A draft layer in the
    last target layer's group is covered by that group's wait."""
    G = layers_per_group
    waits = [layer] if layer % G == 0 else []
    if wait_ahead and (layer + 1) % G == 0 and layer + 1 < n_target:
        waits.append(layer + 1)
    if layer == n_target - 1:
        waits += [l for l in range(n_target, n_layers) if l % G == 0]
    return waits


def owner_tag_of(instance_id: str) -> int:
    """Stable 31-bit tag of LMCACHE_LMCACHE_INSTANCE_ID (not Python's salted hash())."""
    return (xxh64(instance_id.encode(), 0) & 0x7FFFFFFF) or 1


# per-engine segments carry vLLM's random engine id: nothing ever re-attaches to one whose engine died, so the
# scheduler role sweeps the unheld ones of earlier incarnations at start-up (k8s keeps a memory-backed emptyDir
# across container restarts inside a pod: a crash loop would otherwise fill /dev/shm)
ENGINE_POOL_PREFIX = "/b200kv-eng-"


def pool_name_for(vllm_config, cfg: B200KVConfig, chunk_bytes: int = 0) -> str:
    """One segment per engine unless B200KV_POOL_NAME names a shared one (BASELINE.json
    config 3: "shared pinned-host KV pool" across the replicas of a box).  A shared name is
    suffixed with the chunk size: replicas of DIFFERENT models on one box (the chart's modelSpec is
    a list) given the same name get one segment per geometry instead of failing to attach."""
    if cfg.pool_name:
        base = cfg.pool_name if cfg.pool_name.startswith("/") else "/" + cfg.pool_name
        return f"{base}-{chunk_bytes:x}" if chunk_bytes else base
    eid = vllm_config.kv_transfer_config.engine_id or "engine"
    return ENGINE_POOL_PREFIX + "".join(ch for ch in str(eid) if ch.isalnum() or ch in "-_")[:48]


class B200KVConnector(KVConnectorBase_V1, SupportsHMA):
    def __init__(self, vllm_config: "VllmConfig", role: KVConnectorRole,
                 kv_cache_config: "KVCacheConfig | None" = None):
        super().__init__(vllm_config=vllm_config, role=role, kv_cache_config=kv_cache_config)
        ktc = vllm_config.kv_transfer_config
        groups = getattr(kv_cache_config, "kv_cache_groups", None)
        if groups is not None and len(groups) > 1:
            # one paged cache per layer with ONE block table per request is what this engine moves; with several
            # KV-cache groups (hybrid / sliding-window models) block ids differ per group — refuse rather than
            # store pages under the wrong ids
            raise ValueError(f"B200KVConnector supports a single KV-cache group, the model has {len(groups)}: "
                             "start vLLM with --disable-hybrid-kv-cache-manager")
        self.cfg = B200KVConfig.from_env().apply_extra(ktc.kv_connector_extra_config)
        if role == KVConnectorRole.SCHEDULER and getattr(ktc, "kv_load_failure_policy", "recompute") == "fail":
            # vLLM's default (config/kv_transfer.py:70).  This connector never raises on the data path: a short or
            # failed load is REPORTED (get_block_ids_with_load_errors) so that the blocks are recomputed — under the
            # default policy vLLM fails such a request instead.
            logger.warning('b200kv: kv_load_failure_policy is "fail": a chunk that is evicted between lookup and load, an '
                           'expired P/D lease or an unreachable peer will FAIL the request; add '
                           '"kv_load_failure_policy":"recompute" to --kv-transfer-config to recompute instead')
        self.kv_role = ktc.kv_role
        self._block_size = vllm_config.cache_config.block_size
        self._chunk = self.cfg.chunk_size
        if self._chunk % self._block_size:
            raise ValueError(f"chunk size {self._chunk} must be a multiple of block size {self._block_size}")
        self._discard_partial = bool(ktc.get_from_extra_config("discard_partial_chunks", False)) \
            or not self.cfg.save_unfull_chunk
        geom = geometry_from_vllm(vllm_config, self.cfg)
        pc = vllm_config.parallel_config
        self._model = str(vllm_config.model_config.model)
        self._world = pc.tensor_parallel_size
        # the model's KV heads over all ranks and MLA-ness: P/D pairs replicas of different tensor-parallel sizes by them
        self._total_kv_heads = total_kv_heads_of(vllm_config.model_config)
        self._pool_name = pool_name_for(vllm_config, self.cfg, geom.chunk_bytes)
        if role == KVConnectorRole.SCHEDULER:
            try:
                age = int(self.cfg.extra.get("sweep_min_age_s", 60))
                n_swept = KVPool.sweep(ENGINE_POOL_PREFIX, age) + KVPool.sweep("/b200kv-dev-", age)   # pools + tier indices
                if n_swept:
                    logger.warning("b200kv: removed %d pool segment(s) left in /dev/shm by engines that died", n_swept)
            except Exception as e:     # hygiene only
                logger.debug("b200kv: segment sweep skipped (%s)", e)
        self._pool = KVPool(self._pool_name, self.cfg.pool_bytes, geom.chunk_bytes, _lib.POOL_CREATE_OR_ATTACH)
        self._engine: KVEngine | None = None
        self._worker: WorkerState | None = None
        self._wait_ahead, self._n_layers = False, 0   # layer-wise waits one layer ahead (register_kv_caches)
        self._n_target = 0                            # layers before the draft layers (register_kv_caches)
        self._sched: SchedulerState | None = None
        self._controller = None
        self._engine_id = str(ktc.engine_id or "engine")
        self._pd: PDScheduler | None = None
        self._pdw: PDWorker | None = None
        self._remote_computed: dict[str, int] = {}
        self._remote = None     # cache-server tier (LMCACHE_REMOTE_URL), b200kv/remote.py
        self._disk = None       # local-disk tier (LMCACHE_LOCAL_DISK), b200kv/disk.py
        self._disk_dir = self.cfg.disk_dir()       # None: no disk tier (a malformed value raises here)
        self._disk_prefetch = False                # scheduler: prefetch from the disk tier (not on a kv_producer)
        self._disk_counters: tuple = (0, 0)        # worker: last disk counters received from this engine's scheduler
        self._sched_counters: tuple = (0, 0, 0)   # worker: last counters received from this engine's scheduler
        if role == KVConnectorRole.SCHEDULER:
            self._pd = PDScheduler(self._engine_id, self._block_size,
                                   lease_s=float(self.cfg.extra.get("pd_lease_s", 120.0)), tp_size=self._world,
                                   total_kv_heads=self._total_kv_heads, mla=geom.mla)
            seed = self._key_seed(0)
            lease = self.cfg.lookup_lease_ms
            chunk = self._chunk
            pool = self._pool
            include_partial = not self._discard_partial

            self._tiers = None
            if self.cfg.device_tier_gb > 0:      # index-only view of every replica's device tier
                from .device_tier import TierSet
                self._tiers = TierSet(self._engine_id, geom.chunk_bytes, None)
            tiers = self._tiers

            tier_off = os.environ.get("B200KV_TIER_DISABLE_FILE") or None

            def lookup(token_ids):
                if tiers is None or (tier_off and os.path.exists(tier_off)):   # kill switch: what the host pool holds
                    return pool.lookup_tokens(token_ids, chunk, seed, lease, include_partial)
                from .device_tier import combined_prefix_tokens
                from .engine import chunk_keys
                import numpy as np
                toks = np.asarray(token_ids, dtype=np.int32)
                keys = chunk_keys(toks, chunk, seed, include_partial)
                ct = np.minimum(chunk, len(toks) - np.arange(len(keys)) * chunk).astype(np.int32)
                tiers.refresh()
                return combined_prefix_tokens(pool, tiers, keys, ct, lease)

            self._sched = SchedulerState(lookup, self._block_size, self._chunk, self._discard_partial,
                                         self.cfg.save_decode_cache, self.kv_role, async_load=self.cfg.async_load,
                                         priority_limit=self.cfg.priority_limit, draft_layers=geom.draft_layers)
            # the scheduler fetches every TP rank's chunks of a prompt (one seed for MLA: every rank loads the same
            # latent chunks); a kv_producer's scheduler keeps its disk tier for reset_cache only
            seeds = list(dict.fromkeys(self._key_seed(r) for r in range(self._world)))
            self._disk = self._make_disk(seeds)
            self._disk_prefetch = self._disk is not None and self.kv_role != "kv_producer"
            if self.kv_role != "kv_producer":
                self._remote = self._make_remote(seeds)
            if not self.cfg.pool_name:
                # a per-engine segment dies with its engine (vLLM's engine ids are random: nobody would
                # ever attach to it again); a named, shared one stays for the other replicas of the box
                import atexit
                atexit.register(KVPool.unlink, self._pool_name)
        logger.info("b200kv connector role=%s kv_role=%s pool=%s (%.1f GB, chunk %d, fmt %s)",
                    role.name, self.kv_role, self._pool_name, self.cfg.max_local_cpu_size_gb, self._chunk,
                    ("raw", "fp8", "q4")[geometry_from_vllm(self._vllm_config, self.cfg).fmt])

    def _make_remote(self, key_seeds):
        """LMCACHE_REMOTE_URL=lm://host:port (deployment-vllm-multi.yaml:338-345): the cache-server
        tier behind the local pinned pool.  A malformed URL is a fatal misconfiguration."""
        from .remote import RemoteTier, parse_remote_url
        hp = parse_remote_url(self.cfg.remote_url)
        if hp is None:
            return None
        logger.info("b200kv remote tier: %s:%d", *hp)
        return RemoteTier(self._pool, hp[0], hp[1], self._chunk, key_seeds, owner=owner_tag_of(self.cfg.instance_id),
                          include_partial=not self._discard_partial, wait_s=self.cfg.remote_wait_ms / 1e3)

    def _make_disk(self, key_seeds):
        """LMCACHE_LOCAL_DISK + LMCACHE_MAX_LOCAL_DISK_SIZE (deployment-vllm-multi.yaml:334-337): the local-disk
        tier behind the pinned pool.  A malformed value is a fatal misconfiguration; a directory that cannot hold
        the tier is a warning, and the engine runs without it."""
        d = self._disk_dir
        if d is None:
            return None
        from .config import default_disk_dir
        from .disk import DiskTier
        try:
            if d == default_disk_dir():
                os.makedirs(d, exist_ok=True)
                logger.info("b200kv disk tier: LMCACHE_LOCAL_DISK=%s, using %s", self.cfg.local_disk, d)
            tier = DiskTier(self._pool, d, self.cfg.disk_bytes, self._chunk, key_seeds,
                            owner=owner_tag_of(self.cfg.instance_id), include_partial=not self._discard_partial,
                            wait_s=self.cfg.disk_wait_ms / 1e3, prefix_lease_ms=self.cfg.lookup_lease_ms)
        except Exception as e:
            logger.warning("b200kv disk tier in %s unavailable (%s); running without it", d, e)
            return None
        st = tier.file.stats()
        logger.info("b200kv disk tier: %s, %d chunk slots (%.1f GB), %d chunks restored, %s I/O", d, st["n_slots"],
                    st["n_slots"] * st["slot_bytes"] / 1e9, st["n_restored"], "direct" if st["direct_io"] else "buffered")
        return tier

    def _key_seed(self, rank: int) -> int:
        """Same namespace in both roles: derived from the vLLM config only (the tile layout is a
        per-process constant of the attention backend, so it need not enter the scheduler's seed;
        chunks are additionally tagged with their format in the pool)."""
        return geometry_from_vllm(self._vllm_config, self.cfg).key_seed(self._model, self._world, rank)

    # ------------------------------------------------------------------ class-level hooks
    @classmethod
    def get_required_kvcache_layout(cls, vllm_config: "VllmConfig") -> str | None:
        # Both tile orders are supported; NHD is preferred when the backend leaves the choice
        # (vLLM's FlashInfer backend imposes HND, selector.py:124-133).
        return "NHD"

    # ------------------------------------------------------------------ worker side
    def register_kv_caches(self, kv_caches: dict[str, torch.Tensor]):
        """KVConnectorBase_V1.register_kv_caches (base.py:251) — adapter :786-795."""
        if not kv_caches:
            raise ValueError("no KV cache tensors to register")
        # Layer order is the layer index, not the dict's order: the target's layers 0..L-1, then a drafter's
        # L..L+D-1 (vLLM puts them in the same group).  A stable sort keeps DeepSeek-V3.2's indexer caches in the
        # same order as the latent ones.
        kv_caches = dict(sorted(kv_caches.items(), key=lambda kv: _layer_index_of(kv[0])))
        # DeepSeek-V3.2: the latent layers and the indexer caches of the same layers come in one group
        tensors, idx = split_indexer_caches(kv_caches)
        t0 = tensors[0]
        k, v, stride, nb, h, d, tile_layout = paged_layout_of(t0, self._block_size)
        geom0 = geometry_from_vllm(self._vllm_config, self.cfg)
        # only the attention layers call wait_for_layer_load: the hook is keyed by the latent layers' names
        lat_names = [n for n, t in kv_caches.items() if not any(t is x for x in idx)]
        if geom0.draft_layers:
            L, D = geom0.target_layers, geom0.draft_layers
            drafts = [i for i in map(_layer_index_of, lat_names) if i >= L]
            if drafts != list(range(L, L + D)):
                raise ValueError(f"KV cache tensors do not match the model geometry: the speculative config implies "
                                 f"{D} draft layer(s) with indices {L}..{L + D - 1} after the {L} target layers, the "
                                 f"registered layers have {len(drafts)} at or above index {L}: {drafts}")
        cache_dtype = str(self._vllm_config.cache_config.cache_dtype)
        if t0.element_size() != geom0.elem_bytes:
            raise ValueError(f"KV cache tensors hold {t0.element_size()}-byte elements ({t0.dtype}); the vLLM config's "
                             f"cache dtype {cache_dtype!r} implies {geom0.elem_bytes}-byte ones")
        # the tensor's type where it names one; vLLM's uint8 fp8 caches take the flavour the config names
        code, fp8 = dtype_code(t0.dtype, cache_dtype), t0.element_size() == 1
        geom = KVGeometry(n_layers=len(tensors), n_kv_heads=h, head_dim=d, n_blocks=nb,
                          block_tokens=self._block_size, chunk_tokens=self._chunk,
                          elem_bytes=t0.element_size(), block_stride_bytes=stride, fmt=geom0.fmt,
                          layout=tile_layout, dtype=_lib.DTYPE_BF16 if fp8 else (code or _lib.DTYPE_BF16),
                          fp8_dtype=(geom0.fp8_dtype if code is None else code) if fp8 else _lib.DTYPE_E4M3,
                          idx_value_bytes=INDEXER_VALUE_BYTES if idx else 0,
                          idx_scale_bytes=INDEXER_SCALE_BYTES if idx else 0,
                          idx_block_stride_bytes=idx[0].stride(0) if idx else 0,
                          draft_layers=geom0.draft_layers)
        if geom.indexed != geom0.indexed:
            raise ValueError("KV cache tensors " + ("include" if idx else "lack") + " indexer caches, which the "
                             "model config " + ("does not imply" if idx else "implies"))
        if geom.chunk_bytes != geom0.chunk_bytes:
            raise ValueError("KV cache tensors do not match the model geometry the pool was sized for "
                             f"({geom.chunk_bytes} vs {geom0.chunk_bytes} bytes per chunk, {len(tensors)} vs "
                             f"{geom0.n_layers} layers of which {geom0.draft_layers} draft layers)")
        if geom.cache_dtype != geom0.cache_dtype:   # the key seed is derived from the vLLM config's type
            raise ValueError(f"KV cache dtype {t0.dtype} differs from the one the vLLM config implies")
        rank = getattr(self._vllm_config.parallel_config, "rank", 0)
        self._rank = rank
        self._engine = KVEngine(geom, self._pool, device=t0.device.index or 0,
                                staging_bytes=self.cfg.staging_mb << 20, owner=owner_tag_of(self.cfg.instance_id),
                                variant=self.cfg.variant, key_seed=self._key_seed(rank),
                                # a pool shared by the box's replicas is interleaved over the sockets, a
                                # per-engine pool lives on the GPU's own node
                                numa_policy=_lib.NUMA_INTERLEAVE if self.cfg.pool_name else _lib.NUMA_LOCAL)
        logger.info("b200kv pool pages: %s", self._engine.numa_placement())
        self._engine.register_kv_caches(kv_caches if idx else tensors)
        self._layer_index = {name: i for i, name in enumerate(lat_names)}
        self._n_layers, self._n_target = len(lat_names), geom.target_layers
        # DeepSeek-V3.2 runs layer l's indexer, which reads the indexer keys of layer l, BEFORE layer l's attention
        # calls wait_for_layer_load; the indexer calls no connector hook.  Layer-wise loads then wait one layer
        # ahead: layer 0's group in start_load_kv, layer l+1's group in layer l's hook.
        self._wait_ahead = geom.indexed
        self._layer_hooks_seen = 0
        self._worker = WorkerState(self._engine, self._block_size, self._chunk, self.kv_role,
                                   owner_tag=owner_tag_of(self.cfg.instance_id) if self.cfg.pool_name else 0,
                                   stores=not geom.mla or self._tp_rank() == 0)   # MLA: rank 0 stores for all ranks
        if self.cfg.device_tier_gb > 0:
            from .device_tier import LocalTier, TierSet
            fmt_tag = geom.fmt_tag
            try:
                n_slots = max(1, int(self.cfg.device_tier_gb * (1 << 30)) // geom.chunk_bytes)
                self._worker.tiers = TierSet(self._engine_id, geom.chunk_bytes, fmt_tag, importer=self._engine.tier_import)
                self._worker.tier_disable_file = os.environ.get("B200KV_TIER_DISABLE_FILE") or None
                if self.kv_role != "kv_consumer":
                    self._worker.local_tier = LocalTier(self._engine, self._engine_id, n_slots, t0.device.index or 0,
                                                        fmt_tag, owner_tag_of(self.cfg.instance_id))
                    self._worker.tiers.add_local(self._worker.local_tier)
                logger.info("b200kv device tier: %d chunk slots in HBM", n_slots)
            except Exception as e:
                logger.warning("b200kv: device tier unavailable (%s)", e)
                self._worker.tiers = self._worker.local_tier = None
        if self.kv_role != "kv_consumer":
            self._remote = self._make_remote(self._engine.key_seed)
            self._disk = self._make_disk(self._engine.key_seed)
            hooks = [t.push for t in (self._disk, self._remote) if t is not None]   # write through / upload
            if len(hooks) == 1:
                self._worker.on_stored = hooks[0]
            elif hooks:
                self._worker.on_stored = lambda keys: [h(keys) for h in hooks]
        try:
            tp_rank = self._tp_rank()
            publish_ipc(self._engine_id, self._engine, t0.device.index or 0, tp_rank, self._world,
                        total_kv_heads=self._total_kv_heads)   # peers may pull from us
            self._pdw = PDWorker(self._engine, self._engine_id, self._block_size, rank=tp_rank, tp_size=self._world,
                                 total_kv_heads=self._total_kv_heads)
        except Exception as e:  # e.g. VMM-allocated cache (sleep mode): P/D pull unavailable, offload still works
            logger.warning("b200kv: cannot publish CUDA-IPC descriptors (%s); peer pull disabled", e)
        if self.cfg.enable_controller and self.cfg.controller_pull_url and rank == 0:
            from .controller_client import ControllerClient
            self._controller = ControllerClient(
                self.cfg.controller_pull_url, self.cfg.instance_id, self._pool_name, self._engine.key_seed,
                self._chunk, owner_tag=owner_tag_of(self.cfg.instance_id) if self.cfg.pool_name else 0,
                include_partial=not self._discard_partial, heartbeat_s=self.cfg.worker_heartbeat_s,
                ip=self.cfg.advertise_ip)
        logger.info("b200kv registered %d layers (%d draft), %d blocks, stride %d", len(tensors), geom.draft_layers,
                    nb, stride)

    def _tp_rank(self) -> int:
        """This worker's tensor-parallel rank (every rank of an engine shares the engine id)."""
        try:
            from vllm.distributed.parallel_state import get_tensor_model_parallel_rank
            return int(get_tensor_model_parallel_rank())
        except Exception:
            return int(getattr(self._vllm_config.parallel_config, "rank", 0) or 0) % max(self._world, 1)

    def _metas(self) -> list[ReqMeta]:
        md = self._get_connector_metadata()
        assert isinstance(md, B200KVConnectorMetadata)
        return md.requests

    @_traced
    def start_load_kv(self, forward_context: "ForwardContext", **kwargs: Any) -> None:
        if self._worker is None:
            return
        stream = torch.cuda.current_stream()
        md = self._get_connector_metadata()
        if isinstance(md, B200KVConnectorMetadata) and md.sched_counters[0] >= self._sched_counters[0]:
            self._sched_counters = tuple(md.sched_counters)
            self._disk_counters = tuple(md.disk_counters)
        if self._pdw is not None and isinstance(md, B200KVConnectorMetadata) and (md.pd.pulls or md.pd.held):
            self._pdw.start_pulls(md.pd, stream=stream)
        self._layer_hooks_seen = 0
        # A step replayed as ONE full CUDA graph never runs the per-layer hooks (base.py:591-611): use
        # the chunk-wise load there (e.g. a full-prompt hit that only recomputes its last token).
        full_graph = getattr(getattr(forward_context, "cudagraph_runtime_mode", None), "name", "NONE") == "FULL"
        self._worker.start_load(self._metas(), stream=stream,
                                layers_per_group=self.cfg.layer_group if (self.cfg.layerwise and not full_graph) else 0)
        if self._wait_ahead and self._worker.layer_loads:
            self._worker.wait_layer(0, stream)     # layer 0's indexer runs before any hook

    def wait_for_layer_load(self, layer_name: str) -> None:
        """Chunk-wise loads are ordered before the forward pass by a stream wait.  Layer-wise loads
        (B200KV_LAYERWISE=1; LMCache `use_layerwise`, adapter :907-929): the compute stream waits
        here, once per layer group, while later groups are still crossing PCIe.  With indexer caches (DeepSeek-V3.2)
        the wait runs one layer ahead: the next layer's indexer reads its keys before that layer's hook runs.
        A speculative-decoding drafter runs right after the last target layer, on the same stream, and its own hooks
        may not run (CUDA-graph replay): the last target layer's hook also waits for every group holding a draft
        layer, both planes of each included, and a draft layer's hook does nothing."""
        w = self._worker
        if w is None or not w.layer_loads:
            return
        idx = self._layer_index.get(layer_name)
        if idx is None or idx >= self._n_target:
            return
        self._layer_hooks_seen += 1
        for l in hook_waits(idx, self._n_target, self._n_layers, self.cfg.layer_group, self._wait_ahead):
            w.wait_layer(l, torch.cuda.current_stream())

    def save_kv_layer(self, layer_name: str, kv_layer: torch.Tensor, attn_metadata, **kwargs: Any) -> None:
        return  # whole-request store in wait_for_save: CUDA-graph replay skips per-layer hooks (base.py:591-611)

    @_traced
    def wait_for_save(self):
        if self._worker is None:
            return
        if self._worker.layer_loads and self._layer_hooks_seen == 0:
            # the per-layer hooks never ran in this step: do not trust the loaded pages, and stop
            # using the layer-wise path in this process
            logger.error("b200kv: wait_for_layer_load was not called during a step with layer-wise loads; "
                         "falling back to chunk-wise loads")
            self._worker.abandon_layer_loads()
            self.cfg.layerwise = False
        self._worker.layer_loads = []
        self._worker.save(self._metas(), stream=torch.cuda.current_stream())

    @_traced
    def get_finished(self, finished_req_ids: set[str]) -> tuple[set[str] | None, set[str] | None]:
        recv = None
        if self._worker is not None:
            self._worker.reap()
            recv = self._worker.poll_async_loads() or None    # detached pool loads that have landed
        sent = None
        if self._pdw is not None:
            sent, _pulled = self._pdw.poll(block=True)   # P/D pulls are synchronous for the scheduler
            sent = sent or None
        return sent, recv

    def get_block_ids_with_load_errors(self) -> set[int]:
        bad = self._worker.take_load_errors() if self._worker is not None else set()
        if self._pdw is not None:
            bad |= self._pdw.take_failed_blocks()
        return bad

    # ------------------------------------------------------------------ stats (lmcache:* series)
    @_traced
    def get_kv_connector_stats(self):
        """Worker side: deltas since the previous call (base.py:403)."""
        if self._worker is None or self._pool is None:
            return None
        from .metrics import B200KVStats
        ws = self._worker.stats
        ps = self._pool.stats()
        cur = {"num_stored_tokens": ws.num_stored_tokens, "num_loaded_tokens": ws.num_loaded_tokens,
               "retrieve_seconds": ws.retrieve_seconds, "retrieve_calls": ws.retrieve_calls,
               "load_shortfalls": ws.num_load_shortfalls, "num_foreign_loaded_tokens": ws.num_foreign_loaded_tokens,
               "num_tier_local_tokens": ws.num_tier_local_tokens, "num_tier_peer_tokens": ws.num_tier_peer_tokens,
               # the scheduler's counters are per engine, not per TP rank: rank 0 reports them
               "num_hit_tokens": self._sched_counters[1] if getattr(self, "_rank", 0) == 0 else 0,
               "num_requested_tokens": self._sched_counters[2] if getattr(self, "_rank", 0) == 0 else 0,
               "retrieve_bytes": ws.num_loaded_tokens * self._engine.geom.payload_bytes_per_token,
               "store_bytes": ws.num_stored_tokens * self._engine.geom.payload_bytes_per_token}
        if self._disk_dir is not None:
            ds = self._disk.stats() if self._disk is not None else {}
            rank0 = getattr(self, "_rank", 0) == 0     # the scheduler's counters are per engine
            cur.update({"disk_written_chunks": ds.get("written_chunks", 0),
                        "disk_skipped_chunks": ds.get("skipped_chunks", 0),
                        "disk_fetched_chunks": self._disk_counters[0] if rank0 else 0,
                        "disk_corrupt_chunks": self._disk_counters[1] if rank0 else 0})
        prev = getattr(self, "_stats_prev", {})
        delta = {k: v - prev.get(k, 0) for k, v in cur.items()}
        self._stats_prev = cur
        if not any(delta.values()):
            return None
        delta["local_cache_usage_bytes"] = ps["n_used"] * ps["slot_bytes"]
        delta["local_cache_capacity_bytes"] = ps["n_slots"] * ps["slot_bytes"]
        if self._disk is not None:
            delta["disk_usage_bytes"] = self._disk.stats()["usage_bytes"]
        return B200KVStats(delta)

    @classmethod
    def build_kv_connector_stats(cls, data: dict[str, Any] | None = None):
        from .metrics import B200KVStats
        return B200KVStats(data=data) if data is not None else B200KVStats()

    @classmethod
    def build_prom_metrics(cls, vllm_config, metric_types, labelnames, per_engine_labelvalues):
        from .metrics import B200KVPromMetrics
        return B200KVPromMetrics(vllm_config, metric_types, labelnames, per_engine_labelvalues)

    def shutdown(self):
        if self._remote is not None:
            self._remote.close()
            self._remote = None
        if self._disk is not None:
            self._disk.close()
            self._disk = None
        if self._controller is not None:
            self._controller.close()
            self._controller = None
        if self._pdw is not None:
            unpublish_ipc(self._engine_id, self._pdw.rank)
            self._pdw = None
        if self._pd is not None:
            self._pd.close()
        if self._worker is not None and self._worker.tiers is not None:
            if self._worker.local_tier is not None:
                self._worker.local_tier.close()
            self._worker.tiers.close()
            self._worker.tiers = self._worker.local_tier = None
        if getattr(self, "_tiers", None) is not None:
            self._tiers.close()
            self._tiers = None
        if self._engine is not None:
            self._engine.wait_all()
            self._engine.close()
            self._engine = None
        if self._pool is not None:
            self._pool.close()
            self._pool = None
            if self._sched is not None and not self.cfg.pool_name:
                KVPool.unlink(self._pool_name)    # mappings of the workers stay valid until they exit

    # ------------------------------------------------------------------ scheduler side
    @_traced
    def get_num_new_matched_tokens(self, request: "Request", num_computed_tokens: int) -> tuple[int | None, bool]:
        assert self._sched is not None and self._pd is not None
        remote = self._pd.remote_prefill_tokens(request, num_computed_tokens)
        if remote is not None:   # decode side of a disaggregated request: pull from the prefiller
            self._remote_computed[request.request_id] = num_computed_tokens
            return remote, False
        # multimodal items, cache_salt, LoRA adapter and lmcache.tag.* enter the chunk keys (adapter :1168-1172)
        ident = self._sched.identities.get(request.request_id) or request_identity(request)
        prompt = request.prompt_token_ids or []
        # chunks on their way from the local disk, then from the cache server for what is still missing: ask again
        # next step.  The disk's wait ends before the server's begins, so a request waits at most both budgets.
        if self._disk_prefetch and self._disk.prefetch_state(
                request.request_id, prompt if ident is None else ident.apply(prompt)) == self._disk.PENDING:
            return None, False
        if self._remote is not None and self._remote.prefetch_state(
                request.request_id, prompt if ident is None else ident.apply(prompt)) == self._remote.PENDING:
            return None, False   # chunks are on their way from the cache server: ask again next step
        n = self._sched.num_new_matched_tokens(request.request_id, prompt,
                                               request.num_tokens, num_computed_tokens,
                                               int(getattr(request, "priority", 0) or 0), identity=ident)
        return n, bool(self._sched.async_load and n > 0)

    @_traced
    def update_state_after_alloc(self, request: "Request", blocks: "KVCacheBlocks", num_external_tokens: int):
        assert self._sched is not None and self._pd is not None
        if request.request_id in self._remote_computed:
            local = first_group(blocks.get_block_ids()) if blocks is not None else []
            self._pd.after_alloc(request, local, num_external_tokens, self._remote_computed.pop(request.request_id))
            self._sched.unfinished[request.request_id] = request
            return
        self._sched.after_alloc(request, num_external_tokens,
                                blocks.get_block_ids() if blocks is not None else None)

    @_traced
    def build_connector_meta(self, scheduler_output: "SchedulerOutput") -> KVConnectorMetadata:
        assert self._sched is not None and self._pd is not None
        sc = self._sched
        md = B200KVConnectorMetadata(sc.build_meta(scheduler_output), self._pd.build_meta(),
                                     (sc.num_lookups, sc.num_hit_tokens, sc.num_requested_tokens))
        if self._disk is not None:
            ds = self._disk.stats()
            md.disk_counters = (ds["fetched_chunks"], ds["corrupt_chunks"])
        return md

    @_traced
    def request_finished(self, request: "Request", block_ids: list[int]) -> tuple[bool, dict[str, Any] | None]:
        # Offload: the gather that reads a request's pages is ordered before any later forward pass
        # on the compute stream, so blocks may be freed immediately.  Disaggregated prefill: keep
        # the pages (delay_free) until the decoder has pulled them (b200kv/pd.py).
        self._remote_computed.pop(request.request_id, None)   # looked up as a remote prefill but never allocated
        if self._remote is not None:
            self._remote.forget(request.request_id)
        if self._disk is not None:
            self._disk.forget(request.request_id)
        if self._pd is not None:
            ok = True
            st = getattr(request, "status", None)
            if st is not None:
                ok = getattr(st, "name", str(st)) in ("FINISHED_LENGTH_CAPPED", "FINISHED_STOPPED")
            delay, params = self._pd.request_finished(request, block_ids, ok)
            if delay:
                return True, params
        return False, None

    def update_connector_output(self, connector_output):
        if self._pd is not None:
            self._pd.sending_finished(getattr(connector_output, "finished_sending", None))

    def request_finished_all_groups(self, request: "Request", block_ids: tuple[list[int], ...]):
        return self.request_finished(request, block_ids[0] if block_ids else [])

    def reset_cache(self) -> bool | None:
        if self._pool is None:
            return None
        ok = self._pool.clear()
        if self._disk is not None:
            ok = self._disk.clear() and ok
        return ok
