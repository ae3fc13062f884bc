"""Scheduler-side and worker-side state machines of the connector, free of vLLM imports so they
can be unit-tested against fake ``SchedulerOutput``s on CPU.

Behavioural spec: vLLM's vendored LMCache adapter
(vllm/distributed/kv_transfer/kv_connector/v1/lmcache_integration/vllm_v1_adapter.py):

* which tokens a step saves                         — ReqMeta.from_request_tracker  :270-399
* lookup + "recompute the last token" rule          — get_num_new_matched_tokens    :1141-1228
* update_state_after_alloc / can_load               — :1231-1293
* build_connector_meta (new, cached, finished reqs) — :1296-1407
* start_load_kv masks / retrieve call               — :798-905
* wait_for_save masks / store call                  — :1033-1128

Restated, not copied: metadata carries block ids (16x smaller than a slot mapping to pickle
across the scheduler->worker boundary); the slot mapping slot[i] = block[i//bs]*bs + i%bs
(:368-375) is expanded on the worker.
"""
from __future__ import annotations

import logging
import os
from dataclasses import dataclass, field

import numpy as np

logger = logging.getLogger("b200kv")


@dataclass
class LoadSpec:
    vllm_cached_tokens: int      # tokens vLLM's own prefix cache already holds
    external_cached_tokens: int  # tokens the pool holds (whole chunks, maybe a partial tail)
    can_load: bool = False       # set once the scheduler allocated blocks for them


@dataclass
class SaveSpec:
    skip_leading_tokens: int     # already saved (chunk aligned by the worker)
    can_save: bool


@dataclass
class ReqMeta:
    req_id: str
    token_ids: np.ndarray        # int32, the tokens this step may save / load
    block_ids: list[int]
    is_last_prefill: bool = False
    save_spec: SaveSpec | None = None
    load_spec: LoadSpec | None = None
    async_load: bool = False     # load detached from the forward pass; completion reported by req id

    def slot_mapping(self, block_size: int) -> np.ndarray:
        b = np.asarray(self.block_ids, dtype=np.int64)
        sm = (b[:, None] * block_size + np.arange(block_size, dtype=np.int64)[None, :]).reshape(-1)
        return sm[: len(self.token_ids)]


@dataclass
class RequestTracker:
    req_id: str
    prompt_len: int
    token_ids: list[int]
    allocated_block_ids: list[int]
    num_saved_tokens: int = 0
    is_decode_phase: bool = False
    skip_save: bool = False

    def update(self, new_token_ids, new_block_ids, resumed: bool = False):
        """A running request was scheduled again (adapter :214-245)."""
        self.token_ids.extend(new_token_ids)
        if new_block_ids is None:
            new_block_ids = []
        elif isinstance(new_block_ids, tuple):
            new_block_ids = new_block_ids[0] if len(new_block_ids) else []
        if resumed:
            self.allocated_block_ids = list(new_block_ids)
        else:
            self.allocated_block_ids.extend(new_block_ids)
        if len(new_token_ids) == 1:
            self.is_decode_phase = True


def first_group(block_ids):
    """vLLM >= 0.9 hands block ids as one list per KV-cache group; single-group models only."""
    if block_ids is None:
        return []
    if isinstance(block_ids, tuple) or (len(block_ids) and isinstance(block_ids[0], (list, tuple))):
        return list(block_ids[0]) if len(block_ids) else []
    return list(block_ids)


def make_req_meta(tracker: RequestTracker, block_size: int, chunk: int, load_spec: LoadSpec | None,
                  discard_partial_chunks: bool, save_decode_cache: bool = False) -> ReqMeta | None:
    """What this step may save / load for one request (adapter :270-399)."""
    n_in = len(tracker.token_ids)
    is_last_prefill = n_in == tracker.prompt_len
    skip_leading = tracker.num_saved_tokens
    next_boundary = -(-(tracker.num_saved_tokens + 1) // chunk) * chunk
    skip_save = (tracker.skip_save
                 or (tracker.num_saved_tokens > 0 and n_in < next_boundary)
                 or (tracker.is_decode_phase and not save_decode_cache))
    if skip_save and load_spec is None:
        return None
    n_save = (n_in // chunk * chunk) if (not is_last_prefill or discard_partial_chunks) else n_in
    if not skip_save:
        tracker.num_saved_tokens = n_save
    if load_spec is not None and not load_spec.can_load:
        load_spec = None
    n_tok = n_save
    if load_spec is not None:
        n_tok = max(n_tok, min(load_spec.external_cached_tokens, n_in))
    capacity = len(tracker.allocated_block_ids) * block_size
    n_tok = min(n_tok, capacity)
    return ReqMeta(req_id=tracker.req_id,
                   token_ids=np.asarray(tracker.token_ids[:n_tok], dtype=np.int32),
                   block_ids=list(tracker.allocated_block_ids),
                   is_last_prefill=is_last_prefill,
                   save_spec=SaveSpec(skip_leading, not skip_save),   # can be a 0-token save, like the reference
                   load_spec=load_spec)


@dataclass
class KeyIdentity:
    """What, besides its token ids, decides the KV of a request.  The reference adapter overwrites the
    multimodal placeholder tokens with (16 bits of) the item's hash before lookup and before store
    (adapter :198, :344-350, :1168-1172; lmcache_integration/utils.py:63-89,169-209) and carries
    `request_configs` (the `lmcache.*` kv_transfer_params, adapter :102-117) into the chunk key; vLLM's own
    prefix cache also separates requests by `cache_salt` and LoRA adapter.  Here all of it is folded into
    the token stream the chunk keys are hashed from ("key tokens"): placeholder ranges are overwritten
    with 128 bits of the item's identifier, and a salted request has its tokens XORed with a 62-bit salt (low
    31 bits on even positions, high 31 bits on odd ones), so it shares no chunk with an unsalted one or
    with another salt."""
    salt: int = 0
    spans: list = field(default_factory=list)     # (offset, length, int32[4] words of the item's identifier)

    def apply(self, tokens, start: int = 0) -> np.ndarray:
        """Key tokens of `tokens`, which sit at positions [start, start+len) of the request."""
        out = np.array(tokens, dtype=np.int32, copy=True)
        n = len(out)
        if self.salt:
            even = (start & 1) == 0          # parity of the ABSOLUTE position: windows agree with the whole sequence
            lo, hi = np.int32(self.salt & 0x7FFFFFFF), np.int32((self.salt >> 31) & 0x7FFFFFFF)
            out[0::2] ^= lo if even else hi
            out[1::2] ^= hi if even else lo
        for off, length, words in self.spans:
            lo, hi = max(off, start), min(off + length, start + n)
            if lo < hi:
                out[lo - start:hi - start] = words[(np.arange(lo, hi) - off) % len(words)]
        return out


def _hash32(data: bytes, seed: int) -> int:
    from .engine import xxh64
    return xxh64(data, seed) & 0x7FFFFFFF


def request_identity(req) -> KeyIdentity | None:
    """KeyIdentity of a vLLM Request / NewRequestData, or None when the token ids alone decide the KV."""
    spans = []
    feats = getattr(req, "mm_features", None)
    if feats:
        items = [(getattr(f, "identifier", None), getattr(f, "mm_position", None)) for f in feats]
    elif getattr(req, "mm_hashes", None):
        items = list(zip(req.mm_hashes, getattr(req, "mm_positions", None) or []))
    else:
        items = []
    for ident, pos in items:
        if ident is None or pos is None:
            continue
        b = str(ident).encode()
        words = np.array([_hash32(b, j) for j in range(4)], dtype=np.int32)
        spans.append((int(pos.offset), int(pos.length), words))
    parts = []
    salt = getattr(req, "cache_salt", None)
    if salt:
        parts.append("salt=" + str(salt))
    lora = getattr(req, "lora_request", None)
    if lora is not None:
        parts.append("lora=" + str(getattr(lora, "lora_name", None) or getattr(lora, "lora_int_id", lora)))
    sp = getattr(req, "sampling_params", None)
    ktp = ((getattr(sp, "extra_args", None) or {}).get("kv_transfer_params") or {}) if sp is not None else {}
    tags = sorted((k, str(v)) for k, v in ktp.items() if isinstance(k, str) and k.startswith("lmcache.tag."))
    if tags:
        parts.append("tags=" + repr(tags))
    if not spans and not parts:
        return None
    salt = 0
    if parts:
        from .engine import xxh64
        salt = (xxh64("|".join(parts).encode(), 0x6B76) & ((1 << 62) - 1)) or 1
    return KeyIdentity(salt, spans)


def request_skip_save(req) -> bool:
    """Per-request opt-out `kv_transfer_params["lmcache.skip_save"]` (adapter :102-117, :311)."""
    sp = getattr(req, "sampling_params", None)
    extra = getattr(sp, "extra_args", None) or {}
    ktp = extra.get("kv_transfer_params") or {}
    return bool(ktp.get("lmcache.skip_save") or ktp.get("b200kv.skip_save"))


class SchedulerState:
    """Scheduler-role half.  `lookup(token_ids) -> hit tokens` is injected (pool index)."""

    def __init__(self, lookup, block_size: int, chunk: int, discard_partial_chunks: bool,
                 save_decode_cache: bool = False, kv_role: str = "kv_both", async_load: bool = False,
                 priority_limit: int | None = None, draft_layers: int = 0):
        self.lookup = lookup
        # attention layers of a speculative-decoding drafter in the stored chunks (num_new_matched_tokens)
        self.draft_layers = draft_layers
        # requests whose priority value exceeds the limit are served from the cache but not saved
        # (adapter :1163, :1332-1337: `request_priority > config.priority_limit`)
        self.priority_limit = priority_limit
        self._priority: dict[str, int] = {}
        # Asynchronous loads (KVConnectorBase_V1.get_num_new_matched_tokens -> (n, True)): the
        # request waits in WAITING_FOR_REMOTE_KVS while its KV streams in, other requests keep
        # running; vLLM itself recomputes the last token of a full hit
        # (vllm/v1/core/sched/scheduler.py:2069-2101).
        self.async_load = async_load
        self._pending_async: list[ReqMeta] = []
        self._async_saved: dict[str, int] = {}
        self.block_size = block_size
        self.chunk = chunk
        self.discard_partial_chunks = discard_partial_chunks
        self.save_decode_cache = save_decode_cache
        self.kv_role = kv_role
        self.load_specs: dict[str, LoadSpec] = {}
        self.trackers: dict[str, RequestTracker] = {}
        self.unfinished: dict[str, object] = {}
        self.identities: dict[str, KeyIdentity] = {}   # requests whose keys are not a function of the tokens alone
        self.num_lookups = 0
        self.num_hit_tokens = 0
        self.num_requested_tokens = 0

    # get_num_new_matched_tokens (adapter :1141-1228); side-effect free apart from the lease
    def key_tokens(self, req_id: str, tokens, start: int = 0):
        """The token stream chunk keys are hashed from (KeyIdentity); the tokens themselves for plain text."""
        ident = self.identities.get(req_id)
        return tokens if ident is None else ident.apply(tokens, start)

    def num_new_matched_tokens(self, req_id: str, prompt_token_ids, num_tokens: int,
                               num_computed_tokens: int, priority: int = 0, identity: KeyIdentity | None = None) -> int:
        if identity is not None:
            self.identities[req_id] = identity
        if self.kv_role == "kv_producer":
            return 0
        self._priority[req_id] = priority
        hit = int(self.lookup(self.key_tokens(req_id, prompt_token_ids)))
        self.num_lookups += 1
        self.num_hit_tokens += hit
        self.num_requested_tokens += len(prompt_token_ids)
        need = hit - num_computed_tokens
        if self.draft_layers:
            hit = self._draft_hit(hit)
            # A drafter's KV at position i comes from the target's hidden state at i and token i+1.  At hit-1 the
            # stored draft KV used the storing request's token hit, which no chunk key covers: report one token
            # less, still load all `hit`, and vLLM recomputes position hit-1 in the target and the drafter.  This
            # also recomputes the last token of a full-prompt hit, so nothing else is subtracted (async included).
            need = hit - num_computed_tokens - 1
        elif hit == num_tokens and not self.async_load:
            need -= 1  # full-prompt hit: vLLM must still compute the last token
        self.load_specs[req_id] = LoadSpec(num_computed_tokens, hit, False)
        return max(need, 0)

    def _draft_hit(self, hit: int) -> int:
        """The tokens to load when the one before the last is reported as the hit.  A detached load gets blocks for
        the reported tokens only, so the last loaded position, hit-1, must share a block with position hit-2.  A
        whole-chunk hit does (C % bs == 0); one that ends in a partial chunk with hit ≡ 1 (mod bs) does not, and
        is trimmed to its whole chunks."""
        while self.async_load and hit > 0 and (hit - 1) % self.block_size == 0:
            hit = (hit - 1) // self.chunk * self.chunk
        return hit

    # update_state_after_alloc (adapter :1231-1293)
    def after_alloc(self, request, num_external_tokens: int, block_ids=None):
        rid = request.request_id
        self.unfinished[rid] = request
        spec = self.load_specs.get(rid)
        if spec is None:
            return
        spec.can_load = num_external_tokens > 0
        if self.async_load and spec.can_load:
            # the request is not part of this step's SchedulerOutput: emit its load on its own
            self.load_specs.pop(rid)
            n = spec.external_cached_tokens
            toks = self.key_tokens(rid, (request.prompt_token_ids or [])[:n])
            self._pending_async.append(ReqMeta(rid, np.asarray(toks, dtype=np.int32), first_group(block_ids),
                                               load_spec=spec, async_load=True))
            self._async_saved[rid] = n

    # build_connector_meta (adapter :1296-1407)
    def build_meta(self, scheduler_output) -> list[ReqMeta]:
        out: list[ReqMeta] = self._pending_async
        self._pending_async = []
        force_skip = self.kv_role == "kv_consumer"
        for rid in scheduler_output.finished_req_ids:
            self.trackers.pop(rid, None)
            self.unfinished.pop(rid, None)
            self.load_specs.pop(rid, None)
            self._async_saved.pop(rid, None)
            self._priority.pop(rid, None)
            self.identities.pop(rid, None)
        for req in scheduler_output.scheduled_new_reqs:
            if req.req_id not in self.identities:       # normally known since the lookup; producers never look up
                ident = request_identity(req)
                if ident is not None:
                    self.identities[req.req_id] = ident
            spec = self.load_specs.pop(req.req_id, None)
            n_compute = req.num_computed_tokens + scheduler_output.num_scheduled_tokens[req.req_id]
            saved = spec.external_cached_tokens if spec is not None else self._async_saved.pop(req.req_id, 0)
            prompt = req.prompt_token_ids or []
            prio = self._priority.pop(req.req_id, 0)
            tr = RequestTracker(req.req_id, len(prompt), list(self.key_tokens(req.req_id, prompt[:n_compute])),
                                first_group(req.block_ids), num_saved_tokens=saved,
                                skip_save=force_skip or request_skip_save(req)
                                or (self.priority_limit is not None and prio > self.priority_limit))
            self.trackers[req.req_id] = tr
            m = make_req_meta(tr, self.block_size, self.chunk, spec, self.discard_partial_chunks,
                              self.save_decode_cache)
            if m is not None:
                out.append(m)
        cached = scheduler_output.scheduled_cached_reqs
        for i, rid in enumerate(cached.req_ids):
            tr = self.trackers.get(rid)
            if tr is None:
                continue
            n_new = scheduler_output.num_scheduled_tokens[rid]
            req = self.unfinished.get(rid)
            cur = len(tr.token_ids)
            if req is not None:
                new_tokens = list(req.all_token_ids[cur:cur + n_new])
            elif rid in getattr(cached, "all_token_ids", {}):
                new_tokens = list(cached.all_token_ids[rid][cur:cur + n_new])
            else:
                new_tokens = []
            if new_tokens and rid in self.identities:
                new_tokens = list(self.key_tokens(rid, new_tokens, cur))
            resumed = rid in getattr(cached, "resumed_req_ids", ())
            if resumed:
                # Preempted and scheduled again: vLLM recomputes from `num_computed_tokens` (whatever its prefix
                # cache still holds) into a NEW set of blocks (CachedRequestData, vllm/v1/core/sched/output.py:
                # 112-126).  Restart the tracker's view of the sequence; what was saved stays saved.  (The
                # reference adapter appends the new blocks to the old ones here, adapter :214-245.)
                n_comp = cached.num_computed_tokens[i] if getattr(cached, "num_computed_tokens", None) else 0
                ids = req.all_token_ids if req is not None else getattr(cached, "all_token_ids", {}).get(rid, tr.token_ids)
                tr.token_ids = list(self.key_tokens(rid, ids[: n_comp + n_new]))
                tr.allocated_block_ids = first_group(cached.new_block_ids[i])
                tr.is_decode_phase = False
            else:
                tr.update(new_tokens, cached.new_block_ids[i], False)
            m = make_req_meta(tr, self.block_size, self.chunk, None, self.discard_partial_chunks,
                              self.save_decode_cache)
            if m is not None:
                out.append(m)
        return out


@dataclass
class WorkerStats:
    num_stored_tokens: int = 0
    num_loaded_tokens: int = 0
    num_load_shortfalls: int = 0
    num_foreign_loaded_tokens: int = 0   # loaded from chunks another replica stored (shared pool)
    num_tier_local_tokens: int = 0       # loaded from this engine's device tier (no PCIe)
    num_tier_peer_tokens: int = 0        # loaded from a peer replica's device tier (NVLink, no host hop)
    retrieve_seconds: float = 0.0
    retrieve_calls: int = 0


class WorkerState:
    """Worker-role half: turns ReqMeta into engine.store / engine.retrieve calls."""

    def __init__(self, engine, block_size: int, chunk: int, kv_role: str = "kv_both", owner_tag: int = 0,
                 stores: bool = True):
        self.engine = engine
        self.owner_tag = owner_tag   # != 0: count tokens served from chunks stored under another owner tag
        # False on tensor-parallel ranks > 0 of an MLA model: the latent is the same on every rank, so rank 0's
        # copy in the host pool serves all of them and the other ranks only load
        self.stores = stores
        self.block_size = block_size
        self.chunk = chunk
        self.kv_role = kv_role
        self.load_error_blocks: set[int] = set()
        self.pending_tickets: list[int] = []
        self.async_loads: list[tuple[int, str]] = []   # (ticket, req_id) of detached loads in flight
        # layer-wise loads of the current step: (ticket, blocks it fills); the forward pass waits per layer
        self.layer_loads: list[tuple[int, list[int]]] = []
        self.on_stored = None    # callable(chunk keys) after a store was issued (remote tier upload)
        # device chunk tier (b200kv/device_tier.py): this engine's tier, and every tier it can read
        self.local_tier = None
        self.tiers = None
        # operational kill-switch: while this file exists, loads bypass the device tiers (host pool / server only);
        # lets one running deployment be measured with and without the NVLink path (tools/e2e/run_scale.py)
        self.tier_disable_file: str | None = None
        self._tier_pins: list[tuple[object, list]] = []   # (event after the scatter, [(view, key)]) still pinned
        self.event_factory = None   # stream -> object with .query(); default torch.cuda.Event (tests inject one)
        self.stats = WorkerStats()

    def start_load(self, metas: list[ReqMeta], stream=None, layers_per_group: int = 0):
        """start_load_kv (adapter :798-905).  layers_per_group > 0 = LMCache's `use_layerwise`
        (:870-880): the load is issued layer group by layer group and the caller makes the forward
        pass wait per layer (wait_for_layer_load).  The requests of one step that load from the pinned pool are
        handed to the engine together (KVEngine.retrieve_batch: one run table, one launch per staging batch)
        instead of one engine call per request as the reference adapter's loop does."""
        import time
        self.layer_loads = []
        plain = []      # (meta, tokens, sm, masked, n): pool loads that can share one engine op
        for m in metas:
            spec = m.load_spec
            if spec is None or not spec.can_load:
                continue
            n = min(spec.external_cached_tokens, len(m.token_ids))
            if n <= 0:
                continue
            tokens = m.token_ids[:n]
            sm = m.slot_mapping(self.block_size)[:n]
            masked = spec.vllm_cached_tokens // self.chunk * self.chunk
            t0 = time.perf_counter()
            try:
                ret = None
                if self.tiers is not None and not m.async_load and not (
                        self.tier_disable_file and os.path.exists(self.tier_disable_file)):
                    ret = self._load_with_tiers(tokens, sm, masked, stream)   # None: no tier holds any of it
                if ret is None and not m.async_load:
                    plain.append((m, tokens, sm, masked, n))
                    continue
                if ret is None:
                    mask = np.ones(n, dtype=bool)
                    mask[:masked] = False
                    ret, ticket = self.engine.retrieve(tokens, mask, sm, stream="detached", return_ticket=True)
                    self.async_loads.append((ticket, m.req_id))
            except Exception as e:  # no exception on the data path (SURVEY §8b "Errors"): recompute instead
                logger.error("b200kv: retrieve failed for %s: %s", m.req_id, e)
                ret = np.zeros(n, dtype=bool)
                if m.async_load:
                    self.async_loads.append((0, m.req_id))   # still has to be reported as finished
            self.stats.retrieve_seconds += time.perf_counter() - t0
            self._account_load(m, tokens, masked, n, int(ret.sum()))
        if not plain:
            return
        t0 = time.perf_counter()
        if len(plain) > 1 and hasattr(self.engine, "retrieve_batch"):
            try:
                got, ticket = self.engine.retrieve_batch([(tokens, sm, masked) for _m, tokens, sm, masked, _n in plain],
                                                         stream=stream, layers_per_group=layers_per_group)
            except Exception as e:
                logger.error("b200kv: batched retrieve of %d requests failed: %s", len(plain), e)
                got, ticket = np.zeros(len(plain), dtype=np.int64), 0
            if ticket and layers_per_group > 0:
                blocks = []
                for (m, _t, _s, masked, n), g_ in zip(plain, got):
                    blocks += m.block_ids[masked // self.block_size:(masked + int(g_) + self.block_size - 1) // self.block_size]
                self.layer_loads.append((ticket, blocks))
            for (m, tokens, _sm, masked, n), g_ in zip(plain, got):
                self._account_load(m, tokens, masked, n, int(g_))
        else:
            for m, tokens, sm, masked, n in plain:
                mask = np.ones(n, dtype=bool)
                mask[:masked] = False
                try:
                    if layers_per_group > 0:
                        ret, ticket = self.engine.retrieve(tokens, mask, sm, stream=stream, return_ticket=True,
                                                           layers_per_group=layers_per_group)
                        if ticket:
                            self.layer_loads.append((ticket, m.block_ids[masked // self.block_size:
                                                                       (n + self.block_size - 1) // self.block_size]))
                    else:
                        ret = self.engine.retrieve(tokens, mask, sm, stream=stream)
                except Exception as e:
                    logger.error("b200kv: retrieve failed for %s: %s", m.req_id, e)
                    ret = np.zeros(n, dtype=bool)
                self._account_load(m, tokens, masked, n, int(ret.sum()))
        self.stats.retrieve_seconds += time.perf_counter() - t0

    def _account_load(self, m: ReqMeta, tokens, masked: int, n: int, got: int):
        self.stats.retrieve_calls += 1
        self.stats.num_loaded_tokens += got
        if got and self.owner_tag:
            self.stats.num_foreign_loaded_tokens += self._foreign_tokens(tokens, masked, masked + got)
        if masked + got < n:
            # short load: report the blocks vLLM believes are filled so it recomputes them
            # (KVConnectorBase_V1.get_block_ids_with_load_errors, base.py:375-393)
            self.stats.num_load_shortfalls += 1
            first_bad = (masked + got) // self.block_size
            last = (n + self.block_size - 1) // self.block_size
            self.load_error_blocks.update(m.block_ids[first_bad:last])

    def _load_with_tiers(self, tokens, sm, masked: int, stream) -> np.ndarray:
        """Chunk by chunk from the nearest copy: a device tier (own, then a peer's: scatter straight from
        HBM / over NVLink) or the pinned host pool (engine.retrieve).  The loaded tokens form a prefix of
        [masked, n), like the host path."""
        n, C_ = len(tokens), self.chunk
        keys = self.engine._keys(tokens)
        ct = np.minimum(C_, n - np.arange(len(keys)) * C_).astype(np.int32)
        c0 = masked // C_
        self.tiers.refresh()
        src = self.tiers.resolve(keys[c0:], ct[c0:])      # pins what it finds
        if all(s_ is None for s_ in src):
            return None                                   # the ordinary host path (layer-wise etc.) applies
        ret = np.zeros(n, dtype=bool)
        pins, c, n_chunks = [], c0, len(keys)
        try:
            while c < n_chunks:
                e = c
                if src[c - c0] is not None:
                    while e < n_chunks and src[e - c0] is not None:
                        e += 1
                    end = min(e * C_, n)
                    ptrs = [v.base + slot * v.chunk_bytes for v, slot in src[c - c0:e - c0]]
                    self.engine.scatter_chunks(sm[c * C_:end], ptrs, stream)
                    for i in range(c, e):
                        v = src[i - c0][0]
                        pins.append((v, int(keys[i])))
                        if v.local:
                            self.stats.num_tier_local_tokens += int(ct[i])
                        else:
                            self.stats.num_tier_peer_tokens += int(ct[i])
                    ret[c * C_:end] = True
                else:
                    while e < n_chunks and src[e - c0] is None:
                        e += 1
                    end = min(e * C_, n)
                    m2 = np.ones(end, dtype=bool)
                    m2[:c * C_] = False
                    got = int(np.asarray(self.engine.retrieve(tokens[:end], m2, sm[:end], stream=stream)).sum())
                    ret[c * C_:c * C_ + got] = True
                    if got < end - c * C_:
                        break                 # the prefix ends here; later tier pins are dropped below
                c = e
        finally:
            used = {(id(v), k) for v, k in pins}
            unused = [(s_[0], int(keys[c0 + i])) for i, s_ in enumerate(src)
                      if s_ is not None and (id(s_[0]), int(keys[c0 + i])) not in used]
            self.tiers.release(unused)
            if pins:
                self._tier_pins.append((self._tier_event(stream), pins))
        return ret

    def _tier_event(self, stream):
        if self.event_factory is not None:
            return self.event_factory(stream)
        if self.local_tier is not None:
            return self.local_tier._event(stream)
        import torch
        ev = torch.cuda.Event()
        ev.record(stream if stream is not None else torch.cuda.current_stream())
        return ev

    def _foreign_tokens(self, tokens, lo: int, hi: int) -> int:
        """Tokens of [lo, hi) that sit in chunks first stored by ANOTHER instance of a shared pool
        (BASELINE.json config 3): what cross-replica reuse actually served."""
        try:
            n_hit, owners = self.engine.pool.lookup_owner(self.engine._keys(tokens[:hi]))
        except Exception:
            return 0
        out = 0
        for c in range(lo // self.chunk, min(n_hit, (hi + self.chunk - 1) // self.chunk)):
            if int(owners[c]) != self.owner_tag:
                out += min(hi, (c + 1) * self.chunk) - max(lo, c * self.chunk)
        return out

    def save(self, metas: list[ReqMeta], stream=None):
        """wait_for_save (adapter :1033-1128).  Blocks only until the gather kernels are queued;
        the caller's stream is made to wait for them, the D2H runs behind."""
        if self.kv_role == "kv_consumer" or not self.stores:
            return
        work = []     # (meta, tokens, sm, lead, n)
        for m in metas:
            ss = m.save_spec
            if ss is None or not ss.can_save:
                continue
            tokens = m.token_ids
            n = len(tokens)
            if not m.is_last_prefill:
                n = n // self.chunk * self.chunk
            lead = ss.skip_leading_tokens // self.chunk * self.chunk
            if n <= lead:
                continue
            work.append((m, tokens[:n], m.slot_mapping(self.block_size)[:n], lead, n))
        if not work:
            return
        stored = [False] * len(work)
        if len(work) > 1 and hasattr(self.engine, "store_batch"):
            # every request of the step in ONE engine op (one table upload, one launch per staging batch)
            try:
                ticket = self.engine.store_batch([(t, sm, lead) for _m, t, sm, lead, _n in work], stream=stream)
                if ticket:
                    self.pending_tickets.append(ticket)
                stored = [True] * len(work)
            except Exception as e:  # a failed store is a future miss, never a failed request
                logger.error("b200kv: batched store of %d requests failed: %s", len(work), e)
        else:
            for i, (m, t, sm, lead, n) in enumerate(work):
                mask = np.ones(n, dtype=bool)
                mask[:lead] = False
                try:
                    ticket = self.engine.store(t, mask, sm, offset=lead, stream=stream)
                except Exception as e:
                    logger.error("b200kv: store failed for %s: %s", m.req_id, e)
                    continue
                if ticket:
                    self.pending_tickets.append(ticket)
                stored[i] = True
        for ok, (m, tokens, sm, lead, n) in zip(stored, work):
            if not ok:
                continue
            self.stats.num_stored_tokens += n - lead
            if self.on_stored is not None:
                try:
                    self.on_stored(self.engine._keys(tokens)[lead // self.chunk:])
                except Exception as e:
                    logger.error("b200kv: remote upload hook failed for %s: %s", m.req_id, e)
            if self.local_tier is not None:
                try:
                    c0 = lead // self.chunk
                    keys = self.engine._keys(tokens)[c0:]
                    ct = np.minimum(self.chunk, n - (c0 + np.arange(len(keys))) * self.chunk).astype(np.int32)
                    self.local_tier.put(keys, ct, sm[lead:], self.chunk, stream)
                except Exception as e:
                    logger.error("b200kv: device tier store failed for %s: %s", m.req_id, e)
            m.save_spec.skip_leading_tokens = n

    def wait_layer(self, layer: int, stream=None):
        for ticket, _blocks in self.layer_loads:
            self.engine.wait_layer(ticket, layer, stream)

    def abandon_layer_loads(self):
        """The per-layer hooks did not run in this step (e.g. a full CUDA graph replay): the forward
        pass may have read pages that were still in flight.  Report them so vLLM recomputes."""
        for _ticket, blocks in self.layer_loads:
            self.load_error_blocks.update(blocks)
        self.layer_loads = []

    def reap(self):
        self.pending_tickets = [t for t in self.pending_tickets if not self.engine.poll(t)]
        if self.local_tier is not None:
            self.local_tier.poll()
        if self._tier_pins:
            still = []
            for ev, pins in self._tier_pins:
                if ev.query():
                    self.tiers.release(pins)
                else:
                    still.append((ev, pins))
            self._tier_pins = still

    def poll_async_loads(self) -> set[str]:
        """Request ids whose detached load has landed (finished_recving of get_finished)."""
        done, still = set(), []
        for ticket, rid in self.async_loads:
            if ticket == 0 or self.engine.poll(ticket):
                done.add(rid)
            else:
                still.append((ticket, rid))
        self.async_loads = still
        return done

    def take_load_errors(self) -> set[int]:
        e, self.load_error_blocks = self.load_error_blocks, set()
        return e
