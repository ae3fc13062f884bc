"""Disaggregated prefill -> decode hand-off by consumer-side peer pull (SURVEY.md §8a row A9).

Reference behaviour being replaced: LMCache + NIXL push the prefiller's KV into a 1 GiB GPU buffer
on the decoder (`LMCACHE_ENABLE_NIXL`, `LMCACHE_NIXL_*`, helm/templates/deployment-vllm-multi.yaml:
296-324; examples/disaggregated_prefill/start_{prefill,decode}.sh).  The router side of the
protocol is unchanged: route_orchestrated_disaggregated_request sends the prefill request with
`kv_transfer_params{do_remote_decode:true}`, copies the returned `kv_transfer_params` (filling
`remote_host`) into the decode request (src/vllm_router/services/request_service/request.py:
771-778, 823-829).  The parameter names follow vLLM's NixlConnector, which defines that protocol
(vllm/.../v1/nixl/scheduler.py:356-420, 590-690).

Here the decode replica reads the prefill replica's pages directly over NVSwitch
(b200kv_peer_pull_async): no staging buffer, no UCX, no NCCL.  Control plane on one box:
  * every worker (one per tensor-parallel rank) publishes the CUDA-IPC descriptors of its paged cache
    in /dev/shm/b200kv-ipc-<engine_id>.r<rank>.json (b200kv_export_ipc); decode rank r pulls from
    prefill rank r, and the two sides must have the same tensor-parallel size (`tp_size` in the params);
  * the producer keeps a finished request's blocks (`delay_free=True`) until every consumer rank dropped
    a marker /dev/shm/b200kv-done-<producer_engine_id>.r<rank>/<request_id>, or a lease expires;
  * the LEASE is a file /dev/shm/b200kv-lease-<producer_engine_id>/<lease_id>, created by the producer's
    scheduler before it hands out the params and removed by it right before the blocks are freed
    (update_connector_output precedes the free, vllm/v1/core/sched/scheduler.py:2136-2165).  A consumer
    checks it before AND after its pull: a pull that finished while the lease still existed read pages
    that had not been recycled; otherwise the blocks are reported as load errors and recomputed — an
    expired lease can no longer hand recycled pages to a decoder silently.
"""
from __future__ import annotations

import base64
import json
import os
import time
from dataclasses import dataclass, field

import numpy as np

from ._lib import DTYPE_BF16

SHM_DIR = os.environ.get("B200KV_SHM_DIR", "/dev/shm")


def _safe(s: str) -> str:
    return "".join(ch for ch in str(s) if ch.isalnum() or ch in "-_.")[:96]


def _rank_tag(rank: int) -> str:
    return f".r{int(rank)}" if rank else ""      # rank 0 keeps the historical names


def ipc_path(engine_id: str, rank: int = 0) -> str:
    return os.path.join(SHM_DIR, f"b200kv-ipc-{_safe(engine_id)}{_rank_tag(rank)}.json")


def done_dir(engine_id: str, rank: int = 0) -> str:
    return os.path.join(SHM_DIR, f"b200kv-done-{_safe(engine_id)}{_rank_tag(rank)}")


def lease_path(engine_id: str, lease_id: str) -> str:
    return os.path.join(SHM_DIR, f"b200kv-lease-{_safe(engine_id)}", _safe(lease_id))


_PD_TRACE = os.environ.get("B200KV_PD_TRACE")     # file: one JSON line per hand-off event (measurement only)


def trace(event: str, **kw):
    if _PD_TRACE:
        try:
            with open(_PD_TRACE, "a") as f:
                f.write(json.dumps({"t": time.time(), "event": event, **kw}) + "\n")
        except OSError:
            pass


# ------------------------------------------------------------------------------------------------
# publication of a replica's cache (worker role, after register_kv_caches)
# ------------------------------------------------------------------------------------------------
def _dtype_of(geom) -> int:
    """The cache element type of a geometry (KVGeometry.dtype; bf16 for a geometry without one)."""
    return int(getattr(geom, "dtype", DTYPE_BF16))


def _indexer_of(geom) -> int:
    """Bytes per token of a geometry's indexer planes (KVGeometry.idx_token_bytes; 0 = none)."""
    return int(getattr(geom, "idx_token_bytes", 0))


def _draft_of(geom) -> int:
    """Draft layers among a geometry's layers (KVGeometry.draft_layers; 0 for a geometry without the field)."""
    return int(getattr(geom, "draft_layers", 0))


def publish_ipc(engine_id: str, engine, device: int, rank: int = 0, tp_size: int = 1) -> str:
    g = engine.geom
    doc = {"engine_id": engine_id, "device": device, "pid": os.getpid(), "rank": rank, "tp_size": tp_size,
           "n_blocks": g.n_blocks,
           "block_stride": g.stride, "n_layers": g.n_layers, "n_kv_heads": g.n_kv_heads, "head_dim": g.head_dim,
           "block_tokens": g.block_tokens, "elem_bytes": g.elem_bytes, "layout": g.layout, "dtype": _dtype_of(g),
           "indexer": _indexer_of(g), "draft_layers": _draft_of(g),
           "descs": base64.b64encode(engine.export_ipc()).decode()}
    path = ipc_path(engine_id, rank)
    tmp = path + f".{os.getpid()}.tmp"
    with open(tmp, "w") as f:
        json.dump(doc, f)
    os.replace(tmp, path)  # atomic: readers never see a torn file
    os.makedirs(done_dir(engine_id, rank), exist_ok=True)
    return path


def unpublish_ipc(engine_id: str, rank: int = 0):
    for p in (ipc_path(engine_id, rank),):
        try:
            os.unlink(p)
        except OSError:
            pass
    d = done_dir(engine_id, rank)
    if os.path.isdir(d):
        for f in os.listdir(d):
            try:
                os.unlink(os.path.join(d, f))
            except OSError:
                pass
        try:
            os.rmdir(d)
        except OSError:
            pass


class PeerResolver:
    """remote engine_id -> peer_id of this engine; maps the peer's cache on first use."""

    def __init__(self, engine, max_peers: int = 64, rank: int = 0, tp_size: int = 1):
        self.engine = engine
        self.ids: dict[str, int] = {}
        self.max_peers = max_peers
        self.rank, self.tp_size = rank, tp_size

    def resolve(self, remote_engine_id: str) -> int:
        pid = self.ids.get(remote_engine_id)
        if pid is not None:
            return pid
        with open(ipc_path(remote_engine_id, self.rank)) as f:    # the SAME rank's shard of the peer engine
            doc = json.load(f)
        if int(doc.get("tp_size", 1)) != self.tp_size or int(doc.get("rank", 0)) != self.rank:
            raise ValueError(f"peer {remote_engine_id}: tensor-parallel layout {doc.get('rank')}/{doc.get('tp_size')} "
                             f"differs from local {self.rank}/{self.tp_size}")
        g = self.engine.geom
        doc.setdefault("dtype", DTYPE_BF16)   # documents published before the field are bf16 caches
        doc.setdefault("indexer", 0)          # ... and caches without indexer planes
        doc.setdefault("draft_layers", 0)     # ... and replicas without a speculative-decoding drafter
        if (doc["n_layers"], doc["draft_layers"]) != (g.n_layers, _draft_of(g)):
            # a drafter's layers follow the target's in the cache: the pages of a replica with one are not those of
            # a replica without one (or with another drafter)
            raise ValueError(f"peer {remote_engine_id}: n_layers={doc['n_layers']} with {doc['draft_layers']} draft "
                             f"layer(s) differs from local {g.n_layers} with {_draft_of(g)}: replicas pair only "
                             "with the same speculative-decoding drafter, or both without one")
        for k, mine in (("n_kv_heads", g.n_kv_heads), ("head_dim", g.head_dim),
                        ("block_tokens", g.block_tokens), ("elem_bytes", g.elem_bytes), ("layout", g.layout),
                        ("dtype", _dtype_of(g)), ("indexer", _indexer_of(g))):
            if doc[k] != mine:
                raise ValueError(f"peer {remote_engine_id}: {k}={doc[k]} differs from local {mine}")
        pid = len(self.ids)
        if pid >= self.max_peers:
            raise RuntimeError("too many peers")
        self.engine.import_peer(pid, doc["device"], base64.b64decode(doc["descs"]), doc["block_stride"], doc["n_blocks"])
        self.ids[remote_engine_id] = pid
        return pid


def slots_of(block_ids, block_tokens: int, n_tokens: int) -> np.ndarray:
    b = np.asarray(block_ids, dtype=np.int64)
    return (b[:, None] * block_tokens + np.arange(block_tokens, dtype=np.int64)[None, :]).reshape(-1)[:n_tokens]


# ------------------------------------------------------------------------------------------------
# scheduler-role state
# ------------------------------------------------------------------------------------------------
@dataclass
class PullSpec:
    req_id: str
    remote_engine_id: str
    remote_request_id: str
    remote_block_ids: list[int]
    local_block_ids: list[int]
    n_tokens: int          # tokens [skip_tokens, n_tokens) are pulled
    skip_tokens: int = 0   # already computed locally (block aligned): left untouched
    remote_lease_id: str = ""   # the producer's lease on its blocks (checked before and after the pull)


@dataclass
class PDMeta:
    pulls: list[PullSpec] = field(default_factory=list)
    # producer: request ids whose blocks are held for a consumer, with their lease deadline
    held: dict[str, float] = field(default_factory=dict)


class PDScheduler:
    def __init__(self, engine_id: str, block_size: int, lease_s: float = 120.0, tp_size: int = 1,
                 blocks_known_at_alloc: bool = True):
        self.engine_id = engine_id
        self.block_size = block_size
        self.lease_s = lease_s
        self.tp_size = tp_size
        # False under vLLM's LMCacheConnectorV1 wrapper, which drops `blocks` from update_state_after_alloc
        # (lmcache_connector.py:253-262): a pull would have nowhere to land, so remote prefills are declined
        # there and the request is served by the pool lookup / recomputed
        self.blocks_known_at_alloc = blocks_known_at_alloc
        self._pending_pulls: dict[str, PullSpec] = {}
        self._held: dict[str, float] = {}
        self._new_held: dict[str, float] = {}
        self._leases: dict[str, str] = {}      # request id -> lease id (files this scheduler created)

    # ---- consumer -------------------------------------------------------------------------
    def remote_prefill_tokens(self, request, num_computed_tokens: int) -> int | None:
        """Tokens obtainable from a remote prefiller for this request, or None if it is not a
        remote-prefill request (then the ordinary pool lookup applies)."""
        p = getattr(request, "kv_transfer_params", None)
        if not p or not p.get("do_remote_prefill") or not p.get("remote_block_ids") or not p.get("remote_engine_id"):
            return None
        if not self.blocks_known_at_alloc or int(p.get("tp_size") or 1) != self.tp_size:
            return None      # cannot pull (see __init__ / different tensor-parallel layout): ordinary request
        n_prompt = len(request.prompt_token_ids or [])
        n_remote = min(int(p.get("remote_num_tokens") or n_prompt), n_prompt,
                       len(first_group(p["remote_block_ids"])) * self.block_size)
        # the last prompt token is recomputed locally (same rule as a full pool hit)
        return max(min(n_remote, n_prompt - 1) - num_computed_tokens, 0)

    def after_alloc(self, request, local_block_ids: list[int], num_external_tokens: int, num_computed_tokens: int = 0):
        p = getattr(request, "kv_transfer_params", None)
        if not p or not p.get("do_remote_prefill"):
            return
        p["do_remote_prefill"] = False  # consumed (mirrors NixlConnector)
        if num_external_tokens <= 0:
            return
        trace("decode_alloc", req=request.request_id, tokens=int(num_external_tokens))
        self._pending_pulls[request.request_id] = PullSpec(
            req_id=request.request_id, remote_engine_id=str(p["remote_engine_id"]),
            remote_request_id=str(p.get("remote_request_id") or request.request_id),
            remote_block_ids=first_group(p["remote_block_ids"]), local_block_ids=list(local_block_ids),
            n_tokens=num_computed_tokens + num_external_tokens,
            skip_tokens=num_computed_tokens // self.block_size * self.block_size,
            remote_lease_id=str(p.get("remote_lease_id") or ""))

    # ---- producer -------------------------------------------------------------------------
    def request_finished(self, request, block_ids: list[int], finished_ok: bool = True):
        """(delay_free, kv_transfer_params) for a request that ran with do_remote_decode."""
        p = getattr(request, "kv_transfer_params", None)
        if not p or not p.get("do_remote_decode") or not finished_ok or not block_ids:
            return False, None
        deadline = time.monotonic() + self.lease_s
        self._held[request.request_id] = deadline
        self._new_held[request.request_id] = deadline
        n_tok = getattr(request, "num_computed_tokens", None)
        if n_tok is None:
            n_tok = len(request.prompt_token_ids or [])
        lease_id = f"{_safe(request.request_id)[:64]}.{time.time_ns():x}"
        try:       # the lease exists before anybody can learn the block ids
            lp = lease_path(self.engine_id, lease_id)
            os.makedirs(os.path.dirname(lp), exist_ok=True)
            with open(lp, "w"):
                pass
            self._leases[request.request_id] = lease_id
        except OSError:
            lease_id = ""          # no lease file: consumers skip the check (as before), the deadline still frees
        trace("prefill_finished", req=request.request_id, tokens=int(n_tok))
        return True, dict(do_remote_prefill=True, do_remote_decode=False, remote_block_ids=list(block_ids),
                          remote_engine_id=self.engine_id, remote_request_id=request.request_id,
                          remote_host=None, remote_port=None, tp_size=self.tp_size, remote_num_tokens=int(n_tok),
                          remote_lease_id=lease_id)

    def build_meta(self) -> PDMeta:
        m = PDMeta(list(self._pending_pulls.values()), dict(self._new_held))
        self._pending_pulls.clear()
        self._new_held.clear()
        return m

    def sending_finished(self, req_ids):
        """Every worker rank reported the request (pulled, or lease expired).  Called right BEFORE vLLM frees
        the blocks: the lease disappears first, so no consumer can validate a pull against recycled pages."""
        for r in req_ids or ():
            self._held.pop(r, None)
            lease = self._leases.pop(r, None)
            if lease:
                try:
                    os.unlink(lease_path(self.engine_id, lease))
                except OSError:
                    pass

    def close(self):
        self.sending_finished(list(self._leases))
        try:
            os.rmdir(os.path.dirname(lease_path(self.engine_id, "x")))
        except OSError:
            pass


def first_group(block_ids):
    if block_ids and isinstance(block_ids[0], (list, tuple)):
        return list(block_ids[0])
    return list(block_ids or [])


# ------------------------------------------------------------------------------------------------
# worker-role state
# ------------------------------------------------------------------------------------------------
class PDWorker:
    def __init__(self, engine, engine_id: str, block_size: int, resolver=None, rank: int = 0, tp_size: int = 1):
        self.engine = engine
        self.engine_id = engine_id
        self.block_size = block_size
        self.rank = rank
        self.resolver = resolver or PeerResolver(engine, rank=rank, tp_size=tp_size)
        self._inflight: list[tuple[int, PullSpec]] = []   # (ticket, spec)
        self._held: dict[str, float] = {}
        self.failed_blocks: set[int] = set()
        self.n_pulled_tokens = 0
        self.n_lease_failures = 0

    @staticmethod
    def _lease_alive(spec: PullSpec) -> bool:
        return not spec.remote_lease_id or os.path.exists(lease_path(spec.remote_engine_id, spec.remote_lease_id))

    def start_pulls(self, meta: PDMeta, stream=None):
        self._held.update(meta.held)
        for spec in meta.pulls:
            try:
                n = min(spec.n_tokens, len(spec.remote_block_ids) * self.block_size)
                if len(spec.local_block_ids) * self.block_size < n:
                    # fewer local pages than tokens promised to the scheduler: never decode on what was not loaded
                    raise ValueError(f"{len(spec.local_block_ids)} local blocks for {n} external tokens")
                if not self._lease_alive(spec):
                    self.n_lease_failures += 1
                    raise TimeoutError("the producer's lease on the blocks has expired")
                peer = self.resolver.resolve(spec.remote_engine_id)
                src = slots_of(spec.remote_block_ids, self.block_size, n)[spec.skip_tokens:]
                dst = slots_of(spec.local_block_ids, self.block_size, n)[spec.skip_tokens:]
                if len(src) == 0:
                    self._notify_done(spec)
                    continue
                trace("pull_issued", req=spec.req_id, tokens=int(len(src)), rank=self.rank)
                ticket = self.engine.peer_pull(peer, src, dst, stream=stream)
                self._inflight.append((ticket, spec))
                self.n_pulled_tokens += len(src)
            except Exception as e:
                # no exception on the data path: vLLM recomputes the blocks we report
                trace("pull_failed", req=spec.req_id, error=repr(e), rank=self.rank)
                self.failed_blocks.update(spec.local_block_ids)
                self._notify_done(spec)

    def _notify_done(self, spec: PullSpec):
        d = done_dir(spec.remote_engine_id, self.rank)
        try:
            os.makedirs(d, exist_ok=True)
            with open(os.path.join(d, _safe(spec.remote_request_id)), "w"):
                pass
        except OSError:
            pass  # the producer's lease will expire instead

    def poll(self, block: bool = False) -> tuple[set[str], set[str]]:
        """-> (finished_sending, finished_recving) request ids for get_finished().  block=True (what the
        connector uses): wait for this step's pulls — they precede the forward pass in stream order, so this
        costs the pull itself — so that a pull invalidated by an expired lease is reported as load errors in
        the SAME step (get_block_ids_with_load_errors follows get_finished)."""
        recv_done, still = set(), []
        for ticket, spec in self._inflight:
            if block:
                self.engine.wait(ticket)
            if block or self.engine.poll(ticket):
                if not self._lease_alive(spec):     # freed (and maybe recycled) while we were reading
                    self.n_lease_failures += 1
                    self.failed_blocks.update(spec.local_block_ids)
                    trace("pull_invalidated", req=spec.req_id, rank=self.rank)
                else:
                    trace("pull_done", req=spec.req_id, rank=self.rank)
                self._notify_done(spec)
                recv_done.add(spec.req_id)
            else:
                still.append((ticket, spec))
        self._inflight = still
        send_done = set()
        if self._held:
            d = done_dir(self.engine_id, self.rank)
            try:
                marks = set(os.listdir(d))
            except OSError:
                marks = set()
            now = time.monotonic()
            for rid, deadline in list(self._held.items()):
                if _safe(rid) in marks or now > deadline:
                    send_done.add(rid)
                    self._held.pop(rid)
                    try:
                        os.unlink(os.path.join(d, _safe(rid)))     # this rank's own marker directory
                    except OSError:
                        pass
        return send_done, recv_done

    def take_failed_blocks(self) -> set[int]:
        f, self.failed_blocks = self.failed_blocks, set()
        return f
