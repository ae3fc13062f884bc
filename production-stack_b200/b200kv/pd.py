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
    in /dev/shm/b200kv-ipc-<engine_id>.r<rank>.json (b200kv_export_ipc), with the model's total KV-head count;
    at the same tensor-parallel size (`tp_size` in the params) decode rank r pulls from prefill rank r;
  * at different sizes each decode rank pulls its KV heads from the prefill ranks that hold them.  vLLM shards
    T KV heads over t ranks (QKVParallelLinear): rank r holds H = max(1, T // t) heads, global heads
    [r*H, (r+1)*H) when T >= t, else head r // (t / T), replicated t / T times.  For every local head the
    first prefill rank holding it is the source; per (decode rank, prefill rank) pair that is one contiguous
    head slice (head_slices), pulled by the head-slice kernel (b200kv_import_peer_sliced).  An MLA latent (and
    V3.2's indexer plane) is the same on every rank: decode rank c pulls whole pages from prefill rank c % t_p;
  * the producer keeps a finished request's blocks (`delay_free=True`) until every consumer rank dropped
    a marker /dev/shm/b200kv-done-<producer_engine_id>.r<rank>/<request_id>, or a lease expires.  When
    the sizes differ, decode rank c of t_d drops <request_id>.d<c>of<t_d> into the marker directory of EVERY
    prefill rank, also of those it read nothing from, and a prefill rank releases the request once it holds
    all t_d of them;
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
import logging
import os
import re
import time
from dataclasses import dataclass, field

import numpy as np

from ._lib import DTYPE_BF16, LAYOUT_MLA

SHM_DIR = os.environ.get("B200KV_SHM_DIR", "/dev/shm")
logger = logging.getLogger("b200kv")


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
    """The cache element type of a geometry (KVGeometry.cache_dtype, else its dtype; bf16 for a geometry without
    either)."""
    return int(getattr(geom, "cache_dtype", getattr(geom, "dtype", DTYPE_BF16)))


def _indexer_of(geom) -> int:
    """Bytes per token of a geometry's indexer planes (KVGeometry.idx_token_bytes; 0 = none)."""
    return int(getattr(geom, "idx_token_bytes", 0))


def _draft_of(geom) -> int:
    """Draft layers among a geometry's layers (KVGeometry.draft_layers; 0 for a geometry without the field)."""
    return int(getattr(geom, "draft_layers", 0))


def publish_ipc(engine_id: str, engine, device: int, rank: int = 0, tp_size: int = 1, total_kv_heads: int = 0) -> str:
    """total_kv_heads: the model's KV heads over all ranks (model_config.get_total_num_kv_heads()).  A document
    without it pairs with consumers of its own tensor-parallel size only."""
    g = engine.geom
    doc = {"engine_id": engine_id, "device": device, "pid": os.getpid(), "rank": rank, "tp_size": tp_size,
           **({"total_kv_heads": int(total_kv_heads)} if total_kv_heads else {}),
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


# ------------------------------------------------------------------------------------------------
# the head map of a pairing of different tensor-parallel sizes
# ------------------------------------------------------------------------------------------------
def shardable(total_kv_heads: int, tp_size: int) -> bool:
    """vLLM can shard T KV heads over t ranks: t divides T, or T divides t (replication)."""
    T, t = int(total_kv_heads), int(tp_size)
    return T > 0 and t > 0 and (T % t == 0 if T >= t else t % T == 0)


def heads_of_rank(total_kv_heads: int, tp_size: int, rank: int) -> list[int]:
    """Global KV heads that tensor-parallel rank `rank` of `tp_size` holds, in local order (QKVParallelLinear)."""
    T, t = total_kv_heads, tp_size
    if T >= t:
        H = T // t
        return list(range(rank * H, (rank + 1) * H))
    return [rank // (t // T)]


def head_slices(total_kv_heads: int, producer_tp: int, consumer_tp: int, consumer_rank: int):
    """[(producer rank, (peer_heads, src_head0, dst_head0, n_heads))] for consumer rank `consumer_rank`, producer
    ranks ascending: each local head is read from the first producer rank that holds it, and the heads read from one
    producer rank are one contiguous slice on both sides.  ValueError if a size cannot shard the heads."""
    T = int(total_kv_heads)
    for t in (producer_tp, consumer_tp):
        if not shardable(T, t):
            raise ValueError(f"{T} KV heads cannot be sharded over {t} tensor-parallel ranks")
    H_p = max(1, T // producer_tp)
    by_rank: dict[int, list[tuple[int, int]]] = {}
    for h, g in enumerate(heads_of_rank(T, consumer_tp, consumer_rank)):
        p, src = (g // H_p, g % H_p) if T >= producer_tp else (g * (producer_tp // T), 0)
        by_rank.setdefault(p, []).append((src, h))
    out = []
    for p in sorted(by_rank):
        (src0, dst0), n = by_rank[p][0], len(by_rank[p])
        if by_rank[p] != [(src0 + i, dst0 + i) for i in range(n)]:
            raise ValueError(f"heads of producer rank {p} are not one contiguous slice: {by_rank[p]}")
        out.append((p, (H_p, src0, dst0, n)))
    return out


class PeerResolver:
    """remote engine_id -> peer_id of this engine; maps the peer's cache on first use.  A remote engine of another
    tensor-parallel size maps as one peer per producer rank this rank reads from (sources)."""

    def __init__(self, engine, max_peers: int = 64, rank: int = 0, tp_size: int = 1, total_kv_heads: int = 0):
        self.engine = engine
        self.ids: dict = {}     # remote engine_id (same size), or (engine_id, producer rank) -> peer_id
        self.max_peers = max_peers
        self.rank, self.tp_size = rank, tp_size
        self.total_kv_heads = int(total_kv_heads)
        self._sources: dict[str, list] = {}

    def sources(self, remote_engine_id: str, remote_tp_size: int) -> list[tuple[int, tuple | None]]:
        """[(peer_id, head slice or None)] to pull from for a request prefilled by `remote_engine_id` at tensor-parallel
        size `remote_tp_size`: [(resolve(), None)] at this rank's size; else one source per producer rank read."""
        if remote_tp_size == self.tp_size:
            return [(self.resolve(remote_engine_id), None)]
        src = self._sources.get(remote_engine_id)
        if src is not None:
            return src
        g = self.engine.geom
        if getattr(g, "layout", 0) == LAYOUT_MLA:
            pairs = [(self.rank % remote_tp_size, None)]     # the latent is the same on every rank
        elif not self.total_kv_heads:
            raise ValueError(f"peer {remote_engine_id}: tensor-parallel size {remote_tp_size} differs from local "
                             f"{self.tp_size} and the local total KV-head count is not known")
        elif g.n_kv_heads != max(1, self.total_kv_heads // self.tp_size):
            raise ValueError(f"local cache holds {g.n_kv_heads} KV heads, {self.total_kv_heads} heads over "
                             f"{self.tp_size} ranks imply {max(1, self.total_kv_heads // self.tp_size)}")
        else:
            pairs = head_slices(self.total_kv_heads, remote_tp_size, self.tp_size, self.rank)
        src = []
        for p, sl in pairs:
            pid = self.ids.get((remote_engine_id, p))
            if pid is None:
                doc = self._doc(remote_engine_id, p, remote_tp_size)
                if sl is None:
                    self._check(remote_engine_id, doc, "n_kv_heads", g.n_kv_heads)
                else:
                    if int(doc.get("total_kv_heads", 0)) != self.total_kv_heads:
                        raise ValueError(f"peer {remote_engine_id}.r{p}: total_kv_heads={doc.get('total_kv_heads')} "
                                         f"differs from local {self.total_kv_heads} (a replica that does not publish it "
                                         "pairs at its own tensor-parallel size only)")
                    self._check(remote_engine_id, doc, "n_kv_heads", sl[0])   # the head map's per-rank count
                pid = self._import((remote_engine_id, p), doc, sl)
            src.append((pid, sl))
        self._sources[remote_engine_id] = src
        logger.info("b200kv P/D: engine %s at tensor-parallel size %d pairs with local rank %d of %d: %s",
                    remote_engine_id, remote_tp_size, self.rank, self.tp_size,
                    ", ".join(f"rank {p} " + ("whole pages" if sl is None else
                                              f"heads [{sl[1]}, {sl[1] + sl[3]}) -> [{sl[2]}, {sl[2] + sl[3]})")
                              for p, sl in pairs))
        return src

    def _doc(self, remote_engine_id: str, rank: int, tp_size: int) -> dict:
        with open(ipc_path(remote_engine_id, rank)) as f:
            doc = json.load(f)
        if int(doc.get("tp_size", 1)) != tp_size or int(doc.get("rank", 0)) != rank:
            raise ValueError(f"peer {remote_engine_id}: tensor-parallel layout {doc.get('rank')}/{doc.get('tp_size')} "
                             f"differs from the expected {rank}/{tp_size}")
        return doc

    def _import(self, key, doc: dict, head_slice) -> int:
        pid = len(self.ids)
        if pid >= self.max_peers:
            raise RuntimeError("too many peers")
        descs = base64.b64decode(doc["descs"])
        if head_slice is None:
            self.engine.import_peer(pid, doc["device"], descs, doc["block_stride"], doc["n_blocks"])
        else:
            self.engine.import_peer(pid, doc["device"], descs, doc["block_stride"], doc["n_blocks"],
                                    head_slice=head_slice)
        self.ids[key] = pid
        return pid

    def resolve(self, remote_engine_id: str) -> int:
        pid = self.ids.get(remote_engine_id)
        if pid is not None:
            return pid
        with open(ipc_path(remote_engine_id, self.rank)) as f:    # the SAME rank's shard of the peer engine
            doc = json.load(f)
        if int(doc.get("tp_size", 1)) != self.tp_size or int(doc.get("rank", 0)) != self.rank:
            raise ValueError(f"peer {remote_engine_id}: tensor-parallel layout {doc.get('rank')}/{doc.get('tp_size')} "
                             f"differs from local {self.rank}/{self.tp_size}")
        self._check(remote_engine_id, doc, "n_kv_heads", self.engine.geom.n_kv_heads)
        return self._import(remote_engine_id, doc, None)

    def _check(self, remote_engine_id: str, doc: dict, heads_key: str, heads: int):
        """The peer's cache has this engine's geometry; heads_key names the head count compared."""
        g = self.engine.geom
        doc.setdefault("dtype", DTYPE_BF16)   # documents published before the field are bf16 caches (e4m3 on 1-byte ones)
        doc.setdefault("indexer", 0)          # ... and caches without indexer planes
        doc.setdefault("draft_layers", 0)     # ... and replicas without a speculative-decoding drafter
        if (doc["n_layers"], doc["draft_layers"]) != (g.n_layers, _draft_of(g)):
            # a drafter's layers follow the target's in the cache: the pages of a replica with one are not those of
            # a replica without one (or with another drafter)
            raise ValueError(f"peer {remote_engine_id}: n_layers={doc['n_layers']} with {doc['draft_layers']} draft "
                             f"layer(s) differs from local {g.n_layers} with {_draft_of(g)}: replicas pair only "
                             "with the same speculative-decoding drafter, or both without one")
        for k, mine in ((heads_key, heads), ("head_dim", g.head_dim),
                        ("block_tokens", g.block_tokens), ("elem_bytes", g.elem_bytes), ("layout", g.layout),
                        ("dtype", _dtype_of(g)), ("indexer", _indexer_of(g))):
            if doc[k] != mine:
                raise ValueError(f"peer {remote_engine_id}: {k}={doc[k]} differs from local {mine}")


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
    remote_tp_size: int = 0     # the producer's tensor-parallel size (`tp_size` in the params); 0: the consumer's


@dataclass
class PDMeta:
    pulls: list[PullSpec] = field(default_factory=list)
    # producer: request ids whose blocks are held for a consumer, with their lease deadline
    held: dict[str, float] = field(default_factory=dict)


class PDScheduler:
    def __init__(self, engine_id: str, block_size: int, lease_s: float = 120.0, tp_size: int = 1,
                 blocks_known_at_alloc: bool = True, total_kv_heads: int = 0, mla: bool = False):
        self.engine_id = engine_id
        self.block_size = block_size
        self.lease_s = lease_s
        self.tp_size = tp_size
        # the model's head geometry: with it, a producer of another tensor-parallel size is paired (module docstring);
        # without it such a request is declined
        self.total_kv_heads, self.mla = int(total_kv_heads), bool(mla)
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
        if not self.blocks_known_at_alloc or not self.pairs_with(int(p.get("tp_size") or 1)):
            return None      # cannot pull (see __init__ / unpairable tensor-parallel layout): ordinary request
        n_prompt = len(request.prompt_token_ids or [])
        n_remote = min(int(p.get("remote_num_tokens") or n_prompt), n_prompt,
                       len(first_group(p["remote_block_ids"])) * self.block_size)
        # the last prompt token is recomputed locally (same rule as a full pool hit)
        return max(min(n_remote, n_prompt - 1) - num_computed_tokens, 0)

    def pairs_with(self, remote_tp_size: int) -> bool:
        """A producer at tensor-parallel size remote_tp_size can hand its KV to this consumer."""
        if remote_tp_size == self.tp_size:
            return True
        if self.mla:
            return remote_tp_size > 0
        return shardable(self.total_kv_heads, remote_tp_size) and shardable(self.total_kv_heads, self.tp_size)

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
            remote_lease_id=str(p.get("remote_lease_id") or ""), remote_tp_size=int(p.get("tp_size") or 1))

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


_SPLIT = re.compile(r"(.+)\.d(\d+)of(\d+)")


def split_marker(request_id: str, consumer_rank: int, consumer_tp: int) -> str:
    """Marker of consumer rank `consumer_rank` of `consumer_tp` in a pairing of different tensor-parallel sizes."""
    return f"{_safe(request_id)}.d{int(consumer_rank)}of{int(consumer_tp)}"


def split_markers(names) -> dict[str, dict[int, set[int]]]:
    """Marker file names -> {request id: {consumer tp size: consumer ranks that dropped a marker}}."""
    out: dict[str, dict[int, set[int]]] = {}
    for name in names:
        m = _SPLIT.fullmatch(name)
        if m and int(m.group(2)) < int(m.group(3)):
            out.setdefault(m.group(1), {}).setdefault(int(m.group(3)), set()).add(int(m.group(2)))
    return out


def released(ranks_by_tp: dict[int, set[int]]) -> bool:
    """Every consumer rank of some tensor-parallel size has dropped its marker."""
    return any(len(cs) == n for n, cs in ranks_by_tp.items())


def first_group(block_ids):
    if block_ids and isinstance(block_ids[0], (list, tuple)):
        return list(block_ids[0])
    return list(block_ids or [])


# ------------------------------------------------------------------------------------------------
# worker-role state
# ------------------------------------------------------------------------------------------------
class PDWorker:
    def __init__(self, engine, engine_id: str, block_size: int, resolver=None, rank: int = 0, tp_size: int = 1,
                 total_kv_heads: int = 0):
        self.engine = engine
        self.engine_id = engine_id
        self.block_size = block_size
        self.rank, self.tp_size = rank, tp_size
        self.resolver = resolver or PeerResolver(engine, rank=rank, tp_size=tp_size, total_kv_heads=total_kv_heads)
        self._inflight: list[tuple[list[int], PullSpec]] = []   # (tickets, spec): one pull per source
        self._held: dict[str, float] = {}
        self.failed_blocks: set[int] = set()
        self.n_pulled_tokens = 0
        self.n_lease_failures = 0

    @staticmethod
    def _lease_alive(spec: PullSpec) -> bool:
        return not spec.remote_lease_id or os.path.exists(lease_path(spec.remote_engine_id, spec.remote_lease_id))

    def _mismatched(self, spec: PullSpec) -> bool:
        return bool(spec.remote_tp_size) and spec.remote_tp_size != self.tp_size

    def start_pulls(self, meta: PDMeta, stream=None):
        """One pull per source of each request, on `stream`.  The lease is checked before the first and (poll) after
        the last; a request any of whose pulls cannot be issued has all its local blocks reported."""
        self._held.update(meta.held)
        for spec in meta.pulls:
            tickets: list[int] = []
            try:
                n = min(spec.n_tokens, len(spec.remote_block_ids) * self.block_size)
                if len(spec.local_block_ids) * self.block_size < n:
                    # fewer local pages than tokens promised to the scheduler: never decode on what was not loaded
                    raise ValueError(f"{len(spec.local_block_ids)} local blocks for {n} external tokens")
                if not self._lease_alive(spec):
                    self.n_lease_failures += 1
                    raise TimeoutError("the producer's lease on the blocks has expired")
                if self._mismatched(spec):
                    peers = [pid for pid, _ in self.resolver.sources(spec.remote_engine_id, spec.remote_tp_size)]
                else:
                    peers = [self.resolver.resolve(spec.remote_engine_id)]
                src = slots_of(spec.remote_block_ids, self.block_size, n)[spec.skip_tokens:]
                dst = slots_of(spec.local_block_ids, self.block_size, n)[spec.skip_tokens:]
                if len(src) == 0:
                    self._notify_done(spec)
                    continue
                trace("pull_issued", req=spec.req_id, tokens=int(len(src)), rank=self.rank)
                for peer in peers:
                    tickets.append(self.engine.peer_pull(peer, src, dst, stream=stream))
                self._inflight.append((tickets, spec))
                self.n_pulled_tokens += len(src)
            except Exception as e:
                # no exception on the data path: vLLM recomputes the blocks we report
                trace("pull_failed", req=spec.req_id, error=repr(e), rank=self.rank)
                for t in tickets:      # pulls already issued read the producer's pages until they finish
                    self.engine.wait(t)
                self.failed_blocks.update(spec.local_block_ids)
                self._notify_done(spec)

    def _notify_done(self, spec: PullSpec):
        if self._mismatched(spec):    # every producer rank waits for every consumer rank
            marks = [(done_dir(spec.remote_engine_id, p), split_marker(spec.remote_request_id, self.rank, self.tp_size))
                     for p in range(spec.remote_tp_size)]
        else:
            marks = [(done_dir(spec.remote_engine_id, self.rank), _safe(spec.remote_request_id))]
        for d, name in marks:
            try:
                os.makedirs(d, exist_ok=True)
                with open(os.path.join(d, name), "w"):
                    pass
            except OSError:
                pass  # the producer's lease will expire instead

    def poll(self, block: bool = False) -> tuple[set[str], set[str]]:
        """-> (finished_sending, finished_recving) request ids for get_finished().  block=True (what the
        connector uses): wait for this step's pulls — they precede the forward pass in stream order, so this
        costs the pull itself — so that a pull invalidated by an expired lease is reported as load errors in
        the SAME step (get_block_ids_with_load_errors follows get_finished)."""
        recv_done, still = set(), []
        for tickets, spec in self._inflight:
            if block:
                for t in tickets:
                    self.engine.wait(t)
            if block or all(self.engine.poll(t) for t in tickets):
                if not self._lease_alive(spec):     # freed (and maybe recycled) while we were reading
                    self.n_lease_failures += 1
                    self.failed_blocks.update(spec.local_block_ids)
                    trace("pull_invalidated", req=spec.req_id, rank=self.rank)
                else:
                    trace("pull_done", req=spec.req_id, rank=self.rank)
                self._notify_done(spec)
                recv_done.add(spec.req_id)
            else:
                still.append((tickets, spec))
        self._inflight = still
        send_done = set()
        if self._held:
            d = done_dir(self.engine_id, self.rank)
            try:
                marks = set(os.listdir(d))
            except OSError:
                marks = set()
            split = split_markers(marks)
            now = time.monotonic()
            for rid, deadline in list(self._held.items()):
                sid = _safe(rid)
                if sid in marks or released(split.get(sid, {})) or now > deadline:
                    send_done.add(rid)
                    self._held.pop(rid)
                    for name in [sid] + [split_marker(rid, c, n) for n, cs in split.get(sid, {}).items() for c in cs]:
                        try:
                            os.unlink(os.path.join(d, name))     # this rank's own marker directory
                        except OSError:
                            pass
        return send_done, recv_done

    def take_failed_blocks(self) -> set[int]:
        f, self.failed_blocks = self.failed_blocks, set()
        return f
