"""Cross-replica plumbing: exchange the CUDA-IPC descriptors of every replica's paged cache once,
then any replica can `peer_pull` blocks straight out of another replica's HBM over NVSwitch.

Replaces the NIXL/UCX side channel the reference configures (LMCACHE_NIXL_RECEIVER_HOST/PORT,
helm/templates/deployment-vllm-multi.yaml:296-324).  torch.distributed (gloo or nccl) is used for
the one-off handshake only — there is no collective on the data path (SURVEY.md §8e).
"""
from __future__ import annotations

import torch.distributed as dist


def all_gather_bytes(payload: bytes, group=None) -> list[bytes]:
    world = dist.get_world_size(group)
    out: list = [None] * world
    dist.all_gather_object(out, payload, group=group)
    return [bytes(x) for x in out]


def exchange_kv_descriptors(engine, group=None) -> list[bytes]:
    """Every rank exports its descriptors (b200kv_export_ipc, KVGeometry.n_descs of them); returns them indexed by
    rank."""
    return all_gather_bytes(engine.export_ipc(), group)


def connect_all_peers(engine, descs_by_rank: list[bytes], my_rank: int, device_of_rank=None) -> list[int]:
    """Map every other rank's cache into this process (b200kv_import_peer); peer_id == rank."""
    connected = []
    for r, d in enumerate(descs_by_rank):
        if r == my_rank:
            continue
        engine.import_peer(r, device_of_rank(r) if device_of_rank else r, d)
        connected.append(r)
    return connected


def shard_sessions(n_sessions: int, rank: int, world: int) -> range:
    """Requests are the unit of partition (router: round-robin / session hash); contiguous split."""
    per = (n_sessions + world - 1) // world
    return range(min(rank * per, n_sessions), min((rank + 1) * per, n_sessions))
