"""Disaggregated prefill between replicas of different tensor-parallel sizes (CPU, fake engine): the head map, the
resolver's sources and refusals, the done markers, and the scheduler's pairing rule."""
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest

from b200kv import _lib, pd

BS = 16


def shard(T, t):
    """Brute force of vLLM's KV-head sharding: rank -> global heads, built head by head."""
    owners = {r: [] for r in range(t)}
    if T >= t:
        for g in range(T):
            owners[g // (T // t)].append(g)
    else:
        for r in range(t):
            owners[r].append(r * T // t)
    return owners


GRID = [(T, t_p, t_d) for T in (1, 2, 4, 8, 16) for t_p in range(1, 9) for t_d in range(1, 9)
        if t_p != t_d and pd.shardable(T, t_p) and pd.shardable(T, t_d)]


def test_grid_covers_both_directions_and_replication_on_either_side():
    assert len(GRID) > 80
    assert any(t_p < t_d for _, t_p, t_d in GRID) and any(t_p > t_d for _, t_p, t_d in GRID)
    assert any(T < t_d and T >= t_p for T, t_p, t_d in GRID)      # replicated on the consumer side only
    assert any(T < t_p and T >= t_d for T, t_p, t_d in GRID)      # ... on the producer side only
    assert any(T < t_p and T < t_d for T, t_p, t_d in GRID)       # ... on both


@pytest.mark.parametrize("T,t_p,t_d", GRID)
def test_head_map_matches_brute_force(T, t_p, t_d):
    prod, cons = shard(T, t_p), shard(T, t_d)
    for t, owners in ((t_p, prod), (t_d, cons)):
        for r in range(t):
            assert pd.heads_of_rank(T, t, r) == owners[r]
    for c in range(t_d):
        # per head: the first producer rank holding it, and the head's place there
        want = {}
        for h, g in enumerate(cons[c]):
            p = min(r for r in range(t_p) if g in prod[r])
            want[h] = (p, prod[p].index(g))
        slices = pd.head_slices(T, t_p, t_d, c)
        got = {}
        ranks = [p for p, _ in slices]
        assert ranks == sorted(set(ranks))                       # at most one slice per producer rank
        for p, (hp, s0, d0, n) in slices:
            assert hp == len(prod[p]) == max(1, T // t_p) and n >= 1
            assert 0 <= s0 and s0 + n <= hp and 0 <= d0 and d0 + n <= len(cons[c])
            for i in range(n):
                assert d0 + i not in got
                got[d0 + i] = (p, s0 + i)
        assert got == want


def test_unshardable_sizes_are_refused():
    for T, t in ((8, 3), (6, 4), (2, 3), (0, 1)):
        assert not pd.shardable(T, t)
    with pytest.raises(ValueError):
        pd.head_slices(8, 3, 2, 0)


# ------------------------------------------------------------------------------------------------
class FakeEngine:
    def __init__(self, H=4, layout=0, fail_import_of=None):
        self.geom = NS(n_blocks=64, stride=BS * H * 128 * 2, n_layers=2, n_kv_heads=H, head_dim=128, block_tokens=BS,
                       elem_bytes=2, layout=layout)
        self.imported, self.pulls, self.waited, self.done = [], [], [], set()
        self.fail_import_of = fail_import_of

    def export_ipc(self):
        return b"\x07" * (72 * 4)

    def import_peer(self, pid, device, descs, stride, n_blocks, head_slice=None):
        if device == self.fail_import_of:
            raise RuntimeError("peer unreachable")
        self.imported.append((pid, device, stride, n_blocks, head_slice))

    def peer_pull(self, peer, src, dst, stream=None):
        self.pulls.append((peer, np.asarray(src).copy(), np.asarray(dst).copy()))
        return len(self.pulls)

    def poll(self, ticket):
        return ticket in self.done

    def wait(self, ticket):
        self.waited.append(ticket)
        self.done.add(ticket)


@pytest.fixture
def shm(tmp_path, monkeypatch):
    monkeypatch.setattr(pd, "SHM_DIR", str(tmp_path))
    return tmp_path


def publish(eid, T, tp, layout=0, with_total=True, **over):
    for r in range(tp):
        e = FakeEngine(max(1, T // tp) if layout != _lib.LAYOUT_MLA else 1, layout)
        e.geom.__dict__.update(over)
        pd.publish_ipc(eid, e, device=r, rank=r, tp_size=tp, total_kv_heads=T if with_total else 0)


def test_resolver_sources(shm):
    publish("P", 8, 2)
    d = FakeEngine(H=2)
    r = pd.PeerResolver(d, rank=1, tp_size=4, total_kv_heads=8)
    assert r.sources("P", 2) == [(0, (4, 2, 0, 2))]          # heads 2, 3 sit on prefill rank 0 at 2, 3
    assert d.imported == [(0, 0, BS * 4 * 128 * 2, 64, (4, 2, 0, 2))]
    assert r.sources("P", 2) == [(0, (4, 2, 0, 2))] and len(d.imported) == 1    # mapped once
    d1 = FakeEngine(H=8)
    r1 = pd.PeerResolver(d1, rank=0, tp_size=1, total_kv_heads=8)
    assert r1.sources("P", 2) == [(0, (4, 0, 0, 4)), (1, (4, 0, 4, 4))]
    assert [i[1] for i in d1.imported] == [0, 1] and r1.ids == {("P", 0): 0, ("P", 1): 1}
    # the same size takes the unchanged path: the same rank's document, no slice
    publish("Q", 8, 4)
    d4 = FakeEngine(H=2)
    assert pd.PeerResolver(d4, rank=3, tp_size=4, total_kv_heads=8).sources("Q", 4) == [(0, None)]
    assert d4.imported == [(0, 3, BS * 2 * 128 * 2, 64, None)]


def test_resolver_refusals(shm):
    publish("old", 8, 2, with_total=False)
    with pytest.raises(ValueError, match="total_kv_heads"):   # a document without the field: its own size only
        pd.PeerResolver(FakeEngine(H=2), rank=0, tp_size=4, total_kv_heads=8).sources("old", 2)
    publish("P16", 16, 2)
    with pytest.raises(ValueError, match="total_kv_heads"):
        pd.PeerResolver(FakeEngine(H=2), rank=0, tp_size=4, total_kv_heads=8).sources("P16", 2)
    publish("Pd", 8, 2, head_dim=64)
    with pytest.raises(ValueError, match="head_dim"):
        pd.PeerResolver(FakeEngine(H=2), rank=0, tp_size=4, total_kv_heads=8).sources("Pd", 2)
    publish("P", 8, 2)
    with pytest.raises(ValueError, match="not known"):
        pd.PeerResolver(FakeEngine(H=2), rank=0, tp_size=4).sources("P", 2)
    with pytest.raises(ValueError):                            # this rank does not hold the heads the map implies
        pd.PeerResolver(FakeEngine(H=4), rank=0, tp_size=4, total_kv_heads=8).sources("P", 2)
    with pytest.raises(RuntimeError, match="too many peers"):  # max_peers counts (engine, producer rank) pairs
        pd.PeerResolver(FakeEngine(H=8), max_peers=1, rank=0, tp_size=1, total_kv_heads=8).sources("P", 2)
    with pytest.raises(FileNotFoundError):
        pd.PeerResolver(FakeEngine(H=2), rank=0, tp_size=4, total_kv_heads=8).sources("nowhere", 2)


@pytest.mark.parametrize("t_p,t_d", [(4, 2), (2, 8), (1, 4), (4, 1)])
def test_mla_source_is_rank_c_mod_tp(shm, t_p, t_d):
    publish("M", 1, t_p, layout=_lib.LAYOUT_MLA)
    for c in range(t_d):
        d = FakeEngine(H=1, layout=_lib.LAYOUT_MLA)
        assert pd.PeerResolver(d, rank=c, tp_size=t_d).sources("M", t_p) == [(0, None)]
        assert d.imported[0][1] == c % t_p and d.imported[0][4] is None     # whole pages, unsliced


# ------------------------------------------------------------------------------------------------
def test_scheduler_pairs_other_sizes_only_with_head_geometry():
    req = lambda tp: NS(request_id="x", prompt_token_ids=list(range(40)),      # noqa: E731
                        kv_transfer_params={"do_remote_prefill": True, "remote_engine_id": "P",
                                            "remote_block_ids": [[1, 2, 3]], "tp_size": tp})
    assert pd.PDScheduler("D", BS, tp_size=2).remote_prefill_tokens(req(1), 0) is None      # declines, as before
    s = pd.PDScheduler("D", BS, tp_size=2, total_kv_heads=8)
    assert s.remote_prefill_tokens(req(1), 0) == 39
    s.after_alloc(req(1), [4, 5, 6], 39, 0)
    assert s.build_meta().pulls[0].remote_tp_size == 1
    assert pd.PDScheduler("D", BS, tp_size=2, total_kv_heads=8).remote_prefill_tokens(req(3), 0) is None
    assert pd.PDScheduler("D", BS, tp_size=2, total_kv_heads=1).remote_prefill_tokens(req(4), 0) == 39
    assert pd.PDScheduler("D", BS, tp_size=2, mla=True).remote_prefill_tokens(req(8), 0) == 39
    assert pd.PDScheduler("D", BS, tp_size=2, total_kv_heads=8,
                          blocks_known_at_alloc=False).remote_prefill_tokens(req(1), 0) is None


def test_publish_writes_total_kv_heads_only_when_known(shm):
    import json
    publish("A", 8, 1)
    publish("B", 8, 1, with_total=False)
    assert json.load(open(pd.ipc_path("A")))["total_kv_heads"] == 8
    assert "total_kv_heads" not in json.load(open(pd.ipc_path("B")))


# ------------------------------------------------------------------------------------------------
def spec(rid="p-req", t_p=2, lease=""):
    return pd.PullSpec("d-" + rid, "P", rid, [10, 11, 12, 13], [1, 2, 3, 4], 60, remote_lease_id=lease,
                       remote_tp_size=t_p)


def test_worker_pulls_every_source_and_marks_every_producer_rank(shm):
    publish("P", 8, 4)
    d = FakeEngine(H=8)
    w = pd.PDWorker(d, "D", BS, rank=0, tp_size=1, total_kv_heads=8)
    w.start_pulls(pd.PDMeta([spec(t_p=4)], {}))
    assert [p for p, _, _ in d.pulls] == [0, 1, 2, 3]
    assert all(np.array_equal(s, d.pulls[0][1]) and np.array_equal(t, d.pulls[0][2]) for _, s, t in d.pulls)
    assert w.poll() == (set(), set())                          # one source still in flight
    d.done.update({1, 2, 3})
    assert w.poll() == (set(), set())
    d.done.add(4)
    assert w.poll() == (set(), {"d-p-req"}) and w.take_failed_blocks() == set()
    for p in range(4):
        assert os.listdir(pd.done_dir("P", p)) == ["p-req.d0of1"]


def test_a_failed_source_fails_the_whole_request(shm):
    publish("P", 8, 2)
    d = FakeEngine(H=8, fail_import_of=1)                      # prefill rank 1's cache cannot be mapped
    w = pd.PDWorker(d, "D", BS, rank=0, tp_size=1, total_kv_heads=8)
    w.start_pulls(pd.PDMeta([spec()], {}))
    assert w.take_failed_blocks() == {1, 2, 3, 4} and w.poll() == (set(), set())
    # rank 0 read nothing (the sources are resolved before the first pull); both producer ranks are told
    assert d.pulls == [] and all(os.listdir(pd.done_dir("P", p)) == ["p-req.d0of1"] for p in range(2))


def test_lease_checked_before_the_first_pull_and_after_the_last(shm):
    publish("P", 8, 2)
    lease = pd.lease_path("P", "L1")
    os.makedirs(os.path.dirname(lease))
    open(lease, "w").close()
    d = FakeEngine(H=8)
    w = pd.PDWorker(d, "D", BS, rank=0, tp_size=1, total_kv_heads=8)
    w.start_pulls(pd.PDMeta([spec(lease="L1")], {}))
    assert len(d.pulls) == 2
    os.unlink(lease)                                           # freed while the pulls ran
    assert w.poll(block=True)[1] == {"d-p-req"} and w.take_failed_blocks() == {1, 2, 3, 4}
    w.start_pulls(pd.PDMeta([spec(lease="L1")], {}))           # gone before: nothing issued
    assert len(d.pulls) == 2 and w.take_failed_blocks() == {1, 2, 3, 4} and w.n_lease_failures == 2


@pytest.mark.parametrize("t_d", range(1, 9))
def test_producer_releases_once_every_consumer_rank_marked(shm, t_d):
    t_p = 2 if t_d != 2 else 4
    publish("P", 8, t_p)
    producers = [pd.PDWorker(FakeEngine(), "P", BS, rank=p, tp_size=t_p) for p in range(t_p)]
    for w in producers:
        w.start_pulls(pd.PDMeta([], {"p-req": 1e18, "other": 1e18}))
    consumers = [pd.PDWorker(FakeEngine(H=max(1, 8 // t_d)), "D", BS, rank=c, tp_size=t_d, total_kv_heads=8)
                 for c in range(t_d)]
    for c in consumers[:-1]:
        c._notify_done(spec(t_p=t_p))
    assert all(w.poll()[0] == set() for w in producers)       # one consumer rank's marker missing
    consumers[-1]._notify_done(spec(t_p=t_p))
    for p, w in enumerate(producers):
        assert w.poll()[0] == {"p-req"}
        assert os.listdir(pd.done_dir("P", p)) == []           # its markers are removed with it
        assert w.poll()[0] == set()                            # "other" stays held


def test_lease_expiry_releases_without_markers_and_plain_marker_still_releases(shm):
    publish("P", 8, 2)
    w0 = pd.PDWorker(FakeEngine(), "P", BS, rank=0, tp_size=2)
    w0.start_pulls(pd.PDMeta([], {"late": 0.0, "plain": 1e18, "half": 1e18}))
    open(os.path.join(pd.done_dir("P", 0), "plain"), "w").close()
    open(os.path.join(pd.done_dir("P", 0), pd.split_marker("half", 0, 4)), "w").close()
    assert w0.poll()[0] == {"late", "plain"}
    assert os.listdir(pd.done_dir("P", 0)) == ["half.d0of4"]


def test_same_size_markers_keep_their_names(shm):
    publish("P", 8, 2)
    for c in range(2):
        w = pd.PDWorker(FakeEngine(), "D", BS, rank=c, tp_size=2, total_kv_heads=8)
        w._notify_done(spec(t_p=2))
        w._notify_done(pd.PullSpec("d", "P", "zero", [1], [1], 1))          # remote_tp_size 0: the same size
    for c in range(2):
        assert sorted(os.listdir(pd.done_dir("P", c))) == ["p-req", "zero"]
    assert pd.split_markers(["p-req", "a.b.d1of4", "x.d4of4", "y.d0of1"]) == {"a.b": {4: {1}}, "y": {1: {0}}}
