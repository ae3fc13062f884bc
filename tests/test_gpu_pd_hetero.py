"""Disaggregated prefill between replicas of different tensor-parallel sizes on an H100 (-m gpu): each consumer rank
pulls its KV heads from the producer ranks that hold them (b200kv_import_peer_ptrs_sliced / _sliced over CUDA IPC,
kv_head_slice_pull_kernel).  Pulled pages are bit-exact against torch indexing of the model's global KV; heads and
slots outside the pull keep a sentinel."""
import ctypes
import os
import sys

import numpy as np
import pytest

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from b200kv import FMT_RAW, KVEngine, KVGeometry, _lib, pd  # noqa: E402
from b200kv._lib import B200KVError  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L, NB, BS, D = 2, 40, 16, 128
SENTINEL = {2: -21846, 1: 0xA5}          # 0xAAAA as int16, 0xA5 as uint8


def need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device: the product has no CPU fallback")


def global_kv(T, elem, seed):
    """The model's KV of every layer over all T heads, token-major: (2, NB*BS, T, D) of int16 (bf16 bits) or uint8."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    if elem == 2:
        return [torch.randn((2, NB * BS, T, D), generator=g, device="cuda").bfloat16().view(torch.int16)
                for _ in range(L)]
    return [torch.randint(0, 256, (2, NB * BS, T, D), generator=g, device="cuda", dtype=torch.uint8)
            for _ in range(L)]


def to_pages(tok, hnd):
    """Token-major (2, NB*BS, H, D) -> the paged cache (2, NB, BS, H, D) (NHD) or (2, NB, H, BS, D) (HND)."""
    x = tok.reshape(2, NB, BS, tok.shape[2], D)
    return (x.permute(0, 1, 3, 2, 4) if hnd else x).contiguous()


def to_tokens(pages, hnd):
    x = pages.permute(0, 1, 3, 2, 4) if hnd else pages
    return x.reshape(2, NB * BS, x.shape[3], D)


def rank_pages(G, T, t, r, hnd):
    heads = pd.heads_of_rank(T, t, r)
    return [to_pages(x[:, :, heads], hnd) for x in G]


def mapping(rng, n_tok, kind):
    if kind == "tokens":                          # token-granular: every token in another block
        return rng.permutation(NB * BS)[:n_tok].astype(np.int64)
    blocks = rng.permutation(NB)[: (n_tok + BS - 1) // BS]
    return pd.slots_of(blocks, BS, n_tok)


def consumer(T, t_d, elem, hnd):
    H = max(1, T // t_d)
    g = KVGeometry(L, H, D, NB, BS, 256, elem, 0, FMT_RAW, _lib.LAYOUT_HND if hnd else _lib.LAYOUT_NHD)
    pages = [torch.full((2, NB, H, BS, D) if hnd else (2, NB, BS, H, D), SENTINEL[elem], device="cuda",
                        dtype=torch.int16 if elem == 2 else torch.uint8) for _ in range(L)]
    eng = KVEngine(g, None, 0, staging_bytes=0)
    eng.register_kv_ptrs([p[0].data_ptr() for p in pages], [p[1].data_ptr() for p in pages])
    return eng, pages


def expected(G, T, t_d, c, src, dst, elem):
    heads = pd.heads_of_rank(T, t_d, c)
    out = []
    si, di = torch.from_numpy(src).cuda(), torch.from_numpy(dst).cuda()
    for x in G:
        e = torch.full((2, NB * BS, len(heads), D), SENTINEL[elem], device="cuda", dtype=x.dtype)
        e[:, di] = x[:, si][:, :, heads]
        out.append(e)
    return out


# (total KV heads T, producer TP, consumer TP): 1->2, 2->4, 4->2, 2->1 (two sources into one page set), and
# replication (T < t) on the consumer and on the producer side
PAIRINGS = [(8, 1, 2), (8, 2, 4), (8, 4, 2), (8, 2, 1), (2, 1, 4), (2, 4, 1)]


@pytest.mark.parametrize("T,t_p,t_d", PAIRINGS)
@pytest.mark.parametrize("hnd", [False, True], ids=["nhd", "hnd"])
@pytest.mark.parametrize("elem", [2, 1], ids=["bf16", "fp8"])
@pytest.mark.parametrize("kind", ["blocks", "tokens"])
def test_sliced_pull_is_bit_exact(T, t_p, t_d, hnd, elem, kind):
    need_gpu()
    rng = np.random.default_rng(T * 100 + t_p * 10 + t_d + 1000 * hnd + 2000 * elem)
    G = global_kv(T, elem, seed=T * 7 + t_p)
    producers = [rank_pages(G, T, t_p, p, hnd) for p in range(t_p)]
    n_tok, skip = 300, 32                        # a ragged tail and a block-aligned prefix already computed
    src, dst = mapping(rng, n_tok, kind)[skip:], mapping(rng, n_tok, "blocks")[skip:]
    for c in range(t_d):
        eng, pages = consumer(T, t_d, elem, hnd)
        slices = pd.head_slices(T, t_p, t_d, c)
        for pid, (p, sl) in enumerate(slices):
            pp = producers[p]
            eng.import_peer_ptrs(pid, 0, [x[0].data_ptr() for x in pp], [x[1].data_ptr() for x in pp],
                                 peer_block_stride=BS * sl[0] * D * elem, head_slice=sl)
        for pid in range(len(slices)):
            eng.wait(eng.peer_pull(pid, src, dst))
        torch.cuda.synchronize()
        for got, want in zip(pages, expected(G, T, t_d, c, src, dst, elem)):
            assert torch.equal(to_tokens(got, hnd), want), (c, slices)
        assert eng.stats()["p2p_bytes"] == len(src) * 2 * L * D * elem * sum(sl[3] for _, sl in slices)
        eng.close()


def test_refused_slices_install_nothing():
    need_gpu()
    T, elem = 8, 2
    eng, pages = consumer(T, 2, elem, False)                  # H = 4
    peer = [torch.zeros((2, NB, BS, 2, D), device="cuda", dtype=torch.int16) for _ in range(L)]
    k, v = [x[0].data_ptr() for x in peer], [x[1].data_ptr() for x in peer]
    ka = (ctypes.c_void_p * L)(*k)
    va = (ctypes.c_void_p * L)(*v)
    stride = BS * 2 * D * elem
    lib = _lib.lib()
    for bad, st in [((2, 1, 0, 2), stride),                   # outside the peer's heads
                    ((2, 0, 3, 2), stride),                   # outside ours
                    ((2, 0, 0, 0), stride), ((2, -1, 0, 1), stride), ((0, 0, 0, 1), stride),
                    ((2, 0, 0, 2), stride - 16)]:             # a peer block smaller than bs * H_p * D * elem
        sl = _lib.HeadSlice(*bad)
        assert lib.b200kv_import_peer_ptrs_sliced(eng._h, 1, 0, ka, va, st, NB, ctypes.byref(sl)) == _lib.EINVAL, bad
    assert lib.b200kv_import_peer_ptrs_sliced(eng._h, 1, 0, ka, va, stride, NB, None) == _lib.EINVAL
    with pytest.raises(B200KVError) as e:
        eng.peer_pull(1, [0], [0])
    assert e.value.code == _lib.ENOENT                        # the peer id stayed free
    eng.import_peer_ptrs(1, 0, k, v, peer_block_stride=stride, head_slice=(2, 0, 2, 2))
    eng.wait(eng.peer_pull(1, np.arange(BS), np.arange(BS)))
    eng.close()
    # head_dim * elem_bytes not a multiple of 16 (the engine's token row still is)
    g = KVGeometry(L, 2, 8, NB, BS, 256, 1)
    small = [torch.zeros((2, NB, BS, 2, 8), device="cuda", dtype=torch.uint8) for _ in range(L)]
    e2 = KVEngine(g, None, 0, staging_bytes=0)
    e2.register_kv_ptrs([x[0].data_ptr() for x in small], [x[1].data_ptr() for x in small])
    with pytest.raises(B200KVError) as e:
        e2.import_peer_ptrs(0, 0, [x[0].data_ptr() for x in small], [x[1].data_ptr() for x in small],
                            head_slice=(2, 0, 0, 1))
    assert e.value.code == _lib.EINVAL
    e2.close()


@pytest.mark.parametrize("indexed", [False, True], ids=["mla", "v32"])
@pytest.mark.parametrize("t_p,t_d", [(1, 2), (2, 4), (4, 2), (2, 1)])
def test_mla_pairings_pull_whole_pages_from_rank_c_mod_tp(indexed, t_p, t_d):
    """An MLA latent (and V3.2's indexer plane) is the same on every rank: consumer rank c pulls whole pages from
    producer rank c % t_p through the unsliced import; a slice on an MLA engine is refused."""
    need_gpu()
    from tests import test_gpu_plane_table as tpt
    from tests import test_gpu_mla as tm
    from tests import test_gpu_mla_sparse as ts
    rng = np.random.default_rng(7 + t_p * 10 + t_d)
    Lm, NBm, bsm, n_tok = 2, 24, 64, 500
    producers = [tpt.planes(indexed, rng, Lm, NBm, bsm) for _ in range(t_p)]   # distinct pages per rank
    src, dst = ts.mapping(rng, NBm, bsm, n_tok), ts.mapping(rng, NBm, bsm, n_tok, "tokens")
    for c in range(t_d):
        g, lat, idx, _remote, k, v = producers[c % t_p]
        zl = [np.zeros_like(a) for a in lat]
        if indexed:
            zi = [np.zeros_like(b) for b in idx]
            local = ts.to_dev(zl, zi)
        else:
            local = tm.to_dev(zl)
        eng = KVEngine(g, None, 0, staging_bytes=0)
        eng.register_kv_caches(local)
        with pytest.raises(B200KVError) as e:
            eng.import_peer_ptrs(0, 0, k, v, head_slice=(1, 0, 0, 1))
        assert e.value.code == _lib.EINVAL
        eng.import_peer_ptrs(0, 0, k, v)
        eng.wait(eng.peer_pull(0, src, dst))
        torch.cuda.synchronize()
        if indexed:
            el, ei = ts.expected_pages(FMT_RAW, lat, idx, src, dst, 256, zl, zi)
            hl, hi = ts.host_of(local)
            got, want = hl + hi, el + ei
        else:
            got, want = [tm.host_of(t) for t in local], tm._expected_pages(FMT_RAW, lat, src, dst, 256, zl)
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
        eng.close()


# ---- two processes, real CUDA IPC: a TP=2 producer (two ranks in one process), consumers at TP=4 and TP=1 -----
T_IPC, TP_IPC = 8, 2


def _producer(eid, ready, stop, shm_dir):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "production-stack_b200")]
    # one cudaMalloc per tensor: the two ranks' planes must be separate allocations, as in two processes
    os.environ["PYTORCH_NO_CUDA_MEMORY_CACHING"] = "1"
    import torch
    from b200kv import KVEngine, KVGeometry, pd
    pd.SHM_DIR = shm_dir
    torch.cuda.set_device(0)
    G = global_kv(T_IPC, 2, seed=42)
    engines, keep = [], []
    for r in range(TP_IPC):
        pages = rank_pages(G, T_IPC, TP_IPC, r, False)
        eng = KVEngine(KVGeometry(L, T_IPC // TP_IPC, D, NB, BS, 256), None, 0, staging_bytes=0)
        eng.register_kv_ptrs([p[0].data_ptr() for p in pages], [p[1].data_ptr() for p in pages])
        pd.publish_ipc(eid, eng, 0, rank=r, tp_size=TP_IPC, total_kv_heads=T_IPC)
        engines.append(eng)
        keep.append(pages)
    torch.cuda.synchronize()
    ready.set()
    stop.wait(300)
    for r, eng in enumerate(engines):
        pd.unpublish_ipc(eid, r)
        eng.close()


def test_sliced_pull_from_another_process(tmp_path):
    need_gpu()
    import torch.multiprocessing as mp
    shm_dir = str(tmp_path)
    pd.SHM_DIR = shm_dir
    ctx = mp.get_context("spawn")
    ready, stop = ctx.Event(), ctx.Event()
    eid = f"prod-hetero-{os.getpid()}"
    proc = ctx.Process(target=_producer, args=(eid, ready, stop, shm_dir))
    proc.start()
    try:
        assert ready.wait(240), "producer did not come up"
        G = global_kv(T_IPC, 2, seed=42)
        rng = np.random.default_rng(5)
        n_tok, skip = 700, 32
        remote_blocks = [int(x) for x in rng.permutation(NB)[: (n_tok + BS - 1) // BS]]
        for t_d in (4, 1):
            for c in range(t_d):
                eng, pages = consumer(T_IPC, t_d, 2, False)
                w = pd.PDWorker(eng, f"cons{t_d}", BS, rank=c, tp_size=t_d, total_kv_heads=T_IPC)
                local_blocks = [int(x) for x in rng.permutation(NB)[: (n_tok + BS - 1) // BS]]
                rid = f"req-{t_d}-{c}"
                spec = pd.PullSpec("d-" + rid, eid, rid, remote_blocks, local_blocks, n_tok, skip_tokens=skip,
                                   remote_tp_size=TP_IPC)
                w.start_pulls(pd.PDMeta([spec], {}))
                assert w.take_failed_blocks() == set()
                assert w.poll(block=True)[1] == {"d-" + rid}
                src = pd.slots_of(remote_blocks, BS, n_tok)[skip:]
                dst = pd.slots_of(local_blocks, BS, n_tok)[skip:]
                for got, want in zip(pages, expected(G, T_IPC, t_d, c, src, dst, 2)):
                    assert torch.equal(to_tokens(got, False), want)
                for p in range(TP_IPC):     # every producer rank hears from every consumer rank
                    assert os.path.exists(os.path.join(pd.done_dir(eid, p), pd.split_marker(rid, c, t_d)))
                assert len(w.resolver.ids) == len(pd.head_slices(T_IPC, TP_IPC, t_d, c))
                eng.close()
    finally:
        stop.set()
        proc.join(60)
