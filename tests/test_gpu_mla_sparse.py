"""Sparse-attention MLA engines (DeepSeek-V3.2) on an H100 (-m gpu): a latent plane and an indexer plane per layer,
pages as vLLM allocates them ((NB, bs, 576) bf16 latent, (NB, bs, 132) uint8 indexer).  The indexer tile layout is
pinned by vLLM's own ops; every path is bit-exact against tests/mla_sparse_oracle.py (RAW latent, or FP8 latent
records by tests/mla_oracle.py, and the indexer planes verbatim)."""
import os
import sys

import numpy as np
import pytest

from oracle import kv_oracle as ko
from tests import mla_oracle as mo
from tests import mla_sparse_oracle as so

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from b200kv import FMT_FP8, FMT_RAW, KVEngine, KVGeometry, KVPool, _lib  # noqa: E402
from b200kv._lib import B200KVError  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 576
MLA = _lib.LAYOUT_MLA


def need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device: the product has no CPU fallback")


def geom(L, NB, bs, C=256, fmt=FMT_RAW):
    return KVGeometry(L, 1, D, NB, bs, C, 2, 0, fmt, MLA, idx_value_bytes=128, idx_scale_bytes=4)


def mk_host(rng, L, NB, bs):
    """(latent bf16 bit patterns, indexer bytes) host pages; latent groups span very different ranges."""
    lat = []
    for _ in range(L):
        x = rng.standard_normal((NB, bs, D)).astype(np.float32)
        x *= np.exp(rng.uniform(-4, 4, (NB, bs, 5)).repeat([128, 128, 128, 128, 64], axis=-1)).astype(np.float32)
        lat.append(ko.f32_to_bf16_bits_rn(x).reshape(NB, bs, D))
    idx = [rng.integers(0, 256, (NB, bs, so.IDX_TOKEN), dtype=np.uint8) for _ in range(L)]
    return lat, idx


def to_dev(lat, idx):
    """{vLLM layer name: tensor}, a layer's attention then its indexer, as the model runner hands them over."""
    out = {}
    for l, (a, b) in enumerate(zip(lat, idx)):
        out[f"model.layers.{l}.self_attn.attn"] = torch.from_numpy(a.view(np.int16)).view(torch.bfloat16).cuda()
        out[f"model.layers.{l}.self_attn.indexer.k_cache"] = torch.from_numpy(b.copy()).cuda()
    return out


def host_of(caches):
    lat, idx = [], []
    for n, t in caches.items():
        a = t.cpu().contiguous()
        (idx if "indexer" in n else lat).append(a.numpy() if a.dtype == torch.uint8 else a.view(torch.int16).numpy().view(np.uint16))
    return lat, idx


def fill_from(caches, lat, idx):
    for t, h in zip(caches.values(), [x for pair in zip(lat, idx) for x in pair]):
        t.copy_(torch.from_numpy(h.view(np.int16) if h.dtype == np.uint16 else h).view(t.dtype))


def mapping(rng, NB, bs, n_tok, kind="blocks"):
    if kind == "tokens":                                   # token-granular: every token in another block
        return rng.permutation(NB * bs)[:n_tok].astype(np.int64)
    return ko.slot_mapping_from_blocks(rng.permutation(NB)[:(n_tok + bs - 1) // bs], bs, n_tok)


def expected_pages(fmt, lat, idx, sm, dm, C, before_lat, before_idx):
    el, ei = [b.copy() for b in before_lat], [b.copy() for b in before_idx]
    for c in range(0, len(sm), C):
        bits = mo.gather_tokens(lat, sm[c:c + C])
        if fmt == FMT_FP8:
            bits = mo.fp8_unpack_chunk(mo.fp8_pack_chunk(bits))
        mo.scatter_tokens(el, bits, dm[c:c + C])
        so.scatter_slabs(ei, so.gather_slabs(idx, sm[c:c + C], C), dm[c:c + C], C)
    return el, ei


def check_chunk(got, g, lat, idx, sm, fmt):
    """One chunk's bytes (valid tokens only) against the oracle."""
    n, C, L = len(sm), g.chunk_tokens, g.n_layers
    want = so.pack_chunk(lat, idx, sm, C, "fp8" if fmt == FMT_FP8 else "raw")
    tb = mo.MLA_RECORD if fmt == FMT_FP8 else D * 2
    gl, gi = so.split_chunk(got[:g.chunk_bytes], L, C, tb)
    wl, wi = so.split_chunk(want, L, C, tb)
    assert np.array_equal(gl[:, :n], wl[:, :n]), "latent"
    for a, b in zip(so.slab_tokens(gi, n, C), so.slab_tokens(wi, n, C)):
        assert np.array_equal(a, b), "indexer"


def test_tile_layout_is_pinned_by_vllms_indexer_ops():
    """Indexer planes filled by vLLM's indexer_k_quant_and_cache, stored, scattered into fresh planes: vLLM's
    cp_gather_indexer_k_quant_cache reads identical values and scales back, and the chunk equals the oracle's."""
    need_gpu()
    ops = pytest.importorskip("vllm._custom_ops")
    rng = np.random.default_rng(0)
    L, NB, bs, C, n = 2, 24, 64, 256, 600
    lat, _ = mk_host(rng, L, NB, bs)
    caches = to_dev(lat, [np.zeros((NB, bs, 132), np.uint8)] * L)
    sm = mapping(rng, NB, bs, n)
    sm_d = torch.from_numpy(sm).cuda()
    for name, t in caches.items():
        if "indexer" in name:
            k = torch.randn((n, 128), device="cuda:0", dtype=torch.bfloat16) * 3
            ops.indexer_k_quant_and_cache(k, t, sm_d, 128, "ue8m0")
    torch.cuda.synchronize()
    g = geom(L, NB, bs, C)
    eng = KVEngine(g, None, 0, staging_bytes=0)
    eng.register_kv_caches(caches)
    n_chunks = (n + C - 1) // C
    buf = torch.zeros(n_chunks * g.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    hl, hi = host_of(caches)
    got = buf.cpu().numpy()
    for c in range(n_chunks):
        check_chunk(got[c * g.chunk_bytes:], g, hl, hi, sm[c * C:(c + 1) * C], FMT_RAW)
    fresh = {k: torch.zeros_like(t) for k, t in caches.items()}
    eng2 = KVEngine(g, None, 0, staging_bytes=0)
    eng2.register_kv_caches(fresh)
    dm = mapping(np.random.default_rng(1), NB, bs, n)
    eng2.scatter(dm, buf.data_ptr())
    torch.cuda.synchronize()

    def read_back(cache, slots):
        blocks = torch.from_numpy(slots[::bs] // bs).to(torch.int32).cuda()[None]
        vals = torch.zeros((n, 128), dtype=torch.uint8, device="cuda:0")
        scales = torch.zeros((n, 4), dtype=torch.uint8, device="cuda:0")
        ops.cp_gather_indexer_k_quant_cache(cache, vals, scales, blocks, torch.tensor([0, n], dtype=torch.int32, device="cuda:0"))
        return vals.cpu().numpy(), scales.cpu().numpy()

    for name in caches:
        if "indexer" in name:
            a, b = read_back(caches[name], sm), read_back(fresh[name], dm)
            assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), name
            assert np.any(a[1])                                         # the op did write scales
    eng.close()
    eng2.close()


@pytest.mark.parametrize("kind", ["blocks", "tokens"])
@pytest.mark.parametrize("n_tok", [1, 37, 64, 257, 1000])
@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_FP8])
@pytest.mark.parametrize("bs", [16, 64])
def test_gather_scatter_bit_exact(bs, fmt, n_tok, kind):
    need_gpu()
    rng = np.random.default_rng(bs * 1000 + fmt * 100 + n_tok)
    L, C = 3, 256
    NB = 2 * ((1000 + bs - 1) // bs) + 3
    lat, idx = mk_host(rng, L, NB, bs)
    caches = to_dev(lat, idx)
    g = geom(L, NB, bs, C, fmt)
    eng = KVEngine(g, None, 0, staging_bytes=0)
    eng.register_kv_caches(caches)
    sm, dm = mapping(rng, NB, bs, n_tok, kind), mapping(rng, NB, bs, n_tok, kind)
    n_chunks = (n_tok + C - 1) // C
    buf = torch.zeros(n_chunks * g.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    for c in range(n_chunks):
        check_chunk(got[c * g.chunk_bytes:], g, lat, idx, sm[c * C:(c + 1) * C], fmt)
    bl, bi = mk_host(rng, L, NB, bs)
    fill_from(caches, bl, bi)
    eng.scatter(dm, buf.data_ptr())
    torch.cuda.synchronize()
    el, ei = expected_pages(fmt, lat, idx, sm, dm, C, bl, bi)
    hl, hi = host_of(caches)
    for a, e in zip(hl + hi, el + ei):
        assert np.array_equal(a, e)
    eng.close()


@pytest.mark.parametrize("mode", ["chunk", "layer1", "layer3", "batch"])
@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_FP8])
def test_pool_store_retrieve(fmt, mode):
    need_gpu()
    rng = np.random.default_rng(11)
    L, bs, C, NB = 5, 64, 256, 64
    lat, idx = mk_host(rng, L, NB, bs)
    caches = to_dev(lat, idx)
    g = geom(L, NB, bs, C, fmt)
    pool = KVPool(None, 24 * g.chunk_bytes, g.chunk_bytes, 1)
    eng = KVEngine(g, pool, 0, staging_bytes=8 * g.chunk_bytes)
    eng.register_kv_caches(caches)
    lens = [700, 64, 300] if mode == "batch" else [700]
    reqs, off = [], 0
    perm = rng.permutation(NB)
    for i, n in enumerate(lens):
        nb = (n + bs - 1) // bs
        toks = (np.arange(n, dtype=np.int32) + 1000 * i) * 7 % 5000
        reqs.append((toks, ko.slot_mapping_from_blocks(perm[off:off + nb], bs, n)))
        off += nb
    if mode == "batch":
        eng.wait(eng.store_batch([(t, s, 0) for t, s in reqs]))
    else:
        eng.wait(eng.store(reqs[0][0], None, reqs[0][1]))
    for t, _ in reqs:
        assert eng.lookup(t) == len(t)
    # the pool holds the oracle's chunks, tagged with the indexer bit
    slot, n0, tag = pool.acquire(eng._keys(reqs[0][0])[2])
    assert tag == g.fmt_tag and tag & _lib.FMT_TAG_INDEXED
    check_chunk(pool.slot_view(slot), g, lat, idx, reqs[0][1][512:700], fmt)
    pool.release(eng._keys(reqs[0][0])[2])
    bl, bi = mk_host(rng, L, NB, bs)
    fill_from(caches, bl, bi)
    perm2, off, dms = np.random.default_rng(5).permutation(NB), 0, []
    for t, _ in reqs:
        nb = (len(t) + bs - 1) // bs
        dms.append(ko.slot_mapping_from_blocks(perm2[off:off + nb], bs, len(t)))
        off += nb
    if mode == "batch":
        loaded, ticket = eng.retrieve_batch([(t, d, 0) for (t, _), d in zip(reqs, dms)])
        assert list(loaded) == lens
        eng.wait(ticket)
    elif mode == "chunk":
        assert eng.retrieve(reqs[0][0], None, dms[0]).all()
    else:
        G = 1 if mode == "layer1" else 3
        s = torch.cuda.Stream()
        ret, ticket = eng.retrieve(reqs[0][0], None, dms[0], stream=s, return_ticket=True, layers_per_group=G)
        assert ret.all() and ticket
        for layer in range(L):                       # the forward pass waits per layer: latent and indexer
            eng.wait_layer(ticket, layer, s)
            with torch.cuda.stream(s):
                seen = [caches[f"model.layers.{layer}.self_attn.attn"].clone(),
                        caches[f"model.layers.{layer}.self_attn.indexer.k_cache"].clone()]
            s.synchronize()
            el, ei = expected_pages(fmt, [lat[layer]], [idx[layer]], reqs[0][1], dms[0], C, [bl[layer]], [bi[layer]])
            assert np.array_equal(seen[0].cpu().view(torch.int16).numpy().view(np.uint16), el[0]), layer
            assert np.array_equal(seen[1].cpu().numpy(), ei[0]), layer
        eng.wait(ticket)
    torch.cuda.synchronize()
    el, ei = bl, bi
    for (t, sm), dm in zip(reqs, dms):
        el, ei = expected_pages(fmt, lat, idx, sm, dm, C, el, ei)
    hl, hi = host_of(caches)
    for a, e in zip(hl + hi, el + ei):
        assert np.array_equal(a, e)
    eng.close()
    pool.close()


def test_device_tier_gather_scatter_chunks():
    need_gpu()
    rng = np.random.default_rng(3)
    L, bs, C, NB, n_tok = 4, 64, 256, 40, 600
    lat, idx = mk_host(rng, L, NB, bs)
    caches = to_dev(lat, idx)
    for fmt in (FMT_RAW, FMT_FP8):
        g = geom(L, NB, bs, C, fmt)
        eng = KVEngine(g, None, 0, staging_bytes=0)
        eng.register_kv_caches(caches)
        base = eng.tier_create(5)                            # slots of the indexed chunk size
        order = (3, 0, 4)
        ptrs = [base + s * g.chunk_bytes for s in order]
        sm, dm = mapping(rng, NB, bs, n_tok), mapping(rng, NB, bs, n_tok)
        eng.gather_chunks(sm, ptrs)
        torch.cuda.synchronize()
        out = {k: torch.zeros_like(t) for k, t in caches.items()}
        eng2 = KVEngine(g, None, 0, staging_bytes=0)
        eng2.register_kv_caches(out)
        eng2.scatter_chunks(dm, ptrs)
        torch.cuda.synchronize()
        zl, zi = [np.zeros_like(h) for h in lat], [np.zeros_like(h) for h in idx]
        el, ei = expected_pages(fmt, lat, idx, sm, dm, C, zl, zi)
        hl, hi = host_of(out)
        for a, e in zip(hl + hi, el + ei):
            assert np.array_equal(a, e), fmt
        eng2.close()
        eng.close()


def _producer(eid, ready, stop, shm_dir, L, NB, bs):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "production-stack_b200")]
    import torch
    from b200kv import KVEngine, KVGeometry, _lib, pd
    pd.SHM_DIR = shm_dir
    g = torch.Generator(device="cuda:0").manual_seed(42)
    caches = {}
    for l in range(L):
        caches[f"layers.{l}.attn"] = torch.randn((NB, bs, 576), generator=g, device="cuda:0").bfloat16()
        caches[f"layers.{l}.indexer.k_cache"] = torch.randint(0, 256, (NB, bs, 132), generator=g, device="cuda:0",
                                                             dtype=torch.uint8)
    eng = KVEngine(KVGeometry(L, 1, 576, NB, bs, 256, 2, 0, 0, _lib.LAYOUT_MLA, idx_value_bytes=128,
                              idx_scale_bytes=4), None, 0, staging_bytes=0)
    eng.register_kv_caches(caches)
    torch.cuda.synchronize()
    pd.publish_ipc(eid, eng, 0)
    ready.set()
    stop.wait(120)
    pd.unpublish_ipc(eid)
    eng.close()


def test_peer_pull_across_processes(tmp_path):
    need_gpu()
    import ctypes
    import torch.multiprocessing as mp

    from b200kv import pd
    L, NB, bs, n_tok = 4, 48, 64, 1000
    shm_dir = str(tmp_path)
    pd.SHM_DIR = shm_dir
    ctx = mp.get_context("spawn")
    ready, stop = ctx.Event(), ctx.Event()
    eid = f"v32-prod-{os.getpid()}"
    proc = ctx.Process(target=_producer, args=(eid, ready, stop, shm_dir, L, NB, bs))
    proc.start()
    try:
        assert ready.wait(180), "producer did not come up"
        zl = [np.zeros((NB, bs, D), np.uint16) for _ in range(L)]
        zi = [np.zeros((NB, bs, 132), np.uint8) for _ in range(L)]
        local = to_dev(zl, zi)
        eng = KVEngine(geom(L, NB, bs), None, 0, staging_bytes=0)
        eng.register_kv_caches(local)
        assert len(eng.export_ipc()) == 2 * L * ctypes.sizeof(_lib.IpcDesc)   # latent, then indexer planes
        pid = pd.PeerResolver(eng).resolve(eid)
        rng = np.random.default_rng(0)
        src, dst = mapping(rng, NB, bs, n_tok), mapping(rng, NB, bs, n_tok, "tokens")
        eng.wait(eng.peer_pull(pid, src, dst))
        torch.cuda.synchronize()
        g = torch.Generator(device="cuda:0").manual_seed(42)
        wl, wi = [], []
        for _ in range(L):
            wl.append(torch.randn((NB, bs, 576), generator=g, device="cuda:0").bfloat16().cpu().view(torch.int16).numpy().view(np.uint16))
            wi.append(torch.randint(0, 256, (NB, bs, 132), generator=g, device="cuda:0", dtype=torch.uint8).cpu().numpy())
        el, ei = expected_pages(FMT_RAW, wl, wi, src, dst, 256, zl, zi)
        hl, hi = host_of(local)
        for a, e in zip(hl + hi, el + ei):
            assert np.array_equal(a, e)
        assert eng.stats()["p2p_bytes"] == n_tok * L * (D * 2 + 132)
        eng.close()
    finally:
        stop.set()
        proc.join(60)


def test_refused_op_leaves_no_reserved_slots_and_no_pins():
    """As for every other engine: an op refused after reserving / pinning (a token-granular table too large to
    stage) leaves nothing reserved or pinned, and the same keys store and load at once afterwards."""
    need_gpu()
    L, NB, bs, C_ = 1, 8192, 16, 256
    g = geom(L, NB, bs, C_)
    lat = [np.zeros((NB, bs, D), np.uint16)]
    idx = [np.random.default_rng(2).integers(0, 256, (NB, bs, 132), dtype=np.uint8)]
    caches = to_dev(lat, idx)
    n_chunks = 420
    pool = KVPool(None, (n_chunks + 8) * g.chunk_bytes, g.chunk_bytes, 1)
    eng = KVEngine(g, pool, 0, staging_bytes=2 * 512 * g.chunk_bytes)
    eng.register_kv_caches(caches)
    n = n_chunks * C_
    rng = np.random.default_rng(11)
    toks = rng.integers(0, 50000, n).astype(np.int32)
    scattered = (np.arange(n, dtype=np.int64) * 2) % (NB * bs) + (np.arange(n) * 2 // (NB * bs))
    with pytest.raises(B200KVError) as ei:
        eng.store(toks, None, scattered)
    assert ei.value.code == _lib.EINVAL
    st = pool.stats()
    assert st["n_used"] == 0 and pool.check(), st
    sm = ko.slot_mapping_from_blocks(rng.permutation(NB)[: n // bs], bs, n)
    eng.wait(eng.store(toks, None, sm))
    assert pool.stats()["n_stored_chunks"] == n_chunks and eng.lookup(toks) == n
    with pytest.raises(B200KVError):
        eng.retrieve(toks, None, scattered)
    assert pool.clear()
    eng.close()
    pool.close()


def test_set_indexer_refusals():
    need_gpu()
    plain = KVGeometry(2, 1, D, 8, 64, 256, 2, 0, FMT_RAW, MLA)
    caches = [torch.zeros((8, 64, D), device="cuda:0", dtype=torch.bfloat16) for _ in range(2)]
    eng = KVEngine(plain, None, 0, staging_bytes=0)
    eng.register_kv_caches(caches)
    assert _lib.lib().b200kv_set_indexer(eng._h, 128, 4, 64 * 132) == _lib.EBUSY      # after registration
    eng.close()
    kv = KVEngine(KVGeometry(2, 8, 128, 8, 16, 256), None, 0, staging_bytes=0)
    assert _lib.lib().b200kv_set_indexer(kv._h, 128, 4, 16 * 132) == _lib.EINVAL      # not an MLA engine
    kv.close()
    eng = KVEngine(plain, None, 0, staging_bytes=0)
    assert _lib.lib().b200kv_set_indexer(eng._h, 128, 4, 64 * 132 - 16) == _lib.EINVAL   # stride below a tile
    eng.tier_create(1)
    assert _lib.lib().b200kv_set_indexer(eng._h, 128, 4, 64 * 132) == _lib.EBUSY      # tier slots already cut
    eng.close()
    # a pool whose slots are too small for the indexed chunk is refused
    pool = KVPool(None, 4 * plain.chunk_bytes, plain.chunk_bytes, 1)
    with pytest.raises(B200KVError) as e:
        KVEngine(geom(2, 8, 64), pool, 0, staging_bytes=4 * geom(2, 8, 64).chunk_bytes)
    assert e.value.code == _lib.EINVAL
    pool.close()
    # the indexed engine takes the indexer planes in v_ptrs and refuses registration without them
    eng = KVEngine(geom(2, 8, 64), None, 0, staging_bytes=0)
    import ctypes
    ka = (ctypes.c_void_p * 2)(*[c.data_ptr() for c in caches])
    assert _lib.lib().b200kv_register_kv(eng._h, ka, None) == _lib.EINVAL
    eng.close()
