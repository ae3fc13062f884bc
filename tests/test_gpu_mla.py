"""MLA engines on an H100 (-m gpu): one latent plane per layer, pages (NB, bs, 576) as vLLM's MLA backends
allocate them.  RAW is bit-exact against tests/mla_oracle.py's gather/scatter; FP8 latent records (codes,
scales, RoPE) and the pages decoded from them are bit-exact against its codec."""
import os
import sys

import numpy as np
import pytest

from oracle import kv_oracle as ko
from tests import mla_oracle as mo

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from b200kv import FMT_FP8, FMT_Q4, FMT_RAW, KVEngine, KVGeometry, KVPool, _lib  # noqa: E402
from b200kv._lib import B200KVError  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
D = 576
MLA = _lib.LAYOUT_MLA


def need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device: the product has no CPU fallback")


def mk_layers(rng, L, NB, bs, elem=2):
    """Host pages (NB, bs, D): bf16 bit patterns whose 128-element groups span very different ranges, or raw
    bytes for a one-byte (fp8) cache."""
    if elem == 1:
        return [rng.integers(0, 256, (NB, bs, D), dtype=np.uint8) for _ in range(L)]
    out = []
    for _ in range(L):
        x = rng.standard_normal((NB, bs, D)).astype(np.float32)
        x *= np.exp(rng.uniform(-4, 4, (NB, bs, 5)).repeat([128, 128, 128, 128, 64], axis=-1)).astype(np.float32)
        out.append(ko.f32_to_bf16_bits_rn(x).reshape(NB, bs, D))
    return out


def to_dev(layers):
    if layers[0].dtype == np.uint8:
        return [torch.from_numpy(l.copy()).cuda() for l in layers]
    return [torch.from_numpy(l.view(np.int16)).view(torch.bfloat16).cuda() for l in layers]


def host_of(t):
    a = t.cpu().contiguous()
    return a.numpy() if a.dtype == torch.uint8 else a.view(torch.int16).numpy().view(np.uint16)


def geom(L, NB, bs, C=256, elem=2, fmt=FMT_RAW):
    return KVGeometry(L, 1, D, NB, bs, C, elem, 0, fmt, MLA)


def slots(rng, NB, bs, n_tok):
    return ko.slot_mapping_from_blocks(rng.permutation(NB)[:(n_tok + bs - 1) // bs], bs, n_tok)


def raw_chunks(layers, sm, C):
    """Expected RAW chunk bytes (L, 1, C, 1, D per chunk), padded to whole chunks."""
    n = len(sm)
    out = []
    for c in range(0, n, C):
        g = mo.gather_tokens(layers, sm[c:c + C])
        pad = np.zeros(g.shape[:2] + (C,) + g.shape[3:], g.dtype)
        pad[:, :, :g.shape[2]] = g
        out.append(pad.view(np.uint8).reshape(-1))
    return out


def chunk_tokens_of(got, g, n):
    """(L, n, token_bytes) view of the first n tokens of one chunk's bytes."""
    tb = mo.MLA_RECORD if g.fmt == FMT_FP8 else D * g.elem_bytes
    return got[:g.n_layers * g.chunk_tokens * tb].reshape(g.n_layers, g.chunk_tokens, tb)[:, :n]


@pytest.mark.parametrize("n_tok", [1, 63, 64, 65, 255, 256, 257, 1000])
@pytest.mark.parametrize("elem", [2, 1])
@pytest.mark.parametrize("bs", [16, 64, 128])
def test_raw_gather_scatter_bit_exact(bs, elem, n_tok):
    need_gpu()
    rng = np.random.default_rng(bs * 100 + elem * 10 + n_tok)
    L, C = 3, 256
    NB = 2 * ((1000 + bs - 1) // bs) + 3
    host = mk_layers(rng, L, NB, bs, elem)
    dev = to_dev(host)
    g = geom(L, NB, bs, C, elem)
    eng = KVEngine(g, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    sm, dm = slots(rng, NB, bs, n_tok), slots(rng, NB, bs, n_tok)
    n_chunks = (n_tok + C - 1) // C
    buf = torch.zeros(n_chunks * g.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    want = raw_chunks(host, sm, C)
    got = buf.cpu().numpy()
    tb = D * elem
    for c in range(n_chunks):
        n = min(C, n_tok - c * C)
        w = want[c].reshape(L, C, tb)[:, :n]
        assert np.array_equal(chunk_tokens_of(got[c * g.chunk_bytes:], g, n), w), c
    # scatter into pages that hold other data: the mapped slots take the chunk, every other byte stays
    before = mk_layers(rng, L, NB, bs, elem)
    dev2 = to_dev(before)
    for a, b in zip(dev, dev2):
        a.copy_(b)
    eng.scatter(dm, buf.data_ptr())
    torch.cuda.synchronize()
    expect = [b.copy() for b in before]
    mo.scatter_tokens(expect, mo.gather_tokens(host, sm), dm)
    for a, e in zip(dev, expect):
        assert np.array_equal(host_of(a), e)
    eng.close()


@pytest.mark.parametrize("n_tok", [1, 65, 257, 1000])
@pytest.mark.parametrize("bs", [16, 64, 128])
def test_fp8_records_and_decoded_pages_bit_exact(bs, n_tok):
    need_gpu()
    rng = np.random.default_rng(7 + bs + n_tok)
    L, C = 3, 256
    NB = 2 * ((1000 + bs - 1) // bs) + 3
    host = mk_layers(rng, L, NB, bs)
    host[1][0, 0, 128:256] = 0             # a zero group (scale 1)
    dev = to_dev(host)
    g = geom(L, NB, bs, C, fmt=FMT_FP8)
    eng = KVEngine(g, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    sm, dm = slots(rng, NB, bs, n_tok), slots(rng, NB, bs, n_tok)
    sm[0] = 0                               # the zero group takes part
    n_chunks = (n_tok + C - 1) // C
    buf = torch.zeros(n_chunks * g.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    for c in range(n_chunks):
        n = min(C, n_tok - c * C)
        want = mo.fp8_pack_chunk(mo.gather_tokens(host, sm[c * C:c * C + n]))
        rec = chunk_tokens_of(got[c * g.chunk_bytes:], g, n)
        assert np.array_equal(rec[..., :512], want[..., :512]), ("codes", c)
        assert np.array_equal(rec[..., 512:528], want[..., 512:528]), ("scales", c)
        assert np.array_equal(rec[..., 528:], want[..., 528:]), ("rope", c)
    for t in dev:
        t.zero_()
    eng.scatter(dm, buf.data_ptr())
    torch.cuda.synchronize()
    expect = [np.zeros_like(h) for h in host]
    for c in range(n_chunks):
        n = min(C, n_tok - c * C)
        rec = chunk_tokens_of(got[c * g.chunk_bytes:], g, n)
        mo.scatter_tokens(expect, mo.fp8_unpack_chunk(np.ascontiguousarray(rec)), dm[c * C:c * C + n])
    for a, e in zip(dev, expect):
        assert np.array_equal(host_of(a), e)
    assert eng.stats()["n_kernel_launches"] == 2
    eng.close()


def _expected_pages(fmt, host, sm, dm, C, before):
    expect = [b.copy() for b in before]
    for c in range(0, len(sm), C):
        bits = mo.gather_tokens(host, sm[c:c + C])
        if fmt == FMT_FP8:
            bits = mo.fp8_unpack_chunk(mo.fp8_pack_chunk(bits))
        mo.scatter_tokens(expect, bits, dm[c:c + C])
    return expect


@pytest.mark.parametrize("mode", ["chunk", "layer1", "layer3", "batch"])
@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_FP8])
def test_pool_store_retrieve(fmt, mode):
    need_gpu()
    rng = np.random.default_rng(11)
    L, bs, C, NB = 5, 64, 256, 64
    host = mk_layers(rng, L, NB, bs)
    dev = to_dev(host)
    g = geom(L, NB, bs, C, fmt=fmt)
    pool = KVPool(None, 24 * g.chunk_bytes, g.chunk_bytes, 1)
    eng = KVEngine(g, pool, 0, staging_bytes=8 * g.chunk_bytes)
    eng.register_kv_caches(dev)
    lens = [700, 64, 300] if mode == "batch" else [700]
    reqs, off = [], 0
    perm = rng.permutation(NB)
    for i, n in enumerate(lens):
        nb = (n + bs - 1) // bs
        blocks = perm[off:off + nb]
        off += nb
        toks = (np.arange(n, dtype=np.int32) + 1000 * i) * 7 % 5000
        reqs.append((toks, ko.slot_mapping_from_blocks(blocks, bs, n)))
    if mode == "batch":
        eng.wait(eng.store_batch([(t, s, 0) for t, s in reqs]))
    else:
        eng.wait(eng.store(reqs[0][0], None, reqs[0][1]))
    for t, _ in reqs:
        assert eng.lookup(t) == len(t)
    before = mk_layers(rng, L, NB, bs)
    for a, b in zip(dev, to_dev(before)):
        a.copy_(b)
    dms = [slots(np.random.default_rng(99 + i), NB, bs, len(t)) for i, (t, _) in enumerate(reqs)]
    # destination slots of different requests must not overlap: shift them onto disjoint blocks
    if mode == "batch":
        perm2 = np.random.default_rng(5).permutation(NB)
        off, dms = 0, []
        for t, _ in reqs:
            nb = (len(t) + bs - 1) // bs
            dms.append(ko.slot_mapping_from_blocks(perm2[off:off + nb], bs, len(t)))
            off += nb
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
        for layer in range(L):                       # the forward pass waits per layer
            eng.wait_layer(ticket, layer, s)
        s.synchronize()
        eng.wait(ticket)
    torch.cuda.synchronize()
    expect = [b.copy() for b in before]
    for (t, sm), dm in zip(reqs, dms):
        expect = _expected_pages(fmt, host, sm, dm, C, expect)
    for a, e in zip(dev, expect):
        assert np.array_equal(host_of(a), e)
    st = eng.stats()
    n_all = sum(lens)
    per_tok = L * (mo.MLA_RECORD if fmt == FMT_FP8 else D * 2)
    assert st["d2h_bytes"] >= n_all * per_tok and st["n_loaded_tokens"] == n_all
    eng.close()
    pool.close()


def test_device_tier_gather_scatter_chunks():
    need_gpu()
    rng = np.random.default_rng(3)
    L, bs, C, NB, n_tok = 4, 64, 256, 40, 600
    host = mk_layers(rng, L, NB, bs)
    dev = to_dev(host)
    for fmt in (FMT_RAW, FMT_FP8):
        g = geom(L, NB, bs, C, fmt=fmt)
        eng = KVEngine(g, None, 0, staging_bytes=0)
        eng.register_kv_caches(dev)
        tier = torch.zeros((5, g.chunk_bytes), dtype=torch.uint8, device="cuda:0")   # a tier's slot array
        order = (3, 0, 4)                                                             # chunks in slots out of order
        ptrs = [tier[s].data_ptr() for s in order]
        sm, dm = slots(rng, NB, bs, n_tok), slots(rng, NB, bs, n_tok)
        eng.gather_chunks(sm, ptrs)
        ref = torch.zeros(3 * g.chunk_bytes, dtype=torch.uint8, device="cuda:0")
        eng.gather(sm, ref.data_ptr())
        torch.cuda.synchronize()
        for i, s in enumerate(order):
            n = min(C, n_tok - i * C)
            a = chunk_tokens_of(tier[s].cpu().numpy(), g, n)
            b = chunk_tokens_of(ref.cpu().numpy()[i * g.chunk_bytes:], g, n)
            assert np.array_equal(a, b), (fmt, i)
        out = [torch.zeros_like(t) for t in dev]
        eng2 = KVEngine(g, None, 0, staging_bytes=0)
        eng2.register_kv_caches(out)
        eng2.scatter_chunks(dm, ptrs)
        torch.cuda.synchronize()
        expect = _expected_pages(fmt, host, sm, dm, C, [np.zeros_like(h) for h in host])
        for a, e in zip(out, expect):
            assert np.array_equal(host_of(a), e)
        eng2.close()
        eng.close()


def _producer(eid, ready, stop, shm_dir, L, NB, bs):
    sys.path[:0] = [ROOT, os.path.join(ROOT, "production-stack_b200")]
    import torch
    from b200kv import KVEngine, KVGeometry, _lib, pd
    pd.SHM_DIR = shm_dir
    g = torch.Generator(device="cuda:0").manual_seed(42)
    caches = [torch.randn((NB, bs, 576), generator=g, device="cuda:0").bfloat16() for _ in range(L)]
    eng = KVEngine(KVGeometry(L, 1, 576, NB, bs, 256, 2, 0, 0, _lib.LAYOUT_MLA), None, 0, staging_bytes=0)
    eng.register_kv_caches(caches)
    torch.cuda.synchronize()
    pd.publish_ipc(eid, eng, 0)
    ready.set()
    stop.wait(120)
    pd.unpublish_ipc(eid)
    eng.close()


def test_peer_pull_through_one_descriptor_per_layer(tmp_path):
    need_gpu()
    import torch.multiprocessing as mp

    from b200kv import pd
    L, NB, bs, n_tok = 4, 48, 64, 1000
    shm_dir = str(tmp_path)
    pd.SHM_DIR = shm_dir
    ctx = mp.get_context("spawn")
    ready, stop = ctx.Event(), ctx.Event()
    eid = f"mla-prod-{os.getpid()}"
    proc = ctx.Process(target=_producer, args=(eid, ready, stop, shm_dir, L, NB, bs))
    proc.start()
    try:
        assert ready.wait(180), "producer did not come up"
        local = [torch.zeros((NB, bs, D), device="cuda:0", dtype=torch.bfloat16) for _ in range(L)]
        eng = KVEngine(geom(L, NB, bs), None, 0, staging_bytes=0)
        eng.register_kv_caches(local)
        assert len(eng.export_ipc()) == L * _desc_bytes()
        pid = pd.PeerResolver(eng).resolve(eid)
        rng = np.random.default_rng(0)
        src, dst = slots(rng, NB, bs, n_tok), slots(rng, NB, bs, n_tok)
        eng.wait(eng.peer_pull(pid, src, dst))
        torch.cuda.synchronize()
        g = torch.Generator(device="cuda:0").manual_seed(42)
        want = [torch.randn((NB, bs, D), generator=g, device="cuda:0").bfloat16() for _ in range(L)]
        expect = [np.zeros((NB, bs, D), np.uint16) for _ in range(L)]
        mo.scatter_tokens(expect, mo.gather_tokens([host_of(w) for w in want], src), dst)
        for a, e in zip(local, expect):
            assert np.array_equal(host_of(a), e)
        assert eng.stats()["p2p_bytes"] == n_tok * L * D * 2
        eng.close()
    finally:
        stop.set()
        proc.join(60)


def _desc_bytes():
    import ctypes
    return ctypes.sizeof(_lib.IpcDesc)


@pytest.mark.parametrize("change,code", [
    (dict(H=2), _lib.EINVAL), (dict(fmt=FMT_Q4), _lib.ENOTSUP), (dict(fmt=FMT_FP8, D=512), _lib.ENOTSUP),
    (dict(fmt=FMT_FP8, elem=1), _lib.ENOTSUP)])
def test_refused_configurations_return_their_codes(change, code):
    need_gpu()
    p = dict(H=1, D=D, fmt=FMT_RAW, elem=2)
    p.update(change)
    g = KVGeometry(2, p["H"], p["D"], 8, 64, 256, p["elem"], 0, p["fmt"], MLA)
    with pytest.raises(B200KVError) as e:
        KVEngine(g, None, 0, staging_bytes=0)
    assert e.value.code == code


def test_register_refuses_v_pointers():
    need_gpu()
    caches = [torch.zeros((8, 64, D), device="cuda:0", dtype=torch.bfloat16) for _ in range(2)]
    eng = KVEngine(geom(2, 8, 64), None, 0, staging_bytes=0)
    with pytest.raises(ValueError):
        eng.register_kv_ptrs([c.data_ptr() for c in caches], [c.data_ptr() for c in caches])
    import ctypes
    ka = (ctypes.c_void_p * 2)(*[c.data_ptr() for c in caches])
    assert _lib.lib().b200kv_register_kv(eng._h, ka, ka) == _lib.EINVAL       # the C ABI refuses V planes too
    eng.register_kv_caches(caches)
    eng.close()
