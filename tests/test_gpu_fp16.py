"""FP8 and Q4 chunk formats on fp16 KV caches (B200KV_DTYPE_FP16), against their specification
(tests/fp16_oracle.py with dtype="fp16"): codes, scales, Q4 records, MLA latent records and
the decoded pages, bit for bit, on every path — device-resident gather/scatter (block-structured mappings: the
persistent FP8 store; token-granular ones: the cluster kernel), the pool (chunk-wise and layer-wise), the device
tier — for NHD and HND tiles; the tolerance at full Llama-3-8B size; and the refusals."""
import numpy as np
import pytest

from oracle import kv_oracle as ko
from tests import fp16_oracle as fo
from tests import mla_oracle as mo

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import b200kv  # noqa: E402
from b200kv import DTYPE_BF16, DTYPE_FP16, FMT_FP8, FMT_Q4, FMT_RAW, B200KVError, KVEngine, KVGeometry, KVPool  # noqa: E402
from b200kv import _lib  # noqa: E402
from tests.test_gpu_kernels import SMALL, bits_of, logical_bits, need_gpu  # noqa: E402

NAME = {FMT_FP8: "fp8", FMT_Q4: "q4"}


def mk_host_fp16(rng, L, NB, bs, H, D):
    """fp16 bit patterns, N(0,1) scaled per (plane, head) by e^U(-3,3): small heads reach fp16 subnormals."""
    out = []
    for _ in range(L):
        x = rng.standard_normal((2, NB, bs, H, D)).astype(np.float32)
        x *= np.exp(rng.uniform(-3, 3, (2, 1, 1, H, 1))).astype(np.float32)
        out.append(fo.f32_to_fp16_bits_rn(x).reshape(2, NB, bs, H, D))
    return out


def to_dev(layers, dev="cuda:0"):
    return [torch.from_numpy(l.view(np.int16)).view(torch.float16).to(dev) for l in layers]


def to_dev_hnd(layers, dev="cuda:0"):
    """logical (2, NB, bs, H, D) -> vLLM FlashInfer-shaped fp16 tensors: logical (NB, 2, bs, H, D) over [H][bs][D]."""
    out = []
    for l in layers:
        t = torch.from_numpy(l.view(np.int16)).view(torch.float16).to(dev)
        out.append(t.permute(1, 0, 3, 2, 4).contiguous().permute(0, 1, 3, 2, 4))
    return out


def geometry(fmt, hnd, p=SMALL, dtype=DTYPE_FP16):
    return KVGeometry(p["L"], p["H"], p["D"], p["NB"], p["bs"], p["C"], 2,
                      2 * p["bs"] * p["H"] * p["D"] * 2 if hnd else 0, fmt,
                      _lib.LAYOUT_HND if hnd else _lib.LAYOUT_NHD, dtype)


def roundtrip(fmt, bits):
    """decode(encode(bits)) of one chunk per the fp16 oracle."""
    if fmt == FMT_FP8:
        return fo.fp8_unpack_chunk(*fo.fp8_pack_chunk(bits, "fp16"), "fp16")
    return fo.q4_unpack_chunk(*fo.q4_pack_chunk(bits, "fp16"), "fp16")


def oracle_pages(host, fmt, sm, dm, C):
    dst = [np.zeros_like(l) for l in host]
    for c in range((len(sm) + C - 1) // C):
        ko.scatter_tokens(dst, roundtrip(fmt, ko.gather_tokens(host, sm[c * C:(c + 1) * C])), dm[c * C:(c + 1) * C])
    return dst


def check_chunks(got, host, fmt, hnd, sm, geom):
    """Chunk bytes vs the fp16 oracle: FP8 scales always and codes for NHD tiles (HND chunks keep the tiles' order,
    which the decoded pages check); Q4 records, token-major whatever the tiles."""
    C, L, H, D = geom.chunk_tokens, geom.n_layers, geom.n_kv_heads, geom.head_dim
    cb = geom.chunk_bytes
    for c in range((len(sm) + C - 1) // C):
        seg = sm[c * C:(c + 1) * C]
        n = len(seg)
        bits = ko.gather_tokens(host, seg)
        base = c * cb
        if fmt == FMT_FP8:
            codes, scales = fo.fp8_pack_chunk(bits, "fp16")
            so = 2 * L * C * H * D
            assert np.array_equal(got[base + so:base + so + 2 * L * H * 4].view(np.float32), scales.reshape(-1)), c
            if not hnd:
                for plane in range(2 * L):
                    o = base + plane * C * H * D
                    assert np.array_equal(got[o:o + n * H * D], codes[plane // 2, plane % 2].reshape(-1)), (c, plane)
        else:
            codes, sc = fo.q4_pack_chunk(bits, "fp16")
            rec = H * D // 2 + H * (D // 32) * 2
            for plane in range(2 * L):
                o = base + plane * C * rec
                r = got[o:o + n * rec].reshape(n, rec)
                assert np.array_equal(r[:, :H * D // 2], codes[plane // 2, plane % 2].reshape(n, -1)), (c, plane)
                assert np.array_equal(r[:, H * D // 2:].copy().view(np.uint16), sc[plane // 2, plane % 2].reshape(n, -1))


def mappings(rng, p, n_tok, granular):
    if granular:     # every token in another block, unaligned on both sides: the cluster FP8 store
        return (rng.permutation(p["NB"] * p["bs"])[:n_tok].astype(np.int64),
                rng.permutation(p["NB"] * p["bs"])[:n_tok].astype(np.int64))
    nb = (n_tok + p["bs"] - 1) // p["bs"]
    return (ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[:nb], p["bs"], n_tok),
            ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[:nb], p["bs"], n_tok))


@pytest.mark.parametrize("fmt", [FMT_FP8, FMT_Q4])
@pytest.mark.parametrize("hnd", [False, True], ids=["nhd", "hnd"])
@pytest.mark.parametrize("n_tok,granular", [(1, False), (17, False), (256, False), (300, False), (700, False),
                                            (40, True), (600, True)])
def test_fp16_gather_scatter_vs_oracle(fmt, hnd, n_tok, granular):
    need_gpu()
    p = SMALL
    rng = np.random.default_rng(7000 + n_tok + 10 * hnd + 100 * fmt)
    host = mk_host_fp16(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev_hnd(host) if hnd else to_dev(host)
    geom = geometry(fmt, hnd)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    sm, dm = mappings(rng, p, n_tok, granular)
    n_chunks = (n_tok + p["C"] - 1) // p["C"]
    buf = torch.zeros(n_chunks * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    check_chunks(buf.cpu().numpy(), host, fmt, hnd, sm, geom)
    for t in dev:
        t.zero_()
    eng.scatter(dm, buf.data_ptr())
    torch.cuda.synchronize()
    get = logical_bits if hnd else bits_of
    for a, b in zip(dev, oracle_pages(host, fmt, sm, dm, p["C"])):
        assert np.array_equal(get(a), b)
    eng.close()


@pytest.mark.parametrize("fmt", [FMT_FP8, FMT_Q4])
@pytest.mark.parametrize("hnd", [False, True], ids=["nhd", "hnd"])
@pytest.mark.parametrize("group", [0, 2], ids=["chunkwise", "layerwise"])
def test_fp16_pool_round_trip_vs_oracle(fmt, hnd, group):
    """KVEngine.store / retrieve through the pinned pool, a partial last chunk, chunk-wise and layer-wise loads."""
    need_gpu()
    p = SMALL
    rng = np.random.default_rng(8100 + 10 * hnd + fmt + 100 * group)
    host = mk_host_fp16(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev_hnd(host) if hnd else to_dev(host)
    geom = geometry(fmt, hnd)
    pool = KVPool(None, 8 * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=4 * geom.chunk_bytes)
    eng.register_kv_caches(dev)
    n = 2 * p["C"] + 37
    toks = rng.integers(0, 128256, n).astype(np.int32)
    sm, dm = mappings(rng, p, n, False)
    eng.wait(eng.store(toks, None, sm))
    assert eng.lookup(toks) == n
    for t in dev:
        t.zero_()
    ret, ticket = eng.retrieve(toks, None, dm, return_ticket=True, layers_per_group=group)
    assert ret.all()
    if ticket:
        eng.wait(ticket)
    torch.cuda.synchronize()
    get = logical_bits if hnd else bits_of
    for a, b in zip(dev, oracle_pages(host, fmt, sm, dm, p["C"])):
        assert np.array_equal(get(a), b)
    eng.close()
    pool.close()


@pytest.mark.parametrize("fmt", [FMT_FP8, FMT_Q4])
def test_fp16_device_tier_vs_oracle(fmt):
    """gather_chunks / scatter_chunks through device tier slots: the same chunk bytes as gather, the oracle's pages."""
    need_gpu()
    p = SMALL
    rng = np.random.default_rng(8300 + fmt)
    host = mk_host_fp16(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev(host)
    geom = geometry(fmt, False)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    n = 2 * p["C"] + 90
    sm, dm = mappings(rng, p, n, False)
    slots = torch.zeros((4, geom.chunk_bytes), dtype=torch.uint8, device="cuda:0")   # tier slots, taken in any order
    order = (3, 0, 2)
    eng.gather_chunks(sm, [slots[s].data_ptr() for s in order])
    torch.cuda.synchronize()
    got = slots.cpu().numpy()[list(order)].reshape(-1)
    check_chunks(got, host, fmt, False, sm, geom)
    for t in dev:
        t.zero_()
    eng.scatter_chunks(dm, [slots[s].data_ptr() for s in order])
    torch.cuda.synchronize()
    for a, b in zip(dev, oracle_pages(host, fmt, sm, dm, p["C"])):
        assert np.array_equal(bits_of(a), b)
    eng.close()


@pytest.mark.parametrize("bs", [16, 64])
def test_fp16_mla_records_and_pages_vs_oracle(bs):
    need_gpu()
    L, NB, C_, D = 3, 48, 256, mo.MLA_D
    rng = np.random.default_rng(8500 + bs)
    host = []
    for _ in range(L):
        x = rng.standard_normal((NB, bs, D)).astype(np.float32) * np.exp(rng.uniform(-3, 3, (NB, bs, 1))).astype(np.float32)
        host.append(fo.f32_to_fp16_bits_rn(x).reshape(NB, bs, D))
    dev = [torch.from_numpy(l.view(np.int16)).view(torch.float16).cuda() for l in host]
    geom = KVGeometry(L, 1, D, NB, bs, C_, 2, 0, FMT_FP8, _lib.LAYOUT_MLA, DTYPE_FP16)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    n = C_ + 3 * bs + 5
    nb = (n + bs - 1) // bs
    sm = ko.slot_mapping_from_blocks(rng.permutation(NB)[:nb], bs, n)
    dm = ko.slot_mapping_from_blocks(rng.permutation(NB)[:nb], bs, n)
    n_chunks = (n + C_ - 1) // C_
    buf = torch.zeros(n_chunks * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    want_pages = [np.zeros_like(l) for l in host]
    for c in range(n_chunks):
        seg_s, seg_d = sm[c * C_:(c + 1) * C_], dm[c * C_:(c + 1) * C_]
        rec = fo.mla_fp8_pack_chunk(mo.gather_tokens(host, seg_s), "fp16")          # (L, n, 656)
        for l in range(L):
            o = c * geom.chunk_bytes + l * C_ * mo.MLA_RECORD
            assert np.array_equal(got[o:o + len(seg_s) * mo.MLA_RECORD].reshape(len(seg_s), -1), rec[l]), (c, l)
        mo.scatter_tokens(want_pages, fo.mla_fp8_unpack_chunk(rec, "fp16"), seg_d)
    for t in dev:
        t.zero_()
    eng.scatter(dm, buf.data_ptr())
    torch.cuda.synchronize()
    for a, b in zip(dev, want_pages):
        assert np.array_equal(bits_of(a), b)
    eng.close()


@pytest.mark.parametrize("fmt", [FMT_FP8, FMT_Q4])
def test_fp16_tolerance_at_baseline_size(fmt):
    """L = 32, H = 8, D = 128, 8K tokens: decoded values are finite and within the oracle's fp16 tolerance
    (restated in torch on the GPU: the oracle's float64 arrays would take tens of GB at this size)."""
    need_gpu()
    L, H, D, bs, C_, n = 32, 8, 128, 16, 256, 8192
    NB = n // bs
    g = torch.Generator(device="cuda:0").manual_seed(8700 + fmt)
    src = []
    for _ in range(L):
        x = torch.randn((2, NB, bs, H, D), generator=g, device="cuda:0")
        x *= torch.exp(torch.empty((2, 1, 1, H, 1), device="cuda:0").uniform_(-3, 3, generator=g))
        src.append(x.half())
    dev = [t.clone() for t in src]
    geom = KVGeometry(L, H, D, NB, bs, C_, 2, 0, fmt, 0, DTYPE_FP16)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    sm = np.arange(n, dtype=np.int64)
    buf = torch.empty((n // C_) * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    for t in dev:
        t.zero_()
    eng.scatter(sm, buf.data_ptr())
    torch.cuda.synchronize()
    for l in range(L):
        x = src[l].double()                     # (2, NB, bs, H, D), chunk c = blocks [16c, 16c + 16)
        y = dev[l].double()
        assert torch.isfinite(y).all()
        ax = x.abs()
        if fmt == FMT_FP8:
            amax = ax.reshape(2, n // C_, C_, H, D).amax(dim=(2, 4), keepdim=True)
            q = torch.maximum(ax.reshape(2, n // C_, C_, H, D) * 2.0 ** -4, 2.0 ** -10 * amax).reshape(x.shape)
            tol = q + ax * 2.0 ** -11 + 2.0 ** -25
        else:
            amax = ax.reshape(*x.shape[:-1], D // 32, 32).amax(dim=-1, keepdim=True)
            tol = (amax / 7.0 * (1 + 2.0 ** -7) / 2).expand(*x.shape[:-1], D // 32, 32).reshape(x.shape) \
                + ax * 2.0 ** -11 + 2.0 ** -25
        bad = ((x - y).abs() > tol).sum().item()
        assert bad == 0, (l, bad)
    eng.close()


def test_fp16_refusals_and_isolation():
    need_gpu()
    p = SMALL
    # fp16 needs a 16-bit element
    with pytest.raises(B200KVError) as ei:
        KVEngine(KVGeometry(2, 4, 64, 16, 16, 64, 1, 0, FMT_RAW, 0, DTYPE_FP16), None, 0, staging_bytes=0)
    assert ei.value.code == _lib.EINVAL
    rng = np.random.default_rng(8900)
    host = mk_host_fp16(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    # the type is fixed once the cache is registered
    eng = KVEngine(geometry(FMT_FP8, False), None, 0, staging_bytes=0)
    eng.register_kv_caches(to_dev(host))
    with pytest.raises(B200KVError) as ei:
        eng.set_cache_dtype(DTYPE_BF16)
    assert ei.value.code == _lib.EBUSY
    eng.close()
    # a lossy engine refuses a cache of the other 16-bit type, either way round
    for fmt in (FMT_FP8, FMT_Q4):
        e16 = KVEngine(geometry(fmt, False), None, 0, staging_bytes=0)
        with pytest.raises(ValueError):
            e16.register_kv_caches([t.view(torch.bfloat16) for t in to_dev(host)])
        e16.close()
        ebf = KVEngine(geometry(fmt, False, dtype=DTYPE_BF16), None, 0, staging_bytes=0)
        with pytest.raises(ValueError):
            ebf.register_kv_caches(to_dev(host))
        ebf.close()
    # RAW moves bytes: any 16-bit type registers
    er = KVEngine(geometry(FMT_RAW, False, dtype=DTYPE_BF16), None, 0, staging_bytes=0)
    er.register_kv_caches(to_dev(host))
    er.close()
    # a pool shared by a bf16 and an fp16 engine (same keys) never hands one's chunks to the other
    for fmt in (FMT_RAW, FMT_FP8):
        g16, gbf = geometry(fmt, False), geometry(fmt, False, dtype=DTYPE_BF16)
        pool = KVPool(None, 4 * g16.chunk_bytes, g16.chunk_bytes, 1)
        e16 = KVEngine(g16, pool, 0, staging_bytes=2 * g16.chunk_bytes, key_seed=1)
        ebf = KVEngine(gbf, pool, 0, staging_bytes=2 * gbf.chunk_bytes, key_seed=1)
        e16.register_kv_caches(to_dev(host))
        ebf.register_kv_caches([t.view(torch.bfloat16) for t in to_dev(host)])
        toks = np.arange(256, dtype=np.int32)
        sm = ko.slot_mapping_from_blocks(np.arange(16), 16, 256)
        e16.wait(e16.store(toks, None, sm))
        assert ebf.retrieve(toks, None, sm).sum() == 0 and e16.retrieve(toks, None, sm).all()
        torch.cuda.synchronize()
        e16.close()
        ebf.close()
        pool.close()
