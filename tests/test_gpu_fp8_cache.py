"""Q4 chunks of fp8 KV caches (e4m3 and e5m2 pages, B200KV_DTYPE_E4M3 / B200KV_DTYPE_E5M2) against their
specification, tests/fp8_cache_oracle.py: Q4 records and decoded pages bit for bit, for NHD and HND tiles, one and
eight heads, head sizes 64 to 256, block sizes 16 and 64, block-aligned, token-granular and ragged-tail mappings,
every code as a group maximum; the pool chunk-wise, layer-wise and batched; RAW round trips of uint8 pages; e4m3 and
e5m2 chunks kept apart in one pool; FP8 on an fp8 cache stored RAW; and the refusals."""
from types import SimpleNamespace as NS

import numpy as np
import pytest

from oracle import kv_oracle as ko
from tests import fp8_cache_oracle as fo

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from b200kv import FMT_FP8, FMT_Q4, FMT_RAW, B200KVError, KVEngine, KVGeometry, KVPool  # noqa: E402
from b200kv import _lib  # noqa: E402
from tests.test_gpu_kernels import need_gpu  # noqa: E402

DTYPE = {"e4m3": _lib.DTYPE_E4M3, "e5m2": _lib.DTYPE_E5M2}
C = 256


def finite_codes(ft):
    dec = fo.decode_table(ft)
    return np.array([c for c in range(256) if np.isfinite(dec[c])], np.uint8)


def mk_host(rng, ft, L, NB, bs, H, D):
    """fp8 codes, (2, NB, bs, H, D) per layer: every finite code for half the heads, a window of four binades
    (narrow groups, small scales) for the others."""
    fin = finite_codes(ft)
    out = []
    for _ in range(L):
        x = rng.choice(fin, size=(2, NB, bs, H, D)).astype(np.uint8)
        narrow = rng.choice(fin[(fin & 0x7F) < 0x30], size=(2, NB, bs, H, D)).astype(np.uint8)
        x[:, :, :, 1::2] = narrow[:, :, :, 1::2]
        out.append(x)
    return out


def to_dev(layers, dev="cuda:0"):
    return [torch.from_numpy(l).to(dev) for l in layers]


def to_dev_hnd(layers, dev="cuda:0"):
    """logical (2, NB, bs, H, D) -> vLLM FlashInfer-shaped uint8 tensors: logical (NB, 2, bs, H, D) over [H][bs][D]."""
    return [torch.from_numpy(l).to(dev).permute(1, 0, 3, 2, 4).contiguous().permute(0, 1, 3, 2, 4) for l in layers]


def pages_of(t, hnd):
    t = t.permute(1, 0, 2, 3, 4) if hnd else t
    return t.contiguous().cpu().numpy()


def geometry(ft, fmt, hnd, L, NB, bs, H, D):
    return KVGeometry(L, H, D, NB, bs, C, 1, 2 * bs * H * D if hnd else 0, fmt,
                      _lib.LAYOUT_HND if hnd else _lib.LAYOUT_NHD, fp8_dtype=DTYPE[ft])


def roundtrip(ft, codes):
    return fo.q4_unpack_chunk(*fo.q4_pack_chunk(codes, ft), ft)


def oracle_pages(host, ft, sm, dm, dst=None):
    dst = [np.zeros_like(l) for l in host] if dst is None else dst
    for c in range((len(sm) + C - 1) // C):
        ko.scatter_tokens(dst, roundtrip(ft, ko.gather_tokens(host, sm[c * C:(c + 1) * C])), dm[c * C:(c + 1) * C])
    return dst


def check_records(got, host, ft, sm, geom):
    """Q4 records (token-major whatever the tiles) vs the oracle: codes and bf16 scales."""
    L, H, D = geom.n_layers, geom.n_kv_heads, geom.head_dim
    rec = H * D // 2 + H * (D // 32) * 2
    for c in range((len(sm) + C - 1) // C):
        seg = sm[c * C:(c + 1) * C]
        n = len(seg)
        codes, sc = fo.q4_pack_chunk(ko.gather_tokens(host, seg), ft)
        for plane in range(2 * L):
            o = c * geom.chunk_bytes + plane * C * rec
            r = got[o:o + n * rec].reshape(n, rec)
            assert np.array_equal(r[:, :H * D // 2], codes[plane // 2, plane % 2].reshape(n, -1)), (c, plane)
            assert np.array_equal(r[:, H * D // 2:].copy().view(np.uint16), sc[plane // 2, plane % 2].reshape(n, -1))


def gather_scatter_check(eng, dev, host, ft, hnd, sm, dm, geom):
    n_chunks = (len(sm) + C - 1) // C
    buf = torch.zeros(n_chunks * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    check_records(buf.cpu().numpy(), host, ft, sm, geom)
    for t in dev:
        t.zero_()
    eng.scatter(dm, buf.data_ptr())
    torch.cuda.synchronize()
    for a, b in zip(dev, oracle_pages(host, ft, sm, dm)):
        assert np.array_equal(pages_of(a, hnd), b)


@pytest.mark.parametrize("ft", fo.FP8_TYPES)
@pytest.mark.parametrize("hnd", [False, True], ids=["nhd", "hnd"])
@pytest.mark.parametrize("H", [1, 8])
@pytest.mark.parametrize("D", [64, 128, 256])
@pytest.mark.parametrize("bs", [16, 64])
def test_q4_fp8_gather_scatter_vs_oracle(ft, hnd, H, D, bs):
    """Block-aligned runs with a ragged tail (300 tokens: a partial chunk, and a partial HND tile), then
    token-granular mappings (every token in another block, unaligned on both sides)."""
    need_gpu()
    L, NB = 2, 768 // bs
    rng = np.random.default_rng([ft == "e5m2", hnd, H, D, bs])
    host = mk_host(rng, ft, L, NB, bs, H, D)
    dev = to_dev_hnd(host) if hnd else to_dev(host)
    geom = geometry(ft, FMT_Q4, hnd, L, NB, bs, H, D)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    n = 300
    nb = (n + bs - 1) // bs
    sm = ko.slot_mapping_from_blocks(rng.permutation(NB)[:nb], bs, n)
    dm = ko.slot_mapping_from_blocks(rng.permutation(NB)[:nb], bs, n)
    gather_scatter_check(eng, dev, host, ft, hnd, sm, dm, geom)
    for t, s in zip(dev, to_dev_hnd(host) if hnd else to_dev(host)):
        t.copy_(s)
    sm = rng.permutation(NB * bs)[:40].astype(np.int64)
    dm = rng.permutation(NB * bs)[:40].astype(np.int64)
    gather_scatter_check(eng, dev, host, ft, hnd, sm, dm, geom)
    eng.close()


@pytest.mark.parametrize("ft", fo.FP8_TYPES)
@pytest.mark.parametrize("hnd", [False, True], ids=["nhd", "hnd"])
def test_q4_fp8_every_code_as_group_maximum(ft, hnd):
    """All 256 codes, NaN and inf included, each the maximum of one group: records and pages as the oracle says."""
    need_gpu()
    L, NB, bs, H, D = 1, 16, 16, 8, 128
    rng = np.random.default_rng(31 + hnd)
    dec = fo.decode_table(ft)
    groups = np.zeros((256, 32), np.uint8)
    for c in range(256):
        below = [k for k in range(c & 0x7F) if np.isfinite(dec[k])] or [0]
        groups[c] = np.concatenate([[c], rng.choice(below, 31) | (rng.integers(0, 2, 31) << 7)]).astype(np.uint8)
    host = mk_host(rng, ft, L, NB, bs, H, D)
    host[0][0, 0, :8] = groups.reshape(8, H, D)                 # tokens 0..7 of the K plane: 32 groups each
    host[0][1, 0, 8:16] = groups[::-1].reshape(8, H, D)         # tokens 8..15 of the V plane
    dev = to_dev_hnd(host) if hnd else to_dev(host)
    geom = geometry(ft, FMT_Q4, hnd, L, NB, bs, H, D)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    sm = np.arange(64, dtype=np.int64)
    dm = np.arange(64, 128, dtype=np.int64)
    gather_scatter_check(eng, dev, host, ft, hnd, sm, dm, geom)
    eng.close()


@pytest.mark.parametrize("ft", fo.FP8_TYPES)
@pytest.mark.parametrize("hnd", [False, True], ids=["nhd", "hnd"])
@pytest.mark.parametrize("mode", ["chunkwise", "layerwise", "batch"])
def test_q4_fp8_pool_round_trip_vs_oracle(ft, hnd, mode):
    """KVEngine.store / retrieve through the pinned pool with a partial last chunk: chunk-wise, layer-wise, and two
    requests in one batched op."""
    need_gpu()
    L, NB, bs, H, D = 3, 96, 16, 8, 128
    rng = np.random.default_rng(900 + 10 * hnd + len(mode) + (ft == "e5m2"))
    host = mk_host(rng, ft, L, NB, bs, H, D)
    dev = to_dev_hnd(host) if hnd else to_dev(host)
    geom = geometry(ft, FMT_Q4, hnd, L, NB, bs, H, D)
    pool = KVPool(None, 12 * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=4 * geom.chunk_bytes)
    eng.register_kv_caches(dev)
    lens = [2 * C + 37, C + 100] if mode == "batch" else [2 * C + 37]
    perm_s, perm_d = rng.permutation(NB), rng.permutation(NB)
    reqs, b0 = [], 0
    for n in lens:
        nb = (n + bs - 1) // bs
        toks = rng.integers(0, 128256, n).astype(np.int32)
        reqs.append((toks, ko.slot_mapping_from_blocks(perm_s[b0:b0 + nb], bs, n),
                     ko.slot_mapping_from_blocks(perm_d[b0:b0 + nb], bs, n)))
        b0 += nb
    if mode == "batch":
        eng.wait(eng.store_batch([(t, s, 0) for t, s, _ in reqs]))
    else:
        eng.wait(eng.store(reqs[0][0], None, reqs[0][1]))
    for t, _, _ in reqs:
        assert eng.lookup(t) == len(t)
    want = [np.zeros_like(l) for l in host]
    for _, s, d in reqs:
        oracle_pages(host, ft, s, d, want)
    for t in dev:
        t.zero_()
    if mode == "batch":
        loaded, ticket = eng.retrieve_batch([(t, d, 0) for t, _, d in reqs])
        assert list(loaded) == lens
    else:
        ret, ticket = eng.retrieve(reqs[0][0], None, reqs[0][2], return_ticket=True,
                                   layers_per_group=2 if mode == "layerwise" else 0)
        assert ret.all()
    if ticket:
        eng.wait(ticket)
    torch.cuda.synchronize()
    for a, b in zip(dev, want):
        assert np.array_equal(pages_of(a, hnd), b)
    eng.close()
    pool.close()


@pytest.mark.parametrize("ft", fo.FP8_TYPES)
@pytest.mark.parametrize("hnd", [False, True], ids=["nhd", "hnd"])
def test_raw_fp8_pages_round_trip(ft, hnd):
    """RAW moves uint8 pages verbatim, every code included, through the pool."""
    need_gpu()
    L, NB, bs, H, D = 2, 64, 16, 8, 128
    rng = np.random.default_rng(77 + hnd)
    host = [rng.integers(0, 256, (2, NB, bs, H, D)).astype(np.uint8) for _ in range(L)]
    dev = to_dev_hnd(host) if hnd else to_dev(host)
    geom = geometry(ft, FMT_RAW, hnd, L, NB, bs, H, D)
    pool = KVPool(None, 8 * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=4 * geom.chunk_bytes)
    eng.register_kv_caches(dev)
    n = C + 77
    toks = rng.integers(0, 128256, n).astype(np.int32)
    sm = ko.slot_mapping_from_blocks(rng.permutation(NB)[:21], bs, n)
    dm = ko.slot_mapping_from_blocks(rng.permutation(NB)[:21], bs, n)
    eng.wait(eng.store(toks, None, sm))
    for t in dev:
        t.zero_()
    ret, ticket = eng.retrieve(toks, None, dm, return_ticket=True)
    assert ret.all()
    if ticket:
        eng.wait(ticket)
    torch.cuda.synchronize()
    want = [np.zeros_like(l) for l in host]
    ko.scatter_tokens(want, ko.gather_tokens(host, sm), dm)
    for a, b in zip(dev, want):
        assert np.array_equal(pages_of(a, hnd), b)
    eng.close()
    pool.close()


@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_Q4])
def test_e5m2_engine_gets_no_hit_on_e4m3_chunks(fmt):
    need_gpu()
    L, NB, bs, H, D = 2, 32, 16, 8, 128
    rng = np.random.default_rng(5)
    host = mk_host(rng, "e4m3", L, NB, bs, H, D)
    g4, g5 = geometry("e4m3", fmt, False, L, NB, bs, H, D), geometry("e5m2", fmt, False, L, NB, bs, H, D)
    pool = KVPool(None, 4 * g4.chunk_bytes, g4.chunk_bytes, 1)
    e4 = KVEngine(g4, pool, 0, staging_bytes=2 * g4.chunk_bytes, key_seed=1)    # same keys on purpose
    e5 = KVEngine(g5, pool, 0, staging_bytes=2 * g5.chunk_bytes, key_seed=1)
    e4.register_kv_caches(to_dev(host))
    e5.register_kv_caches(to_dev(host))
    toks = np.arange(C, dtype=np.int32)
    sm = ko.slot_mapping_from_blocks(np.arange(16), bs, C)
    e4.wait(e4.store(toks, None, sm))
    assert e5.retrieve(toks, None, sm).sum() == 0 and e4.retrieve(toks, None, sm).all()
    torch.cuda.synchronize()
    e4.close()
    e5.close()
    pool.close()


def test_fp8_format_on_fp8_cache_stores_raw_chunks():
    """B200KV_FORMAT=fp8 with --kv-cache-dtype fp8: the geometry is RAW, so an explicitly RAW e4m3 engine sharing the
    pool and keys hits its chunks, and they hold the pages' bytes."""
    need_gpu()
    pytest.importorskip("vllm")
    from b200kv.config import B200KVConfig
    from b200kv.connector import geometry_from_vllm
    L, NB, bs, H, D = 2, 32, 16, 8, 128
    mc = NS(model="synth", dtype=torch.bfloat16, use_mla=False, get_num_layers=lambda pc: L,
            get_num_kv_heads=lambda pc: H, get_head_size=lambda: D)
    vc = NS(model_config=mc, parallel_config=NS(tensor_parallel_size=1, rank=0),
            cache_config=NS(block_size=bs, cache_dtype="fp8"))
    cfg = B200KVConfig()
    cfg.fmt = FMT_FP8
    g = geometry_from_vllm(vc, cfg, n_blocks=NB)
    assert (g.fmt, g.elem_bytes, g.cache_dtype, g.fmt_tag) == (FMT_RAW, 1, _lib.DTYPE_E4M3, 0)
    rng = np.random.default_rng(9)
    host = mk_host(rng, "e4m3", L, NB, bs, H, D)
    pool = KVPool(None, 4 * g.chunk_bytes, g.chunk_bytes, 1)
    ea = KVEngine(g, pool, 0, staging_bytes=2 * g.chunk_bytes, key_seed=3)
    eb = KVEngine(geometry("e4m3", FMT_RAW, False, L, NB, bs, H, D), pool, 0, staging_bytes=2 * g.chunk_bytes,
                  key_seed=3)
    dev_a, dev_b = to_dev(host), [torch.zeros((2, NB, bs, H, D), dtype=torch.uint8, device="cuda:0") for _ in range(L)]
    ea.register_kv_caches(dev_a)
    eb.register_kv_caches(dev_b)
    toks = np.arange(C, dtype=np.int32)
    sm = ko.slot_mapping_from_blocks(np.arange(16), bs, C)
    ea.wait(ea.store(toks, None, sm))
    ret, ticket = eb.retrieve(toks, None, sm, return_ticket=True)
    assert ret.all()
    if ticket:
        eb.wait(ticket)
    torch.cuda.synchronize()
    for a, b in zip(dev_a, dev_b):
        assert torch.equal(a[:, :16], b[:, :16])
    ea.close()
    eb.close()
    pool.close()


def test_fp8_dtype_refusals():
    need_gpu()
    L, NB, bs, H, D = 2, 16, 16, 8, 128
    # E5M2 needs a 1-byte element, FP16 a 2-byte one
    with pytest.raises(B200KVError) as ei:
        KVEngine(KVGeometry(L, H, D, NB, bs, C, 2, 0, FMT_RAW, 0, fp8_dtype=_lib.DTYPE_E5M2), None, 0,
                 staging_bytes=0)
    assert ei.value.code == _lib.EINVAL
    with pytest.raises(B200KVError) as ei:
        KVEngine(KVGeometry(L, H, D, NB, bs, C, 1, 0, FMT_RAW, 0, _lib.DTYPE_FP16), None, 0, staging_bytes=0)
    assert ei.value.code == _lib.EINVAL
    host = mk_host(np.random.default_rng(1), "e5m2", L, NB, bs, H, D)
    eng = KVEngine(geometry("e5m2", FMT_Q4, False, L, NB, bs, H, D), None, 0, staging_bytes=0)
    # a tensor that names its fp8 type must be the engine's; a uint8 one (vLLM's) is taken as the geometry says
    with pytest.raises(ValueError, match="float8_e5m2"):
        eng.register_kv_caches([t.view(torch.float8_e4m3fn) for t in to_dev(host)])
    eng.register_kv_caches([t.view(torch.float8_e5m2) for t in to_dev(host)])
    with pytest.raises(B200KVError) as ei:          # the type is fixed once the cache is registered
        eng.set_cache_dtype(_lib.DTYPE_E4M3)
    assert ei.value.code == _lib.EBUSY
    eng.close()
    # FP8 of fp8 pages stays refused by the engine
    with pytest.raises(B200KVError) as ei:
        KVEngine(geometry("e4m3", FMT_FP8, False, L, NB, bs, H, D), None, 0, staging_bytes=0)
    assert ei.value.code == _lib.ENOTSUP
