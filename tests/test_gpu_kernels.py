"""GPU parity tests (run on an H100 with -m gpu): every CUDA path, called through the C ABI,
against the oracle on the same seeded inputs — bit-exact for RAW and for the FP8 codes/scales."""
import numpy as np
import pytest

from oracle import kv_oracle as ko
from tests import oracle_c

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

import b200kv  # noqa: E402
from b200kv import FMT_FP8, FMT_RAW, VARIANT_BULK, VARIANT_LDG, KVEngine, KVGeometry, KVPool  # noqa: E402


def need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device: the product has no CPU fallback")


def bits_of(t):  # torch bf16 tensor -> numpy uint16
    return t.detach().cpu().contiguous().view(torch.int16).numpy().view(np.uint16)


def mk_host_layers(rng, L, NB, bs, H, D):
    out = []
    for _ in range(L):
        x = rng.standard_normal((2, NB, bs, H, D)).astype(np.float32)
        x *= np.exp(rng.uniform(-3, 3, (2, 1, 1, H, 1))).astype(np.float32)
        out.append(ko.f32_to_bf16_bits_rn(x).reshape(2, NB, bs, H, D))
    return out


def to_dev(layers, dev="cuda:0"):
    return [torch.from_numpy(l.view(np.int16)).view(torch.bfloat16).to(dev) for l in layers]


SMALL = dict(L=3, NB=96, bs=16, H=8, D=128, C=256)


@pytest.mark.parametrize("variant", [VARIANT_BULK, VARIANT_LDG])
@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_FP8])
@pytest.mark.parametrize("n_tok", [1, 15, 16, 17, 255, 256, 257, 700, 1024])
def test_gather_scatter_device_resident_vs_oracle(variant, fmt, n_tok):
    need_gpu()
    if fmt == FMT_FP8 and variant == VARIANT_LDG:
        pytest.skip("variant only selects the RAW copy kernel")
    p = SMALL
    rng = np.random.default_rng(1000 + n_tok)
    host = mk_host_layers(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev(host)
    geom = KVGeometry(p["L"], p["H"], p["D"], p["NB"], p["bs"], p["C"], 2, 0, fmt)
    eng = KVEngine(geom, None, 0, staging_bytes=0, variant=variant)
    eng.register_kv_caches(dev)
    nb = (n_tok + p["bs"] - 1) // p["bs"]
    sm = ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[:nb], p["bs"], n_tok)
    dm = ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[:nb], p["bs"], n_tok)
    n_chunks = (n_tok + p["C"] - 1) // p["C"]
    buf = torch.zeros(n_chunks * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    name = "fp8" if fmt == FMT_FP8 else "raw"
    want, cb, so = oracle_c.gather(host, sm, p["C"], name)
    assert cb == geom.chunk_bytes
    got = buf.cpu().numpy()
    # compare only bytes that carry tokens (the tail of a partial chunk is unspecified)
    for c in range(n_chunks):
        n = min(p["C"], n_tok - c * p["C"])
        tb = geom.token_bytes // (2 if fmt == FMT_FP8 else 1)
        for plane in range(2 * p["L"]):
            o = c * cb + plane * p["C"] * tb
            assert np.array_equal(got[o:o + n * tb], want[o:o + n * tb]), (c, plane)
        if fmt == FMT_FP8:
            s = c * cb + so
            assert np.array_equal(got[s:s + 2 * p["L"] * p["H"] * 4], want[s:s + 2 * p["L"] * p["H"] * 4])
    # scatter back into zeroed pages at other blocks
    for t in dev:
        t.zero_()
    eng.scatter(dm, buf.data_ptr())
    torch.cuda.synchronize()
    dst = [np.zeros_like(l) for l in host]
    oracle_c.scatter(dst, dm, p["C"], want, cb, so, name)
    for a, b in zip(dev, dst):
        assert np.array_equal(bits_of(a), b)
    assert eng.stats()["n_kernel_launches"] == 2
    assert eng.last_kernel_ms(0) > 0 and eng.last_kernel_ms(1) > 0
    eng.close()


@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_FP8])
def test_store_retrieve_through_pool_vs_oracle_engine(fmt):
    """lmcache_engine.store / .retrieve call shapes of the adapter (masks, offsets, partial
    chunk, dedupe, prefix stop) — same calls into the oracle engine and the CUDA engine."""
    need_gpu()
    p = SMALL
    rng = np.random.default_rng(7)
    host = mk_host_layers(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev(host)
    geom = KVGeometry(p["L"], p["H"], p["D"], p["NB"], p["bs"], p["C"], 2, 0, fmt)
    pool = KVPool(None, 6 * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=2 * geom.chunk_bytes)   # ring smaller than the op
    eng.register_kv_caches(dev)
    oe = ko.OracleEngine(p["C"], "fp8" if fmt == FMT_FP8 else "raw")
    n = 3 * p["C"] + 37
    toks = rng.integers(0, 128256, n).astype(np.int32)
    sm = ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[: (n + 15) // 16], 16, n)
    # 1) store with chunk 0 masked out (offset = C): engine must not see a prefix hit
    mask = np.ones(n, bool)
    mask[: p["C"]] = False
    eng.wait(eng.store(toks, mask, sm, offset=p["C"]))
    oe.store(toks, mask, host, sm, offset=p["C"])
    assert eng.lookup(toks) == oe.lookup(toks) == 0
    # 2) full store: only chunk 0 is new
    before = pool.stats()["n_stored_chunks"]
    eng.wait(eng.store(toks, None, sm))
    oe.store(toks, np.ones(n, bool), host, sm)
    assert pool.stats()["n_stored_chunks"] - before == 1
    assert eng.lookup(toks) == oe.lookup(toks) == n
    assert eng.lookup(toks[: 2 * p["C"] + 5]) == oe.lookup(toks[: 2 * p["C"] + 5]) == 2 * p["C"]
    # 3) retrieve with the first chunk masked (vLLM prefix-cache hit), into other blocks
    dm = ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[: (n + 15) // 16], 16, n)
    for t in dev:
        t.zero_()
    ret = eng.retrieve(toks, mask, dm)
    torch.cuda.synchronize()
    dst = [np.zeros_like(l) for l in host]
    want = oe.retrieve(toks, mask, dst, dm)
    assert np.array_equal(ret, want)
    for a, b in zip(dev, dst):
        assert np.array_equal(bits_of(a), b)
    # 4) a request sharing only the first two chunks: retrieve stops at the first miss
    toks2 = toks.copy()
    toks2[2 * p["C"] + 3] += 1
    ret2 = eng.retrieve(toks2, None, dm)
    want2 = oe.retrieve(toks2, np.ones(n, bool), [np.zeros_like(l) for l in host], dm)
    assert np.array_equal(ret2, want2) and ret2.sum() == 2 * p["C"]
    eng.wait_all()
    st = eng.stats()
    assert st["d2h_bytes"] > 0 and st["h2d_bytes"] > 0 and st["n_kernel_launches"] >= 4
    eng.close()
    pool.close()


def test_fp8_dequantised_values_within_stated_tolerance():
    need_gpu()
    p = SMALL
    rng = np.random.default_rng(11)
    host = mk_host_layers(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev(host)
    geom = KVGeometry(p["L"], p["H"], p["D"], p["NB"], p["bs"], p["C"], 2, 0, FMT_FP8)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    n = 512
    sm = ko.slot_mapping_from_blocks(np.arange(n // 16), 16, n)
    buf = torch.zeros(2 * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    for t in dev:
        t.zero_()
    eng.scatter(sm, buf.data_ptr())
    torch.cuda.synchronize()
    for l in range(p["L"]):
        x = ko.bf16_bits_to_f32(host[l][:, : n // 16])
        y = ko.bf16_bits_to_f32(bits_of(dev[l])[:, : n // 16])
        # tolerance from SURVEY §8c: max(2^-4|x|, 2^-10 absmax) + 2^-8|x|, absmax per (chunk,plane,head)
        xc = x.reshape(2, 2, 16, 16, p["H"], p["D"])          # (kv, chunk, blocks, tok, H, D)
        amax = np.abs(xc).max(axis=(2, 3, 5), keepdims=True)
        tol = np.maximum(np.abs(xc) * 2.0 ** -4, amax * 2.0 ** -10) + np.abs(xc) * 2.0 ** -8
        assert (np.abs(y.reshape(xc.shape) - xc) <= tol).all()
    eng.close()


def test_token_granular_slot_mapping_and_other_layouts():
    """Arbitrary (non block-structured) slot mappings, FlashInfer (NB,2,..) and cross-layer
    (NB,L,2,..) paged layouts: same bytes as the oracle."""
    need_gpu()
    L, NB, bs, H, D, C_ = 2, 64, 16, 4, 64, 64
    rng = np.random.default_rng(21)
    host = mk_host_layers(rng, L, NB, bs, H, D)
    n = 150
    sm = rng.permutation(NB * bs)[:n].astype(np.int64)          # every token somewhere else
    want, cb, so = oracle_c.gather(host, sm, C_, "raw")
    geom = KVGeometry(L, H, D, NB, bs, C_, 2, 0, FMT_RAW)
    # (a) FlashAttention layout, token-granular mapping
    dev = to_dev(host)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    buf = torch.zeros(3 * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    tb = geom.token_bytes
    for c in range(3):
        nn = min(C_, n - c * C_)
        for plane in range(2 * L):
            o = c * cb + plane * C_ * tb
            assert np.array_equal(got[o:o + nn * tb], want[o:o + nn * tb])
    eng.close()
    # (b) FlashInfer layout (NB, 2, bs, H, D): block stride = 2 tiles
    fi = [t.permute(1, 0, 2, 3, 4).contiguous() for t in dev]
    g2 = KVGeometry(L, H, D, NB, bs, C_, 2, 2 * bs * H * D * 2, FMT_RAW)
    e2 = KVEngine(g2, None, 0, staging_bytes=0)
    e2.register_kv_caches(fi, layout="fi")
    buf.zero_()
    e2.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(buf.cpu().numpy()[: 2 * cb], got[: 2 * cb])
    e2.close()
    # (c) cross-layer blocks (NB, L, 2, bs, H, D): one contiguous tile group per block
    xl = torch.stack([t.permute(1, 0, 2, 3, 4) for t in dev], dim=1).contiguous()
    tile = bs * H * D * 2
    g3 = KVGeometry(L, H, D, NB, bs, C_, 2, 2 * L * tile, FMT_RAW)
    e3 = KVEngine(g3, None, 0, staging_bytes=0)
    base = xl.data_ptr()
    e3.register_kv_ptrs([base + (2 * l) * tile for l in range(L)], [base + (2 * l + 1) * tile for l in range(L)])
    buf.zero_()
    e3.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    assert np.array_equal(buf.cpu().numpy()[: 2 * cb], got[: 2 * cb])
    e3.close()


def test_bad_arguments_are_errors_not_crashes():
    need_gpu()
    geom = KVGeometry(2, 4, 64, 16, 16, 64)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    buf = torch.zeros(geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    with pytest.raises(b200kv.B200KVError):
        eng.gather(np.arange(16), buf.data_ptr())           # KV not registered
    dev = [torch.zeros((2, 16, 16, 4, 64), dtype=torch.bfloat16, device="cuda:0") for _ in range(2)]
    eng.register_kv_caches(dev)
    with pytest.raises(b200kv.B200KVError):
        eng.gather(np.array([16 * 16]), buf.data_ptr())     # slot out of range
    with pytest.raises(b200kv.B200KVError):
        eng.gather(np.array([-1]), buf.data_ptr())
    with pytest.raises(b200kv.B200KVError):
        eng.store(np.arange(16), None, np.arange(16))       # no pool attached
    # an op whose run table would not fit the 1 MiB table slot is refused, not truncated
    # (token-granular mapping: one 12-byte run per token)
    big = KVEngine(KVGeometry(2, 4, 64, 8192, 16, 64), None, 0, staging_bytes=0)
    bdev = [torch.zeros((2, 8192, 16, 4, 64), dtype=torch.bfloat16, device="cuda:0") for _ in range(2)]
    big.register_kv_caches(bdev)
    n_big = 100_000
    bbuf = torch.zeros(((n_big + 63) // 64) * big.geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    with pytest.raises(b200kv.B200KVError) as ei:
        big.gather((np.arange(n_big, dtype=np.int64) * 7) % (8192 * 16), bbuf.data_ptr())
    assert ei.value.code == b200kv._lib.EINVAL
    big.close()
    hnd = [t.permute(0, 1, 3, 2, 4).contiguous().permute(0, 1, 3, 2, 4) for t in dev]
    with pytest.raises(ValueError):
        eng.register_kv_caches(hnd)                          # HND tensors on an engine built for NHD
    with pytest.raises(NotImplementedError):
        eng.register_kv_caches([t.permute(0, 1, 4, 3, 2).contiguous().permute(0, 1, 4, 3, 2) for t in dev])
    eng.close()


def test_eviction_under_pressure_keeps_results_exact():
    """Pool of 3 chunks, 5 requests of 2 chunks: LRU evicts; whatever lookup reports as present
    must still round-trip bit-exactly."""
    need_gpu()
    p = SMALL
    rng = np.random.default_rng(31)
    host = mk_host_layers(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev(host)
    geom = KVGeometry(p["L"], p["H"], p["D"], p["NB"], p["bs"], p["C"])
    pool = KVPool(None, 3 * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=2 * geom.chunk_bytes)
    eng.register_kv_caches(dev)
    reqs = []
    for r in range(5):
        toks = rng.integers(0, 1000, 2 * p["C"]).astype(np.int32)
        sm = ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[:32], 16, 2 * p["C"])
        eng.wait(eng.store(toks, None, sm))
        reqs.append((toks, sm))
    st = pool.stats()
    assert st["n_used"] <= 3 and st["n_evicted_chunks"] >= 6
    scratch = to_dev([np.zeros_like(l) for l in host])
    e2 = KVEngine(geom, pool, 0, staging_bytes=2 * geom.chunk_bytes)
    e2.register_kv_caches(scratch)
    hit_any = False
    for toks, sm in reqs:
        hit = eng.lookup(toks)
        ret = e2.retrieve(toks, None, sm)
        torch.cuda.synchronize()
        assert ret.sum() == hit
        if hit:
            hit_any = True
            got = ko.gather_tokens([bits_of(t) for t in scratch], sm[:hit])
            assert np.array_equal(got, ko.gather_tokens(host, sm[:hit]))
    assert hit_any
    e2.close()
    eng.close()
    pool.close()


def test_peer_pull_same_device_and_cross_device():
    need_gpu()
    L, NB, bs, H, D = 3, 64, 16, 8, 128
    rng = np.random.default_rng(41)
    host = mk_host_layers(rng, L, NB, bs, H, D)
    geom = KVGeometry(L, H, D, NB, bs, 256)
    n = 300
    src = ko.slot_mapping_from_blocks(rng.permutation(NB)[:19], 16, n)
    dst = ko.slot_mapping_from_blocks(rng.permutation(NB)[:19], 16, n)
    devices = [0] + ([1] if torch.cuda.device_count() > 1 else [])
    for pd in devices:
        producer = to_dev(host, f"cuda:{pd}")
        local = [torch.zeros_like(t, device="cuda:0") for t in producer]
        eng = KVEngine(geom, None, 0, staging_bytes=0)
        eng.register_kv_caches(local)
        eng.import_peer_ptrs(1, pd, [t[0].data_ptr() for t in producer], [t[1].data_ptr() for t in producer])
        eng.wait(eng.peer_pull(1, src, dst))
        torch.cuda.synchronize()
        got = ko.gather_tokens([bits_of(t) for t in local], dst)
        assert np.array_equal(got, ko.gather_tokens(host, src))
        untouched = np.ones(NB * bs, bool)
        untouched[dst] = False
        assert not np.stack([bits_of(t) for t in local]).reshape(L, 2, NB * bs, H, D)[:, :, untouched].any()
        assert eng.stats()["p2p_bytes"] == n * 2 * L * H * D * 2
        eng.close()


@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_FP8])
def test_full_size_llama3_8b_round_trip_properties(fmt):
    """BASELINE.json config sizes (L=32, H=8, D=128, 8K-token prompt = 1 GiB): size-independent
    properties instead of the oracle — RAW: retrieve(store(x)) == x bit-for-bit; FP8: idempotence
    (re-quantising the dequantised pages reproduces codes and scales exactly) + tolerance."""
    need_gpu()
    L, NB, bs, H, D, C_ = 32, 1536, 16, 8, 128, 256
    g = torch.Generator(device="cuda:0").manual_seed(0)
    dev = [torch.randn((2, NB, bs, H, D), generator=g, device="cuda:0", dtype=torch.float32).bfloat16()
           for _ in range(L)]
    geom = KVGeometry(L, H, D, NB, bs, C_, 2, 0, fmt)
    n = 8192
    pool = KVPool(None, 32 * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=8 * geom.chunk_bytes)
    eng.register_kv_caches(dev)
    perm = torch.randperm(NB, generator=torch.Generator().manual_seed(1234)).numpy()
    sm = ko.slot_mapping_from_blocks(perm[: n // 16], 16, n)
    dm = ko.slot_mapping_from_blocks(perm[n // 16: 2 * (n // 16)], 16, n)
    toks = (np.arange(n) * 2654435761 % 128256).astype(np.int32)
    eng.wait(eng.store(toks, None, sm))
    assert eng.lookup(toks) == n
    ret = eng.retrieve(toks, None, dm)
    torch.cuda.synchronize()
    assert ret.all()
    sidx = torch.from_numpy(sm).cuda()
    didx = torch.from_numpy(dm).cuda()
    for t in dev:
        flat = t.view(2, NB * bs, H * D)
        a, b = flat[:, sidx], flat[:, didx]
        if fmt == FMT_RAW:
            assert torch.equal(a.view(torch.int16), b.view(torch.int16))
        else:
            af, bf = a.float(), b.float()
            amax = af.view(2, n // C_, C_, H, D).abs().amax(dim=(2, 4), keepdim=True)
            tol = torch.maximum(af.abs() * 2.0 ** -4, (amax * 2.0 ** -10).expand(2, n // C_, C_, H, D).reshape(af.shape)) \
                + af.abs() * 2.0 ** -8
            assert bool(((af - bf).abs() <= tol).all())
    if fmt == FMT_FP8:
        # idempotence: gather(dst pages) twice gives identical bytes, and quantising the
        # dequantised values reproduces the same codes (values already on the e4m3 grid * scale)
        b1 = torch.zeros((n // C_) * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
        b2 = torch.zeros_like(b1)
        eng.gather(dm, b1.data_ptr())
        for t in dev:
            flat = t.view(2, NB * bs, H * D)
            flat[:, sidx] = flat[:, didx]
        eng.gather(sm, b2.data_ptr())
        torch.cuda.synchronize()
        assert torch.equal(b1, b2)
    eng.close()
    pool.close()


@pytest.mark.parametrize("n_tok", [40, 256, 1000])
def test_fp8_store_token_granular_and_block_mappings(n_tok):
    """FP8 store with a token-granular mapping (40 single-token runs, walked by warp 0 in
    parallel) and block-structured ones: the oracle's codes and scales, bit for bit."""
    need_gpu()
    p = SMALL
    rng = np.random.default_rng(77 + n_tok)
    host = mk_host_layers(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev(host)
    geom = KVGeometry(p["L"], p["H"], p["D"], p["NB"], p["bs"], p["C"], 2, 0, FMT_FP8)
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(dev)
    sm = rng.permutation(p["NB"] * p["bs"])[:n_tok].astype(np.int64) if n_tok == 40 else \
        ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[: (n_tok + 15) // 16], 16, n_tok)
    n_chunks = (n_tok + p["C"] - 1) // p["C"]
    buf = torch.zeros(n_chunks * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    want, cb, so = oracle_c.gather(host, sm, p["C"], "fp8")
    got = buf.cpu().numpy()
    tb = geom.token_bytes // 2
    for c in range(n_chunks):
        n = min(p["C"], n_tok - c * p["C"])
        for plane in range(2 * p["L"]):
            o = c * cb + plane * p["C"] * tb
            assert np.array_equal(got[o:o + n * tb], want[o:o + n * tb]), (c, plane)
        s = c * cb + so
        assert np.array_equal(got[s:s + 2 * p["L"] * p["H"] * 4], want[s:s + 2 * p["L"] * p["H"] * 4])
    eng.close()


# ------------------------------------------------------------------------------------------------
# HND tiles: [H][block_tokens][D] inside a block — the layout vLLM's FlashInfer backend imposes.
# Logical content (what the model sees) must equal the oracle's, whatever the order.
# ------------------------------------------------------------------------------------------------
def to_dev_hnd(layers, dev="cuda:0"):
    """host logical (2, NB, bs, H, D) -> device tensors shaped like vLLM's FlashInfer cache:
    logical (NB, 2, bs, H, D) over physical (NB, 2, H, bs, D)."""
    out = []
    for l in layers:
        t = torch.from_numpy(l.view(np.int16)).view(torch.bfloat16).to(dev)
        phys = t.permute(1, 0, 3, 2, 4).contiguous()          # (NB, 2, H, bs, D)
        out.append(phys.permute(0, 1, 3, 2, 4))               # logical view, HND strides
    return out


def logical_bits(t):  # (NB, 2, bs, H, D) logical view -> numpy (2, NB, bs, H, D)
    return bits_of(t.permute(1, 0, 2, 3, 4).contiguous())


@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_FP8])
@pytest.mark.parametrize("n_tok", [1, 15, 16, 17, 40, 256, 300, 1000])
def test_hnd_store_retrieve_matches_oracle(n_tok, fmt):
    need_gpu()
    p = SMALL
    rng = np.random.default_rng(500 + n_tok)
    host = mk_host_layers(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev_hnd(host)
    assert tuple(dev[0].stride()[2:]) == (p["D"], p["bs"] * p["D"], 1)
    geom = KVGeometry(p["L"], p["H"], p["D"], p["NB"], p["bs"], p["C"], 2, 2 * p["bs"] * p["H"] * p["D"] * 2,
                      fmt, b200kv._lib.LAYOUT_HND)
    pool = KVPool(None, 8 * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=4 * geom.chunk_bytes)
    eng.register_kv_caches(dev)
    if n_tok == 40:      # token-granular: every token in another block, unaligned on both sides
        sm = rng.permutation(p["NB"] * p["bs"])[:n_tok].astype(np.int64)
        dm = rng.permutation(p["NB"] * p["bs"])[:n_tok].astype(np.int64)
    else:
        nb = (n_tok + 15) // 16
        sm = ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[:nb], 16, n_tok)
        dm = ko.slot_mapping_from_blocks(rng.permutation(p["NB"])[:nb], 16, n_tok)
    toks = rng.integers(0, 1000, n_tok).astype(np.int32)
    eng.wait(eng.store(toks, None, sm))
    assert eng.lookup(toks) == n_tok
    for t in dev:
        t.zero_()
    ret = eng.retrieve(toks, None, dm)
    torch.cuda.synchronize()
    assert ret.all()
    want = [np.zeros_like(l) for l in host]
    oe = ko.OracleEngine(p["C"], "fp8" if fmt == FMT_FP8 else "raw")
    oe.store(toks, np.ones(n_tok, bool), host, sm)
    oe.retrieve(toks, np.ones(n_tok, bool), want, dm)
    for a, b in zip(dev, want):
        assert np.array_equal(logical_bits(a), b)       # FP8: same codes and scales => same bf16 bits
    # device-resident halves too, and the chunk keeps whole tiles verbatim
    buf = torch.zeros(((n_tok + p["C"] - 1) // p["C"]) * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    src = to_dev_hnd(host)
    e2 = KVEngine(geom, None, 0, staging_bytes=0)
    e2.register_kv_caches(src)
    e2.gather(sm, buf.data_ptr())
    if n_tok >= 16 and n_tok != 40 and fmt == FMT_RAW:
        tile = p["bs"] * p["H"] * p["D"] * 2
        first_tile = buf[:tile].cpu().numpy().view(np.uint16).reshape(p["H"], p["bs"], p["D"])
        blk = int(sm[0]) // 16
        assert np.array_equal(first_tile, host[0][0, blk].transpose(1, 0, 2))     # layer 0, K, [H][bs][D]
    for t in src:
        t.zero_()
    e2.scatter(dm, buf.data_ptr())
    torch.cuda.synchronize()
    for a, b in zip(src, want):
        assert np.array_equal(logical_bits(a), b)
    e2.close()
    eng.close()
    pool.close()


def test_hnd_peer_pull_and_format_isolation():
    need_gpu()
    L, NB, bs, H, D = 2, 64, 16, 8, 128
    rng = np.random.default_rng(91)
    host = mk_host_layers(rng, L, NB, bs, H, D)
    geom = KVGeometry(L, H, D, NB, bs, 256, 2, 2 * bs * H * D * 2, FMT_RAW, b200kv._lib.LAYOUT_HND)
    producer = to_dev_hnd(host)
    local = to_dev_hnd([np.zeros_like(l) for l in host])
    eng = KVEngine(geom, None, 0, staging_bytes=0)
    eng.register_kv_caches(local)
    eng.import_peer_ptrs(2, 0, [t[:, 0].data_ptr() for t in producer], [t[:, 1].data_ptr() for t in producer])
    n = 200
    src = np.concatenate([ko.slot_mapping_from_blocks(rng.permutation(NB)[:10], 16, 160),
                          rng.permutation(NB * bs)[:40].astype(np.int64)])          # whole tiles + ragged
    dst = np.concatenate([ko.slot_mapping_from_blocks(rng.permutation(NB)[:10], 16, 160),
                          (np.arange(40) + 11 * 16 * 3 + 5).astype(np.int64)])
    dst_blocks_used = set(int(x) // 16 for x in dst[:160])
    dst[160:] = [s for s in range(NB * bs) if s // 16 not in dst_blocks_used][5:45]
    eng.wait(eng.peer_pull(2, src, dst))
    torch.cuda.synchronize()
    got = ko.gather_tokens([logical_bits(t) for t in local], dst)
    assert np.array_equal(got, ko.gather_tokens(host, src))
    eng.close()
    # a pool shared by an NHD and an HND engine never serves one's chunks to the other
    g_n = KVGeometry(L, H, D, NB, bs, 256)
    g_h = KVGeometry(L, H, D, NB, bs, 256, 2, 2 * bs * H * D * 2, FMT_RAW, b200kv._lib.LAYOUT_HND)
    pool = KVPool(None, 4 * g_n.chunk_bytes, g_n.chunk_bytes, 1)
    e_n = KVEngine(g_n, pool, 0, staging_bytes=2 * g_n.chunk_bytes, key_seed=1)
    e_h = KVEngine(g_h, pool, 0, staging_bytes=2 * g_h.chunk_bytes, key_seed=1)
    e_n.register_kv_caches(to_dev(host))
    e_h.register_kv_caches(local)
    toks = np.arange(256, dtype=np.int32)
    sm = ko.slot_mapping_from_blocks(np.arange(16), 16, 256)
    e_n.wait(e_n.store(toks, None, sm))
    assert e_h.retrieve(toks, None, sm).sum() == 0 and e_n.retrieve(toks, None, sm).all()
    e_n.close()
    e_h.close()
    pool.close()


@pytest.mark.parametrize("layout", ["nhd", "hnd"])
@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_FP8])
@pytest.mark.parametrize("group", [1, 2, 5])
def test_layerwise_retrieve_matches_oracle(group, fmt, layout):
    """lmcache_engine.retrieve_layer semantics (adapter :870-880, :907-929): same pages as the
    chunk-wise retrieve; a stream that waited for layer l sees layers <= l complete."""
    need_gpu()
    L, NB, bs, H, D, C_ = 5, 96, 16, 8, 128, 256
    rng = np.random.default_rng(900 + group)
    host = mk_host_layers(rng, L, NB, bs, H, D)
    hnd = layout == "hnd"
    dev = to_dev_hnd(host) if hnd else to_dev(host)
    geom = KVGeometry(L, H, D, NB, bs, C_, 2, 2 * bs * H * D * 2 if hnd else 0, fmt,
                      b200kv._lib.LAYOUT_HND if hnd else b200kv._lib.LAYOUT_NHD)
    pool = KVPool(None, 8 * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=8 * geom.chunk_bytes)
    eng.register_kv_caches(dev)
    n = 2 * C_ + 70
    toks = rng.integers(0, 1000, n).astype(np.int32)
    sm = ko.slot_mapping_from_blocks(rng.permutation(NB)[: (n + 15) // 16], 16, n)
    dm = ko.slot_mapping_from_blocks(rng.permutation(NB)[: (n + 15) // 16], 16, n)
    eng.wait(eng.store(toks, None, sm))
    for t in dev:
        t.zero_()
    side = torch.cuda.Stream()
    ret, ticket = eng.retrieve(toks, None, dm, stream=torch.cuda.current_stream(), return_ticket=True,
                               layers_per_group=group)
    assert ret.all() and ticket
    want = [np.zeros_like(l) for l in host]
    oe = ko.OracleEngine(C_, "fp8" if fmt == FMT_FP8 else "raw")
    oe.store(toks, np.ones(n, bool), host, sm)
    oe.retrieve(toks, np.ones(n, bool), want, dm)
    get = (lambda t: logical_bits(t)) if hnd else bits_of
    for l in range(L):
        eng.wait_layer(ticket, l, side)          # what wait_for_layer_load does on the compute stream
        side.synchronize()
        assert np.array_equal(get(dev[l]), want[l]), f"layer {l} not complete after its wait"
    eng.wait(ticket)
    eng.wait_layer(ticket, 0, side)              # finished tickets: no-op
    assert eng.stats()["n_loaded_tokens"] == n
    eng.close()
    pool.close()


# ------------------------------------------------------------------------------------------------
# The default FP8 store is the persistent warp-specialised kernel (kv_fp8_store3_kernel; TMA tensor maps on
# NHD pages, bulk copies on HND pages); ops it does not take (token-granular mappings) run the cluster
# kernel.  Both must produce the same chunk, byte for byte, and the tests above hold whichever runs
# against the oracle.  Geometries: the test one (H=8, D=128), D=64, and Llama-3-8B's 32 layers.
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hnd", [False, True])
@pytest.mark.parametrize("shape", [(3, 8, 128, 96), (2, 4, 64, 96), (32, 8, 128, 160)], ids=["L3H8D128", "L2H4D64", "L32H8D128"])
@pytest.mark.parametrize("n_tok", [1, 16, 17, 255, 256, 257, 700, 1024, 2048])
def test_fp8_persistent_store_equals_cluster_kernel_and_oracle(monkeypatch, hnd, shape, n_tok):
    need_gpu()
    L, H, D, NB = shape
    bs, C_ = 16, 256
    if n_tok > NB * bs or (L == 32 and n_tok not in (257, 2048)):
        pytest.skip("more tokens than pages / full-depth model checked at two sizes only")
    rng = np.random.default_rng(9100 + n_tok + L)
    host = mk_host_layers(rng, L, NB, bs, H, D)
    dev = to_dev_hnd(host) if hnd else to_dev(host)
    geom = KVGeometry(L, H, D, NB, bs, C_, 2, 2 * bs * H * D * 2 if hnd else 0, FMT_FP8,
                      b200kv._lib.LAYOUT_HND if hnd else b200kv._lib.LAYOUT_NHD)
    sm = ko.slot_mapping_from_blocks(rng.permutation(NB)[: (n_tok + bs - 1) // bs], bs, n_tok)
    n_chunks = (n_tok + C_ - 1) // C_
    out, launches = [], []
    for ver in ("3", "1"):
        monkeypatch.setenv("B200KV_FP8_STORE", ver)
        eng = KVEngine(geom, None, 0, staging_bytes=0)
        eng.register_kv_caches(dev)
        buf = torch.zeros(n_chunks * geom.chunk_bytes, dtype=torch.uint8, device="cuda:0")
        eng.gather(sm, buf.data_ptr())
        torch.cuda.synchronize()
        out.append(buf.cpu().numpy())
        eng.close()
    if not np.array_equal(out[0], out[1]):
        bad = np.flatnonzero(out[0] != out[1])
        pytest.fail(f"{len(bad)} bytes differ, first at {bad[:8]} (chunk bytes {geom.chunk_bytes}, scales at {geom.chunk_bytes - 2 * L * H * 4})")
    if not hnd and L <= 3:      # and directly against the C oracle (NHD chunk layout)
        want, cb, so = oracle_c.gather(host, sm, C_, "fp8")
        got = out[0]
        for c in range(n_chunks):
            n = min(C_, n_tok - c * C_)
            for plane in range(2 * L):
                o = c * cb + plane * C_ * H * D
                assert np.array_equal(got[o:o + n * H * D], want[o:o + n * H * D]), (c, plane)
            assert np.array_equal(got[c * cb + so:c * cb + so + 2 * L * H * 4], want[c * cb + so:c * cb + so + 2 * L * H * 4])


def test_refused_op_leaves_no_reserved_slots_and_no_pins():
    """An op whose run table does not fit (token-granular mapping over hundreds of chunks) is refused with
    -EINVAL *after* pool slots were reserved / chunks pinned: nothing may stay reserved (later stores of the
    same keys would see -EEXIST until the stale-writer reclaim) or pinned (could never be evicted)."""
    need_gpu()
    L, NB, bs, H, D, C_ = 1, 8192, 16, 1, 64, 256
    geom = KVGeometry(L, H, D, NB, bs, C_, 2, 0, FMT_RAW)
    dev = [torch.randn((2, NB, bs, H, D), device="cuda:0").bfloat16() for _ in range(L)]
    n_chunks = 420
    pool = KVPool(None, (n_chunks + 8) * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=2 * 512 * geom.chunk_bytes)    # one batch holds the whole op
    eng.register_kv_caches(dev)
    n = n_chunks * C_
    rng = np.random.default_rng(11)
    toks = rng.integers(0, 50000, n).astype(np.int32)
    scattered = (np.arange(n, dtype=np.int64) * 2) % (NB * bs) + (np.arange(n) * 2 // (NB * bs))   # no two neighbours adjacent
    assert len(np.unique(scattered)) == n
    with pytest.raises(b200kv.B200KVError) as ei:
        eng.store(toks, None, scattered)                    # > 87 381 runs: the table refuses it
    assert ei.value.code == b200kv._lib.EINVAL
    st = pool.stats()
    assert st["n_used"] == 0 and pool.check(), st             # every reservation was aborted
    # the same keys can be stored right away (block-structured mapping now), and loaded
    sm = ko.slot_mapping_from_blocks(rng.permutation(NB)[: n // bs], bs, n)
    eng.wait(eng.store(toks, None, sm))
    assert pool.stats()["n_stored_chunks"] == n_chunks and eng.lookup(toks) == n
    with pytest.raises(b200kv.B200KVError):
        eng.retrieve(toks, None, scattered)                 # refused after pinning 420 chunks ...
    assert pool.clear()                                      # ... none of which stayed pinned (clear() fails with pins)
    eng.close()
    pool.close()


# ------------------------------------------------------------------------------------------------
# One engine op for the requests of a step (b200kv_store_batch_async / b200kv_load_batch_async): same bytes in
# the pool and in the pages as one op per request, for every format and tile order; partial chunks sit in the
# MIDDLE of a batch (every request's ragged tail), each request stops at its own first miss.
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hnd", [False, True])
@pytest.mark.parametrize("fmt", [FMT_RAW, FMT_FP8, b200kv.FMT_Q4])
@pytest.mark.parametrize("layerwise", [0, 2])
def test_batch_ops_equal_per_request_ops_and_oracle(fmt, hnd, layerwise):
    need_gpu()
    p = SMALL
    rng = np.random.default_rng(77 + fmt)
    host = mk_host_layers(rng, p["L"], p["NB"], p["bs"], p["H"], p["D"])
    dev = to_dev_hnd(host) if hnd else to_dev(host)
    stride = 2 * p["bs"] * p["H"] * p["D"] * 2 if hnd else 0
    geom = KVGeometry(p["L"], p["H"], p["D"], p["NB"], p["bs"], p["C"], 2, stride, fmt,
                      b200kv._lib.LAYOUT_HND if hnd else b200kv._lib.LAYOUT_NHD)
    pool = KVPool(None, 16 * geom.chunk_bytes, geom.chunk_bytes, 1)
    eng = KVEngine(geom, pool, 0, staging_bytes=8 * geom.chunk_bytes)
    eng.register_kv_caches(dev)
    name = {FMT_RAW: "raw", FMT_FP8: "fp8", b200kv.FMT_Q4: "q4"}[fmt]
    oe = ko.OracleEngine(p["C"], name)
    C_, bs = p["C"], p["bs"]
    lens = [C_ + 37, 5, 2 * C_, 2 * C_ - 1]                 # ragged tails in the middle of the batch (84 of 96 pages)
    perm = rng.permutation(p["NB"])
    toks, sms, o = [], [], 0
    for n in lens:
        nb = (n + bs - 1) // bs
        toks.append(rng.integers(0, 128256, n).astype(np.int32))
        sms.append(ko.slot_mapping_from_blocks(perm[o:o + nb], bs, n))
        o += nb
    # request 3 is stored from its second chunk on (offset = C): its first chunk stays a miss
    offs = [0, 0, 0, C_]
    t = eng.store_batch(list(zip(toks, sms, offs)))
    assert t != 0
    eng.wait(t)
    assert eng.stats()["n_store_ops"] == 1
    for tk, sm, off in zip(toks, sms, offs):
        m = np.ones(len(tk), bool)
        m[:off] = False
        oe.store(tk, m, host, sm, off)
    assert [eng.lookup(tk) for tk in toks] == [oe.lookup(tk) for tk in toks] == [lens[0], lens[1], lens[2], 0]
    # load: other pages; request 2 with its first chunk masked; request 3 misses at once (chunk 0 absent)
    dperm = rng.permutation(p["NB"])
    dms, o = [], 0
    for n in lens:
        nb = (n + bs - 1) // bs
        dms.append(ko.slot_mapping_from_blocks(dperm[o:o + nb], bs, n))
        o += nb
    for tns in dev:
        tns.zero_()
    skips = [0, 0, C_, 0]
    got, ticket = eng.retrieve_batch(list(zip(toks, dms, skips)), layers_per_group=layerwise)
    if layerwise:
        for l in range(0, p["L"], layerwise):
            eng.wait_layer(ticket, l)
    torch.cuda.synchronize()
    assert list(got) == [lens[0], lens[1], lens[2] - C_, 0]
    assert eng.stats()["n_load_ops"] == 1
    dst = [np.zeros_like(l) for l in host]
    for tk, dm, sk in zip(toks, dms, skips):
        m = np.ones(len(tk), bool)
        m[:sk] = False
        oe.retrieve(tk, m, dst, dm)
    for a, b in zip(dev, dst):
        assert np.array_equal(logical_bits(a) if hnd else bits_of(a), b)
    eng.close()
    pool.close()
