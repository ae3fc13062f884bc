"""fp8 KV caches (--kv-cache-dtype fp8 / fp8_e4m3 / fp8_e5m2) without a GPU: the Q4 specification in
tests/fp8_cache_oracle.py against exact rational arithmetic for every code, its error bound, the vLLM config
mapping, key seeds and format tags, and the P/D pairing rule."""
from __future__ import annotations

import json
from fractions import Fraction
from types import SimpleNamespace as NS

import numpy as np
import pytest

from b200kv import _lib
from oracle import kv_oracle as ko
from tests import fp8_cache_oracle as fo

LLAMA = "meta-llama/Meta-Llama-3-8B"


# ---------------------------------------------------------------------------------------------------------------
# exact reference: rationals only, nothing shared with the oracle but the code -> value tables
# ---------------------------------------------------------------------------------------------------------------
def _round_sig(v: Fraction, bits: int) -> Fraction:
    """v rounded to `bits` significant bits, ties to even (v > 0, no exponent limit: bf16 and fp32 cover every
    value here)."""
    e = 0
    while v >= 2 ** (e + 1):
        e += 1
    while v < 2 ** e:
        e -= 1
    q = v / Fraction(2) ** (e - bits + 1)
    n = int(q)
    r = q - n
    if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2):
        n += 1
    return n * Fraction(2) ** (e - bits + 1)


def _rint_even(v: Fraction) -> int:
    n = int(np.floor(float(v))) if v.denominator != 1 else int(v)
    while Fraction(n) > v:
        n -= 1
    while Fraction(n + 1) <= v:
        n += 1
    r = v - n
    return n + 1 if r > Fraction(1, 2) or (r == Fraction(1, 2) and n % 2) else n


def _nearest_code(v: Fraction, ft: str) -> int:
    """The code of `ft` nearest to v (ties to the even code), saturated to the largest finite magnitude."""
    grid = [Fraction(float(x)) for x in fo.decode_table(ft)[:fo.MAX_FINITE_CODE[ft] + 1]]
    a = min(abs(v), grid[-1])
    best = min(range(len(grid)), key=lambda c: (abs(grid[c] - a), c % 2))
    return best | (0x80 if v < 0 else 0)


def _exact_roundtrip(group: list[int], ft: str) -> list[int]:
    """Q4 store -> load of one group of finite codes in rational arithmetic."""
    dec = fo.decode_table(ft)
    xs = [Fraction(float(dec[c])) for c in group]
    amax = max(abs(x) for x in xs)
    if amax == 0:
        return [0] * len(group)
    s = _round_sig(_round_sig(amax / 7, 24), 8)          # fl32(amax / 7), then bf16_rn
    inv = _round_sig(1 / s, 24)                           # fl32(1 / s)
    out = []
    for x in xs:
        q = _rint_even(x * inv)
        assert abs(q) <= 7
        y = q * s
        out.append(0 if y == 0 else _nearest_code(y, ft))   # q = 0 gives +0
    return out


def _roundtrip(codes: np.ndarray, ft: str) -> np.ndarray:
    q, s = fo.q4_pack_chunk(codes, ft)
    return fo.q4_unpack_chunk(q, s, ft)


@pytest.mark.parametrize("ft", fo.FP8_TYPES)
def test_every_code_as_group_maximum_matches_exact_arithmetic(ft):
    """Each of the 256 codes is the maximum of a group whose other 31 codes are every smaller magnitude it can
    hold (both signs); finite groups are compared with rational arithmetic, the others with the stated rules."""
    rng = np.random.default_rng(7)
    dec = fo.decode_table(ft)
    groups = np.zeros((256, 32), np.uint8)
    for c in range(256):
        m = c & 0x7F
        finite_below = [k for k in range(m + 1) if np.isfinite(dec[k])]
        others = rng.choice(finite_below, 31) | (rng.integers(0, 2, 31) << 7)
        groups[c] = np.concatenate([[c], others]).astype(np.uint8)
    got = _roundtrip(groups.reshape(1, 1, 256, 1, 32), ft).reshape(256, 32)
    for c in range(256):
        m = c & 0x7F
        if np.isnan(dec[m]):                                   # NaN poisons the group: every element NaN
            assert np.all(got[c] == fo.NAN_CODE), (ft, hex(c))
        elif np.isinf(dec[m]):                                 # e5m2 inf: s = inf, 0 * inf = NaN, -1 * inf saturates
            assert got[c][0] == 0xFB and np.all(got[c][1:] == fo.NAN_CODE), (ft, hex(c))
        else:
            assert got[c].tolist() == _exact_roundtrip(groups[c].tolist(), ft), (ft, hex(c))


@pytest.mark.parametrize("ft", fo.FP8_TYPES)
def test_every_code_alone_in_its_group(ft):
    """A group of one code and 31 zeros: the code's own round trip, for all 256 codes."""
    groups = np.zeros((256, 32), np.uint8)
    groups[:, 5] = np.arange(256)
    got = _roundtrip(groups.reshape(1, 1, 256, 1, 32), ft).reshape(256, 32)
    for c in range(256):
        want = _exact_roundtrip(groups[c].tolist(), ft) if np.isfinite(fo.decode_table(ft)[c]) else None
        if want is not None:
            assert got[c].tolist() == want, (ft, hex(c))
    # a finite maximum is reproduced exactly: q = +-7 and 7 * s rounds back to it
    finite = [c for c in range(256) if np.isfinite(fo.decode_table(ft)[c]) and c & 0x7F]
    assert all(got[c, 5] == c for c in finite), ft


@pytest.mark.parametrize("ft", fo.FP8_TYPES)
def test_round_trip_is_within_half_a_step_plus_one_fp8_rounding(ft):
    rng = np.random.default_rng(11)
    dec = fo.decode_table(ft)
    finite = np.array([c for c in range(256) if np.isfinite(dec[c])], np.uint8)
    codes = rng.choice(finite, size=(2, 2, 64, 4, 128)).astype(np.uint8)
    # narrow-range groups as well: maxima in every binade, subnormals included
    codes[0, 0, :32] = (codes[0, 0, :32] & 0x87) | (rng.integers(0, 16, (32, 4, 128)) << 3).astype(np.uint8) & 0x78
    codes = np.where(np.isfinite(dec[codes]), codes, 0).astype(np.uint8)
    x = dec[codes]
    xh = dec[_roundtrip(codes, ft)]
    assert np.all(np.abs(x - xh) <= fo.q4_fp8_tolerance(x, ft))


def test_q4_record_of_an_fp8_cache_is_the_16bit_record():
    """The record layout does not depend on the cache type: what a bf16 cache holding the same values stores."""
    rng = np.random.default_rng(3)
    codes = rng.integers(0, 0x78, size=(1, 2, 16, 8, 64)).astype(np.uint8) | (rng.integers(0, 2, (1, 2, 16, 8, 64)) << 7).astype(np.uint8)
    x = fo.codes_to_f64(codes, "e4m3").astype(np.float32)      # every e4m3 value is a bf16 value
    bits = ko.f32_to_bf16_bits_rn(x)
    assert np.array_equal(ko.bf16_bits_to_f32(bits), x)
    q8, s8 = fo.q4_pack_chunk(codes, "e4m3")
    q16, s16 = ko.q4_pack_chunk(bits)
    assert np.array_equal(q8, q16) and np.array_equal(s8, s16)


def test_encode_matches_torch_for_every_finite_fp32_neighbour():
    """encode_rn_satfinite agrees with torch's round-to-nearest-even cast wherever the cast does not overflow."""
    import torch
    for ft in fo.FP8_TYPES:
        grid = fo.decode_table(ft)[:fo.MAX_FINITE_CODE[ft] + 1]
        mids = (grid[1:] + grid[:-1]) / 2
        v = np.concatenate([grid, mids, np.nextafter(mids, 0), np.nextafter(mids, np.inf)])
        v = np.concatenate([v, -v]).astype(np.float32)
        want = torch.from_numpy(v).to(fo._TORCH[ft]).view(torch.uint8).numpy()
        assert np.array_equal(fo.encode_rn_satfinite(v, ft), want), ft
        assert fo.encode_rn_satfinite(np.array([1e30, -np.inf, np.nan]), ft).tolist() == \
            [fo.MAX_FINITE_CODE[ft], 0x80 | fo.MAX_FINITE_CODE[ft], fo.NAN_CODE]


# ---------------------------------------------------------------------------------------------------------------
# vLLM config -> geometry
# ---------------------------------------------------------------------------------------------------------------
def _vllm_config(cache_dtype, mla=False):
    import torch
    mc = NS(model="synth-llama-3", dtype=torch.bfloat16, use_mla=mla, get_num_layers=lambda pc: 32,
            get_num_kv_heads=lambda pc: 1 if mla else 8, get_head_size=lambda: 576 if mla else 128)
    return NS(model_config=mc, parallel_config=NS(tensor_parallel_size=1, rank=0),
              cache_config=NS(block_size=16, cache_dtype=cache_dtype))


@pytest.mark.parametrize("cache,fmt,elem,dtype,want_fmt", [
    ("fp8", _lib.FMT_RAW, 1, _lib.DTYPE_E4M3, _lib.FMT_RAW),
    ("fp8", _lib.FMT_FP8, 1, _lib.DTYPE_E4M3, _lib.FMT_RAW),         # the pages already are fp8
    ("fp8", _lib.FMT_Q4, 1, _lib.DTYPE_E4M3, _lib.FMT_Q4),
    ("fp8_e4m3", _lib.FMT_FP8, 1, _lib.DTYPE_E4M3, _lib.FMT_RAW),
    ("fp8_e4m3", _lib.FMT_Q4, 1, _lib.DTYPE_E4M3, _lib.FMT_Q4),
    ("fp8_e5m2", _lib.FMT_RAW, 1, _lib.DTYPE_E5M2, _lib.FMT_RAW),
    ("fp8_e5m2", _lib.FMT_FP8, 1, _lib.DTYPE_E5M2, _lib.FMT_RAW),
    ("fp8_e5m2", _lib.FMT_Q4, 1, _lib.DTYPE_E5M2, _lib.FMT_Q4),
    ("fp8_per_token_head", _lib.FMT_RAW, 1, _lib.DTYPE_BF16, _lib.FMT_RAW),
    ("fp8_inc", _lib.FMT_RAW, 1, _lib.DTYPE_BF16, _lib.FMT_RAW),
    ("bfloat16", _lib.FMT_Q4, 2, _lib.DTYPE_BF16, _lib.FMT_Q4),
    ("float16", _lib.FMT_FP8, 2, _lib.DTYPE_FP16, _lib.FMT_FP8),
])
def test_geometry_from_vllm_fp8_cache(cache, fmt, elem, dtype, want_fmt):
    pytest.importorskip("vllm")
    from b200kv.config import B200KVConfig
    from b200kv.connector import geometry_from_vllm
    cfg = B200KVConfig()
    cfg.fmt = fmt
    g = geometry_from_vllm(_vllm_config(cache), cfg)
    assert (g.elem_bytes, g.cache_dtype, g.fmt) == (elem, dtype, want_fmt)
    if elem == 1:   # dtype keeps naming the 16-bit type; the fp8 type is fp8_dtype
        assert (g.dtype, g.fp8_dtype) == (_lib.DTYPE_BF16, dtype)
    if want_fmt == _lib.FMT_Q4 and elem == 1:
        # Llama-3-8B: a 576-byte record per token and plane, against 1024 bytes RAW
        assert g.chunk_bytes == 32 * 2 * 256 * 576
        raw = geometry_from_vllm(_vllm_config(cache), B200KVConfig())
        assert raw.chunk_bytes == 32 * 2 * 256 * 1024 and g.chunk_bytes / raw.chunk_bytes == 0.5625


@pytest.mark.parametrize("cache", ["fp8_per_token_head", "fp8_inc"])
def test_q4_on_other_1_byte_caches_is_refused_at_start_up(cache):
    pytest.importorskip("vllm")
    from b200kv.config import B200KVConfig
    from b200kv.connector import geometry_from_vllm
    cfg = B200KVConfig()
    cfg.fmt = _lib.FMT_Q4
    with pytest.raises(ValueError, match=f"q4.*{cache}"):
        geometry_from_vllm(_vllm_config(cache), cfg)


def test_mla_fp8_latent_cache():
    """MLA with an fp8 latent cache (576 uint8): RAW as before, FP8 stored RAW, Q4 refused by the engine."""
    pytest.importorskip("vllm")
    from b200kv.config import B200KVConfig
    from b200kv.connector import geometry_from_vllm
    cfg = B200KVConfig()
    cfg.fmt = _lib.FMT_FP8
    g = geometry_from_vllm(_vllm_config("fp8", mla=True), cfg)
    assert (g.elem_bytes, g.fmt, g.head_dim, g.mla) == (1, _lib.FMT_RAW, 576, True)
    assert g.chunk_bytes == 32 * 256 * 576
    cfg.fmt = _lib.FMT_Q4
    with pytest.raises(_lib.B200KVError):
        geometry_from_vllm(_vllm_config("fp8", mla=True), cfg).chunk_bytes


def test_engine_geometry_rules_for_1_byte_caches():
    from b200kv import KVGeometry
    g = lambda **kw: KVGeometry(**{**dict(n_layers=2, n_kv_heads=8, head_dim=128, n_blocks=4, elem_bytes=1), **kw})
    assert g(fmt=_lib.FMT_Q4).chunk_bytes == 2 * 2 * 256 * 576
    with pytest.raises(_lib.B200KVError):
        g(fmt=_lib.FMT_FP8).chunk_bytes                         # FP8 of fp8 pages stays refused by the engine
    with pytest.raises(_lib.B200KVError):
        g(fmt=_lib.FMT_Q4, head_dim=48).chunk_bytes              # D % 32
    with pytest.raises(_lib.B200KVError):
        g(fmt=_lib.FMT_Q4, n_kv_heads=1, head_dim=32).chunk_bytes   # H * D % 64: 18-byte records
    assert g(fmt=_lib.FMT_Q4, n_kv_heads=1, head_dim=64).chunk_bytes == 2 * 2 * 256 * 36


def test_dtype_code():
    import torch
    from b200kv.engine import dtype_code
    assert dtype_code(torch.bfloat16) == _lib.DTYPE_BF16 and dtype_code(torch.float16) == _lib.DTYPE_FP16
    assert dtype_code(torch.float8_e4m3fn) == _lib.DTYPE_E4M3 and dtype_code(torch.float8_e5m2) == _lib.DTYPE_E5M2
    assert dtype_code(torch.uint8) is None                      # vLLM's fp8 caches: the config names the type
    assert dtype_code(torch.uint8, "fp8") == dtype_code(torch.uint8, "fp8_e4m3") == _lib.DTYPE_E4M3
    assert dtype_code(torch.uint8, "fp8_e5m2") == _lib.DTYPE_E5M2
    assert dtype_code(torch.uint8, "fp8_inc") is None and dtype_code(torch.float32) is None


# ---------------------------------------------------------------------------------------------------------------
# key seeds and format tags: literal values; everything but e5m2 is what it was before the fp8 types existed
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("elem,fmt,dtype,seed,tag", [
    (2, _lib.FMT_RAW, _lib.DTYPE_BF16, 0xa546d4bc64f13a93, 0x0),
    (2, _lib.FMT_Q4, _lib.DTYPE_BF16, 0xb7fd2487deea335d, 0x2),
    (2, _lib.FMT_Q4, _lib.DTYPE_FP16, 0x39ba3fed61f3365f, 0x10002),
    (1, _lib.FMT_RAW, _lib.DTYPE_E4M3, 0x3199885ea8d7b62c, 0x0),
    (1, _lib.FMT_Q4, _lib.DTYPE_E4M3, 0x099c865463b83989, 0x2),
])
def test_seeds_and_tags_are_unchanged(elem, fmt, dtype, seed, tag):
    from b200kv import KVGeometry
    g = KVGeometry(32, 8, 128, 1024, elem_bytes=elem, fmt=fmt, dtype=dtype)
    assert g.key_seed(LLAMA, 1, 0) == seed and g.fmt_tag == tag


def test_e5m2_seeds_and_tags_are_their_own():
    from b200kv import KVGeometry, xxh64
    from b200kv.engine import DEFAULT_SEED
    for fmt in (_lib.FMT_RAW, _lib.FMT_Q4):
        for layout in (_lib.LAYOUT_NHD, _lib.LAYOUT_HND):
            e4 = KVGeometry(32, 8, 128, 1024, elem_bytes=1, fmt=fmt, layout=layout)
            e5 = KVGeometry(32, 8, 128, 1024, elem_bytes=1, fmt=fmt, layout=layout, fp8_dtype=_lib.DTYPE_E5M2)
            base = f"{LLAMA}|1|0|32|8|128|1|256|{fmt}|{layout}"
            assert e4.key_seed(LLAMA) == xxh64(base.encode(), DEFAULT_SEED)
            assert e5.key_seed(LLAMA) == xxh64((base + "|e5m2").encode(), DEFAULT_SEED) != e4.key_seed(LLAMA)
            assert e4.fmt_tag == fmt | (layout << 8)
            assert e5.fmt_tag == fmt | (layout << 8) | (_lib.DTYPE_E5M2 << 16)
    assert KVGeometry(32, 8, 128, 1024, fmt=_lib.FMT_Q4, fp8_dtype=_lib.DTYPE_E5M2, elem_bytes=1).key_seed(LLAMA) == \
        0xa6a7ed1dec26a60f


# ---------------------------------------------------------------------------------------------------------------
# P/D: e4m3 and e5m2 peers refuse to pair
# ---------------------------------------------------------------------------------------------------------------
class _PdEngine:
    def __init__(self, dtype=None):
        g = dict(n_blocks=64, stride=2048, n_layers=2, n_kv_heads=2, head_dim=64, block_tokens=16, elem_bytes=1,
                 layout=0)
        if dtype is not None:
            g["dtype"] = dtype
        self.geom = NS(**g)

    def export_ipc(self):
        return b"\x07" * (72 * 4)

    def import_peer(self, pid, device, descs, stride, n_blocks):
        self.imported = (pid, device, len(descs), stride, n_blocks)


def test_pd_refuses_e4m3_with_e5m2(tmp_path, monkeypatch):
    from b200kv import pd
    monkeypatch.setattr(pd, "SHM_DIR", str(tmp_path))
    path = pd.publish_ipc("P-e5m2", _PdEngine(_lib.DTYPE_E5M2), device=0)
    assert json.load(open(path))["dtype"] == 2
    with pytest.raises(ValueError, match="dtype"):
        pd.PeerResolver(_PdEngine(_lib.DTYPE_E4M3)).resolve("P-e5m2")
    assert pd.PeerResolver(_PdEngine(_lib.DTYPE_E5M2)).resolve("P-e5m2") == 0
    pd.publish_ipc("P-e4m3", _PdEngine(_lib.DTYPE_E4M3), device=0)
    with pytest.raises(ValueError, match="dtype"):
        pd.PeerResolver(_PdEngine(_lib.DTYPE_E5M2)).resolve("P-e4m3")


def test_pd_document_without_dtype_is_e4m3_on_1_byte_caches(tmp_path, monkeypatch):
    from b200kv import pd
    monkeypatch.setattr(pd, "SHM_DIR", str(tmp_path))
    path = pd.publish_ipc("P-old", _PdEngine(_lib.DTYPE_E4M3), device=0)
    doc = json.load(open(path))
    assert doc.pop("dtype") == _lib.DTYPE_E4M3
    with open(path, "w") as f:
        json.dump(doc, f)
    assert pd.PeerResolver(_PdEngine(_lib.DTYPE_E4M3)).resolve("P-old") == 0
    with pytest.raises(ValueError, match="dtype"):
        pd.PeerResolver(_PdEngine(_lib.DTYPE_E5M2)).resolve("P-old")
