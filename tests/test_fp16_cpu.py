"""fp16 KV caches in the FP8 and Q4 chunk formats, CPU side: the fp16 rules of the oracle (tolerances, finiteness,
idempotence, an exhaustive check of every finite fp16 group maximum, the bf16 default unchanged), the cache type
vLLM's config implies, the key namespace and format tags, and the P/D dtype check."""
import json
import os
from types import SimpleNamespace as NS

import numpy as np
import pytest

from oracle import kv_oracle as ko
from tests import fp16_oracle as fo
from tests import mla_oracle as mo

from b200kv import _lib  # noqa: E402

FP16_MAX_BITS = 0x7BFF     # 65504


def fp16_bits(x):
    return fo.f32_to_fp16_bits_rn(np.asarray(x, np.float32))


def random_fp16_chunk(rng, L=2, n=64, H=4, D=64):
    x = rng.standard_normal((L, 2, n, H, D)).astype(np.float32)
    x *= np.exp(rng.uniform(-6, 6, (L, 2, 1, H, 1))).astype(np.float32)
    return fp16_bits(x)


def adversarial_fp16_chunk(rng, H=8, n=32, D=64):
    """(1, 2, n, H, D) fp16 bits, one kind of group per head: ±65504, subnormals only, all zero, one outlier per
    32-element group over small values, one outlier per head, and the smallest normals."""
    x = np.zeros((1, 2, n, H, D), np.float32)
    x[..., 0, :] = rng.choice([-65504.0, 65504.0, 1.0, -0.5, 3e-5], (1, 2, n, D))
    sub = rng.integers(1, 0x400, (1, 2, n, D)).astype(np.uint16) | (rng.integers(0, 2, (1, 2, n, D)).astype(np.uint16) << 15)
    bits = fp16_bits(x)
    bits[..., 1, :] = sub                                             # head 1: fp16 subnormals
    # head 2 stays all zero
    y = rng.standard_normal((1, 2, n, D)).astype(np.float32) * 1e-3   # head 3: one outlier per Q4 group
    y[..., ::32] = rng.choice([-3e4, 3e4, 1e3], y[..., ::32].shape)
    bits[..., 3, :] = fp16_bits(y)
    z = rng.standard_normal((1, 2, n, D)).astype(np.float32) * 1e-2   # head 4: one outlier for the whole head
    z[0, :, 0, 0] = 6e4
    bits[..., 4, :] = fp16_bits(z)
    bits[..., 5, :] = fp16_bits(rng.choice([6.1035e-05, -6.1035e-05, 0.0], (1, 2, n, D)))
    bits[..., 6, :] = fp16_bits(rng.uniform(-65504, 65504, (1, 2, n, D)))
    bits[..., 7, :] = fp16_bits(rng.standard_normal((1, 2, n, D)) * 1e-6)   # mostly subnormal
    return bits


def _chunks(rng):
    return [("random", random_fp16_chunk(rng)), ("adversarial", adversarial_fp16_chunk(rng))]


# ---------------------------------------------------------------------------------------------------------------
# oracle: the bf16 default is what it was
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spread", [0.0, 6.0], ids=["narrow", "wide"])
def test_bf16_equals_the_bf16_oracle(spread):
    """tests/fp16_oracle.py with its default dtype="bf16" is exactly oracle/kv_oracle.py and tests/mla_oracle.py: the
    fp16 codecs are the bf16 ones with only the two conversions swapped."""
    rng = np.random.default_rng(1)
    x = rng.standard_normal((2, 2, 40, 4, 64)).astype(np.float32) * 3
    x *= np.exp(rng.uniform(-spread, spread, (2, 2, 1, 4, 1))).astype(np.float32)
    b = ko.f32_to_bf16_bits_rn(x).reshape(x.shape)
    b[0, 0, :, 1] = 0                                                    # an all-zero head
    c0, s0 = ko.fp8_pack_chunk(b)
    for kw in ({}, {"dtype": "bf16"}):
        c1, s1 = fo.fp8_pack_chunk(b, **kw)
        assert np.array_equal(c0, c1) and np.array_equal(s0, s1)
        assert np.array_equal(ko.fp8_unpack_chunk(c0, s0), fo.fp8_unpack_chunk(c0, s0, **kw))
    xf = ko.bf16_bits_to_f32(b)
    per = np.broadcast_to(s0[:, :, None, :, None], b.shape)
    assert np.array_equal(ko.fp8_tolerance(xf, per), fo.fp8_tolerance(xf, per))
    q0, t0 = ko.q4_pack_chunk(b)
    for kw in ({}, {"dtype": "bf16"}):
        q1, t1 = fo.q4_pack_chunk(b, **kw)
        assert np.array_equal(q0, q1) and np.array_equal(t0, t1)
        assert np.array_equal(ko.q4_unpack_chunk(q0, t0), fo.q4_unpack_chunk(q0, t0, **kw))
    assert np.array_equal(ko.q4_tolerance(xf), fo.q4_tolerance(xf))
    m = ko.f32_to_bf16_bits_rn(rng.standard_normal((3, 1, 10, 1, 576)).astype(np.float32)).reshape(3, 1, 10, 1, 576)
    m[0, 0, 0, 0, :128] = 0                                              # an all-zero latent group
    r0 = mo.fp8_pack_chunk(m)
    for kw in ({}, {"dtype": "bf16"}):
        assert np.array_equal(r0, fo.mla_fp8_pack_chunk(m, **kw))
        assert np.array_equal(mo.fp8_unpack_chunk(r0), fo.mla_fp8_unpack_chunk(r0, **kw))
    assert np.array_equal(mo.fp8_tolerance(m), fo.mla_fp8_tolerance(m))


def test_fp16_conversions_are_exact_and_round_to_nearest_even():
    allb = np.arange(0x7C00, dtype=np.uint16)                   # every finite non-negative fp16
    f = fo.fp16_bits_to_f32(allb)
    assert np.array_equal(fo.f32_to_fp16_bits_rn(f), allb)
    # ties to even: halfway between 1 and 1 + 2^-10 goes to 1, between 1 + 2^-10 and 1 + 2^-9 to 1 + 2^-9
    assert fo.f32_to_fp16_bits_rn(np.float32(1 + 2.0 ** -11)) == 0x3C00
    assert fo.f32_to_fp16_bits_rn(np.float32(1 + 3 * 2.0 ** -11)) == 0x3C02
    assert fo.f32_to_fp16_bits_rn(np.float32(2.0 ** -25)) == 0                 # half the smallest subnormal: even
    assert fo.f32_to_fp16_bits_rn(np.float32(3 * 2.0 ** -25)) == 2


# ---------------------------------------------------------------------------------------------------------------
# oracle: fp16 rules
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["random", "adversarial"])
def test_fp8_fp16_tolerance_finite_and_idempotent(kind):
    rng = np.random.default_rng(2)
    bits = dict(_chunks(rng))[kind]
    codes, scales = fo.fp8_pack_chunk(bits, "fp16")
    out = fo.fp8_unpack_chunk(codes, scales, "fp16")
    x = fo.fp16_bits_to_f32(bits).astype(np.float64)
    y = fo.fp16_bits_to_f32(out).astype(np.float64)
    assert np.isfinite(y).all()
    per = np.broadcast_to(scales[:, :, None, :, None], bits.shape).astype(np.float64)
    assert np.all(np.abs(x - y) <= fo.fp8_tolerance(x, per, "fp16"))
    c2, s2 = fo.fp8_pack_chunk(out, "fp16")                     # re-quantising the decoded chunk changes nothing
    assert np.array_equal(c2, codes) and np.array_equal(s2, scales)
    assert np.array_equal(fo.fp8_unpack_chunk(c2, s2, "fp16"), out)


@pytest.mark.parametrize("kind", ["random", "adversarial"])
def test_q4_fp16_tolerance_and_finite(kind):
    rng = np.random.default_rng(3)
    bits = dict(_chunks(rng))[kind]
    codes, sc = fo.q4_pack_chunk(bits, "fp16")
    out = fo.q4_unpack_chunk(codes, sc, "fp16")
    x = fo.fp16_bits_to_f32(bits).astype(np.float64)
    y = fo.fp16_bits_to_f32(out).astype(np.float64)
    assert np.isfinite(y).all()
    assert np.all(np.abs(x - y) <= fo.q4_tolerance(x, "fp16"))
    # the record layout is the bf16 one: scales are bf16 bits of absmax / 7
    amax = np.abs(x.reshape(*x.shape[:-1], -1, ko.Q4_GROUP)).max(-1)
    want = np.where(amax == 0, 0x3F80, ko.f32_to_bf16_bits_rn((amax / 7).astype(np.float32)).reshape(amax.shape))
    assert np.array_equal(sc, want)


def test_fp16_tolerance_is_tight_enough_to_catch_bf16_decoding():
    """The failure the fp16 rules fix: fp16 bits decoded as bf16 are far outside the tolerance."""
    rng = np.random.default_rng(4)
    bits = fp16_bits(rng.standard_normal((1, 2, 64, 4, 64)))
    x = fo.fp16_bits_to_f32(bits).astype(np.float64)
    codes, scales = fo.fp8_pack_chunk(bits)                              # read as bf16
    wrong = fo.fp16_bits_to_f32(fo.fp8_unpack_chunk(codes, scales)).astype(np.float64)
    c16, s16 = fo.fp8_pack_chunk(bits, "fp16")
    per = np.broadcast_to(s16[:, :, None, :, None], bits.shape)
    assert np.mean((wrong == 0) & (x != 0)) > 0.5                       # most values come back as 0
    assert np.mean(np.abs(x - wrong) > fo.fp8_tolerance(x, per, "fp16")) > 0.5
    right = fo.fp16_bits_to_f32(fo.fp8_unpack_chunk(c16, s16, "fp16")).astype(np.float64)
    assert np.median(np.abs(x - right) / np.maximum(np.abs(x), 1e-30)) < 0.05


def test_mla_fp16_records():
    rng = np.random.default_rng(5)
    x = rng.standard_normal((3, 1, 40, 1, 576)).astype(np.float32) * np.exp(rng.uniform(-8, 8, (3, 1, 40, 1, 1)))
    bits = fp16_bits(np.clip(x, -65504, 65504))
    bits[0, 0, 0, 0, :128] = 0x7BFF                                     # ±65504 groups
    bits[0, 0, 1, 0, :] = rng.integers(1, 0x400, 576)                   # subnormals only
    bits[0, 0, 2, 0, :] = 0
    rec = fo.mla_fp8_pack_chunk(bits, "fp16")
    assert rec.shape == (3, 40, mo.MLA_RECORD)
    assert np.array_equal(rec[..., mo.MLA_ROPE_OFF:].copy().view("<u2"), bits[:, 0, :, 0, 512:])   # RoPE: fp16 bits
    out = fo.mla_fp8_unpack_chunk(rec, "fp16")
    xs = fo.fp16_bits_to_f32(bits).astype(np.float64)
    ys = fo.fp16_bits_to_f32(out).astype(np.float64)
    assert np.isfinite(ys).all()
    assert np.all(np.abs(xs - ys) <= fo.mla_fp8_tolerance(bits, "fp16"))
    assert np.array_equal(fo.mla_fp8_pack_chunk(out, "fp16"), rec)


def test_every_finite_fp16_maximum_decodes_to_a_finite_value():
    """Exhaustive over the group maximum: the largest FP8 and Q4 codes of a group whose |max| is any finite fp16
    value decode to a finite fp16 value (no saturation step is needed in the decoders)."""
    m = np.arange(1, FP16_MAX_BITS + 1, dtype=np.uint16)                # every finite positive fp16
    N = len(m)
    # FP8: one head per maximum, elements (+m, -m)
    fp8 = np.stack([m, m | 0x8000], axis=-1).reshape(N, 1, 1, 1, 2)
    codes, scales = fo.fp8_pack_chunk(fp8, "fp16")
    assert np.all((codes & 0x7F) == 0x7E)                               # ±448: the largest code
    out = fo.fp8_unpack_chunk(codes, scales, "fp16")
    assert np.all((out & 0x7C00) != 0x7C00), "FP8 decoded to inf or NaN"
    assert np.all((out & 0x7FFF) <= m[:, None, None, None, None])       # never above the maximum
    # Q4: one group per maximum, elements (+m, -m, 0, ...)
    q4 = np.zeros((N, 1, 1, 1, ko.Q4_GROUP), np.uint16)
    q4[..., 0], q4[..., 1] = m[:, None, None, None], (m | 0x8000)[:, None, None, None]
    codes, sc = fo.q4_pack_chunk(q4, "fp16")
    assert np.all(codes[..., 0] == 0x97)                                # +7 low nibble, -7 high nibble
    out = fo.q4_unpack_chunk(codes, sc, "fp16")
    assert np.all((out & 0x7C00) != 0x7C00), "Q4 decoded to inf or NaN"
    top = fo.fp16_bits_to_f32(out[..., 0].reshape(-1))
    assert top[-1] == 65408.0 and top.max() == 65408.0                  # the largest case: absmax 65504


# ---------------------------------------------------------------------------------------------------------------
# geometry from vLLM's config, key namespace, format tags
# ---------------------------------------------------------------------------------------------------------------
def _vllm_config(model_dtype, cache_dtype):
    import torch
    mc = NS(model="synth-llama-2", dtype=getattr(torch, model_dtype), use_mla=False, get_num_layers=lambda pc: 32,
            get_num_kv_heads=lambda pc: 8, get_head_size=lambda: 128)
    return NS(model_config=mc, parallel_config=NS(tensor_parallel_size=1, rank=0),
              cache_config=NS(block_size=16, cache_dtype=cache_dtype))


@pytest.mark.parametrize("model,cache,elem,dtype", [
    ("float16", "auto", 2, _lib.DTYPE_FP16),
    ("bfloat16", "auto", 2, _lib.DTYPE_BF16),
    ("bfloat16", "float16", 2, _lib.DTYPE_FP16),
    ("float16", "bfloat16", 2, _lib.DTYPE_BF16),
    ("float16", "fp8", 1, _lib.DTYPE_BF16),
    ("float16", "fp8_e4m3", 1, _lib.DTYPE_BF16),
    ("bfloat16", "fp8_e5m2", 1, _lib.DTYPE_BF16),
    ("float32", "auto", 4, _lib.DTYPE_BF16),
])
def test_geometry_from_vllm_cache_dtype(model, cache, elem, dtype):
    pytest.importorskip("vllm")
    from b200kv.config import B200KVConfig
    from b200kv.connector import geometry_from_vllm
    cfg = B200KVConfig()
    cfg.fmt = _lib.FMT_FP8
    g = geometry_from_vllm(_vllm_config(model, cache), cfg)
    assert (g.elem_bytes, g.dtype) == (elem, dtype)


def test_key_seed_and_format_tags():
    from b200kv import KVGeometry, xxh64
    from b200kv.engine import DEFAULT_SEED
    for fmt in (_lib.FMT_RAW, _lib.FMT_FP8, _lib.FMT_Q4):
        for layout in (_lib.LAYOUT_NHD, _lib.LAYOUT_HND):
            g = KVGeometry(32, 8, 128, 1024, 16, 256, 2, 0, fmt, layout)
            today = xxh64(f"m|2|1|32|8|128|2|256|{fmt}|{layout}".encode(), DEFAULT_SEED)
            assert g.key_seed("m", 2, 1) == today                       # bf16 keys are what they were
            g16 = KVGeometry(32, 8, 128, 1024, 16, 256, 2, 0, fmt, layout, _lib.DTYPE_FP16)
            assert g16.key_seed("m", 2, 1) != today                     # RAW included
            assert g16.key_seed("m", 2, 1) == xxh64(f"m|2|1|32|8|128|2|256|{fmt}|{layout}|fp16".encode(), DEFAULT_SEED)
            assert g.fmt_tag == fmt | (layout << 8)                     # bf16 tags are what they were
            assert g16.fmt_tag == fmt | (layout << 8) | (1 << 16)
    gm = KVGeometry(61, 1, 576, 64, 64, 256, 2, 0, _lib.FMT_FP8, _lib.LAYOUT_MLA, _lib.DTYPE_FP16)
    assert gm.key_seed("m", 8, 3) == gm.key_seed("m", 8, 0)             # MLA still shares one seed per stage
    assert gm.fmt_tag == _lib.FMT_FP8 | (_lib.LAYOUT_MLA << 8) | (1 << 16)


# ---------------------------------------------------------------------------------------------------------------
# P/D: producer and consumer must agree on the cache dtype
# ---------------------------------------------------------------------------------------------------------------
class _PdEngine:
    def __init__(self, dtype=None):
        g = dict(n_blocks=64, stride=4096, n_layers=2, n_kv_heads=2, head_dim=8, block_tokens=16, elem_bytes=2, layout=0)
        if dtype is not None:
            g["dtype"] = dtype
        self.geom = NS(**g)

    def export_ipc(self):
        return b"\x07" * (72 * 4)

    def import_peer(self, pid, device, descs, stride, n_blocks):
        self.imported = (pid, device, len(descs), stride, n_blocks)


def test_pd_dtype_mismatch_is_refused(tmp_path, monkeypatch):
    from b200kv import pd
    monkeypatch.setattr(pd, "SHM_DIR", str(tmp_path))
    pd.publish_ipc("P-fp16", _PdEngine(_lib.DTYPE_FP16), device=0)
    with pytest.raises(ValueError, match="dtype"):
        pd.PeerResolver(_PdEngine(_lib.DTYPE_BF16)).resolve("P-fp16")
    assert pd.PeerResolver(_PdEngine(_lib.DTYPE_FP16)).resolve("P-fp16") == 0


def test_pd_document_without_dtype_reads_as_bf16(tmp_path, monkeypatch):
    from b200kv import pd
    monkeypatch.setattr(pd, "SHM_DIR", str(tmp_path))
    path = pd.publish_ipc("P-old", _PdEngine(_lib.DTYPE_BF16), device=0)
    doc = json.load(open(path))
    assert doc.pop("dtype") == _lib.DTYPE_BF16
    with open(path, "w") as f:
        json.dump(doc, f)                                                # as a producer without the field wrote it
    assert pd.PeerResolver(_PdEngine(_lib.DTYPE_BF16)).resolve("P-old") == 0
    assert pd.PeerResolver(_PdEngine()).resolve("P-old") == 0           # a geometry without the field is bf16 too
    with pytest.raises(ValueError, match="dtype"):
        pd.PeerResolver(_PdEngine(_lib.DTYPE_FP16)).resolve("P-old")
    assert os.path.exists(path)
