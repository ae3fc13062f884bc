"""CPU specification of the FP8 and Q4 chunk formats for fp16 KV caches (B200KV_DTYPE_FP16) — TEST
INFRASTRUCTURE ONLY.

Extends oracle/kv_oracle.py (K/V FP8 and Q4) and tests/mla_oracle.py (MLA FP8 latent records), which specify
the formats for bf16 caches.  Every codec here takes ``dtype="bf16"`` (the default) or ``dtype="fp16"``.  The
computation is the same for both types, and only the two conversions depend on the type: 16-bit bits -> fp32,
and fp32 -> 16-bit bits.  With ``dtype="bf16"`` every function returns exactly what its counterpart in those
two modules returns; tests/test_fp16_cpu.py checks that.  The fp16 rules:

* absmax is taken on the 16-bit magnitude bits with the sign cleared.  Integer order equals magnitude order for
  fp16 as for bf16.  Only the conversion of that maximum to fp32 differs, and it is exact either way.
* FP8: scale = fl32(absmax / 448), codes = e4m3_rn_satfinite(fl32(x * fl32(448 / absmax))), with x converted
  exactly from fp16.  This is the bf16 rule.
* Q4: the record layout is unchanged, and the group scale stays bf16 bits, bf16_rn(absmax / 7).  bf16 keeps the
  range that fp16 lacks for groups of small values, and the record format does not depend on the cache type.
* MLA FP8 record: the same 656 bytes.  The 512 codes and 4 fp32 scales follow the FP8 rule per 128-element group.
  The 64 RoPE elements are the cache's own 16-bit bits, copied verbatim, so they are fp16 bits in an fp16 cache.
  That departs from vLLM's fp8_ds_mla, whose RoPE part is bf16.  Such chunks carry the fp16 format tag and key
  seed, so they are never read as the bf16 record.
* decode: one rounding, fp32 product -> fp16, round to nearest even.  It never goes through bf16.
* no inf from finite input.  FP8 decodes to at most 448 * fl32(absmax / 448), which rounds to absmax or below in
  fp16.  Q4's bf16_rn(absmax / 7) may round up, but 7 * bf16_rn(absmax / 7) stays finite for every finite fp16
  absmax; the worst case is absmax 65504 -> 65408.  tests/test_fp16_cpu.py checks every finite maximum.
* non-finite inputs are out of scope, as they are for bf16.

The CUDA kernels (kv_fp8_store3 / kv_fp8_store / kv_fp8_load / kv_q4_store / kv_q4_load / kv_mla_fp8_store /
kv_mla_fp8_load, built for Src<kFp16>) follow this file bit for bit.
"""
from __future__ import annotations

import numpy as np

from oracle import kv_oracle as ko
from tests import mla_oracle as mo

DTYPES = ("bf16", "fp16")


# ---------------------------------------------------------------------------------------------
# the two conversions that depend on the cache type
# ---------------------------------------------------------------------------------------------
def fp16_bits_to_f32(u16: np.ndarray) -> np.ndarray:
    return np.ascontiguousarray(u16, dtype=np.uint16).view(np.float16).astype(np.float32)


def f32_to_fp16_bits_rn(x: np.ndarray) -> np.ndarray:
    """fp32 -> fp16 round-to-nearest-even, subnormals included (what __float2half_rn does for finite values)."""
    return np.ascontiguousarray(x, dtype=np.float32).astype(np.float16).view(np.uint16)


def bits_to_f32(u16: np.ndarray, dtype: str = "bf16") -> np.ndarray:
    """16-bit cache bit patterns of `dtype` -> fp32 (exact)."""
    assert dtype in DTYPES, dtype
    return ko.bf16_bits_to_f32(u16) if dtype == "bf16" else fp16_bits_to_f32(u16)


def f32_to_bits_rn(x: np.ndarray, dtype: str = "bf16") -> np.ndarray:
    """fp32 -> 16-bit bit patterns of `dtype`, one round-to-nearest-even."""
    assert dtype in DTYPES, dtype
    return ko.f32_to_bf16_bits_rn(x) if dtype == "bf16" else f32_to_fp16_bits_rn(x)


# ---------------------------------------------------------------------------------------------
# K/V FP8 (oracle/kv_oracle.py fp8_*)
# ---------------------------------------------------------------------------------------------
def fp8_pack_chunk(chunk_bits: np.ndarray, dtype: str = "bf16"):
    """(L, 2, n, H, D) 16-bit bit patterns of `dtype` -> (codes uint8 same shape, scales f32 (L,2,H)).
    One scale per (chunk, layer, K/V, head): scale = absmax/448, codes = e4m3(x * (448/absmax)); absmax == 0 ->
    scale 1."""
    L, two, n, H, D = chunk_bits.shape
    mag = (chunk_bits & 0x7FFF).astype(np.uint16)
    amax_bits = mag.max(axis=(2, 4)) if n else np.zeros((L, two, H), np.uint16)  # (L, 2, H)
    amax = bits_to_f32(amax_bits, dtype)
    zero = amax_bits == 0
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = np.where(zero, np.float32(1.0), np.float32(448.0) / amax).astype(np.float32)
        scale = np.where(zero, np.float32(1.0), amax / np.float32(448.0)).astype(np.float32)
    x = bits_to_f32(chunk_bits, dtype)
    y = (x * inv[:, :, None, :, None]).astype(np.float32)
    return ko.f32_to_e4m3_satfinite(y), scale


def fp8_unpack_chunk(codes: np.ndarray, scales: np.ndarray, dtype: str = "bf16") -> np.ndarray:
    """Inverse: rn(float(e4m3) * scale) to `dtype`, as uint16 bit patterns."""
    x = ko._E4M3_DEC[codes] * scales[:, :, None, :, None].astype(np.float32)
    return f32_to_bits_rn(x.astype(np.float32), dtype)


def fp8_tolerance(x: np.ndarray, scale_per_elem: np.ndarray, dtype: str = "bf16") -> np.ndarray:
    """Stated tolerance of the fp8 path:
    bf16: |x - x̂| <= max(2^-4 |x|, 2^-10 * absmax) + 2^-8 |x|             with absmax = 448 * scale
    fp16: |x - x̂| <= max(2^-4 |x|, 2^-10 * absmax) + 2^-11 |x| + 2^-25

    fp16 derivation.  y = fl32(x * inv) is the scaled value, c its e4m3 code, x̂ = fp16_rn(fl32(dec(c) * scale)).
    * e4m3: in binade [2^e, 2^(e+1)) the grid step is 2^(e-3), so |y - dec(c)| <= 2^(e-4).  The error reaches
      2^(e-4) only for |y| >= 2^e (1 + 2^-4), hence |y - dec(c)| <= 2^-4 |y| / (1 + 2^-4).  Below 2^-6 the grid
      is 2^-9, so |y - dec(c)| <= 2^-10, i.e. 2^-10 * scale <= 2^-10 * absmax in x units.
    * fp32: fl32(448/absmax), fl32(x * inv) and fl32(dec * scale) add at most ~4 * 2^-24 |x|.
    * fp16: one RN rounding of the result.  It adds <= 2^-11 |x̂| for normal results and <= 2^-25 (half the
      subnormal quantum 2^-24) for subnormal ones.  |x̂| <= |x| (1 + 2^-4) + ..., so 2^-11 |x̂| is 2^-11 |x| plus
      at most 2^-15 |x|.
    The e4m3 term falls short of 2^-4 |x| by 2^-4 |x| (2^-4 / (1 + 2^-4)) > 2^-9 |x|.  That covers the fp32 terms
    and the 2^-15 |x|.  What remains is 2^-11 |x| + 2^-25: the bf16 bound's re-rounding term 2^-8 |x| replaced by
    fp16's.  tests/test_fp16_cpu.py checks the bound on adversarial groups (±65504, subnormals, outliers)."""
    assert dtype in DTYPES, dtype
    if dtype == "bf16":
        return ko.fp8_tolerance(x, scale_per_elem)
    ax = np.abs(x)
    return np.maximum(ax * 2.0 ** -4, 2.0 ** -10 * 448.0 * scale_per_elem) + ax * 2.0 ** -11 + 2.0 ** -25


# ---------------------------------------------------------------------------------------------
# K/V Q4 (oracle/kv_oracle.py q4_*)
# ---------------------------------------------------------------------------------------------
def q4_pack_chunk(chunk_bits: np.ndarray, dtype: str = "bf16"):
    """(L, 2, n, H, D) 16-bit bit patterns of `dtype` -> (codes uint8 (L,2,n,H,D/2), scales uint16 bf16 bits
    (L,2,n,H,D/G)).  The scales are bf16 whatever the cache type."""
    G = ko.Q4_GROUP
    L, two, n, H, D = chunk_bits.shape
    assert D % G == 0
    x = bits_to_f32(chunk_bits, dtype).reshape(L, two, n, H, D // G, G)
    amax = np.abs(x).max(axis=-1)
    s_bits = np.where(amax == 0, ko.f32_to_bf16_bits_rn(np.float32(1.0)),
                      ko.f32_to_bf16_bits_rn((amax / np.float32(7.0)).astype(np.float32)))
    s = ko.bf16_bits_to_f32(s_bits)
    # one IEEE division per group, then rint of the EXACT product x * inv (float64 holds it exactly: 24 + 24 bits)
    inv = (np.float32(1.0) / s).astype(np.float32)
    q = np.clip(np.rint(x.astype(np.float64) * inv[..., None].astype(np.float64)), -7, 7).astype(np.int8)
    q = q.reshape(L, two, n, H, D)
    nib = (q & 0xF).astype(np.uint8)
    codes = (nib[..., 0::2] | (nib[..., 1::2] << 4)).astype(np.uint8)
    return codes, s_bits.astype(np.uint16)


def q4_unpack_chunk(codes: np.ndarray, scale_bits: np.ndarray, dtype: str = "bf16") -> np.ndarray:
    """Inverse: rn(code * scale) to `dtype`, as uint16 bit patterns."""
    L, two, n, H, Dh = codes.shape
    lo = (codes & 0xF).astype(np.int8)
    hi = (codes >> 4).astype(np.int8)
    lo = np.where(lo > 7, lo - 16, lo)
    hi = np.where(hi > 7, hi - 16, hi)
    q = np.empty((L, two, n, H, 2 * Dh), dtype=np.float32)
    q[..., 0::2], q[..., 1::2] = lo, hi
    s = ko.bf16_bits_to_f32(scale_bits)
    x = (q.reshape(L, two, n, H, -1, ko.Q4_GROUP) * s[..., None]).astype(np.float32)
    return f32_to_bits_rn(x.reshape(L, two, n, H, 2 * Dh), dtype)


def q4_tolerance(x: np.ndarray, dtype: str = "bf16") -> np.ndarray:
    """bf16: oracle/kv_oracle.py q4_tolerance, |x - x̂| <= step/2 + 2^-7 |x| with step = absmax/7 * (1 + 2^-7).
    fp16: |x - x̂| <= step/2 + 2^-11 |x| + 2^-25.

    fp16 derivation (the scale s is still bf16, s <= absmax/7 * (1 + 2^-8)).  q = rint(x * inv) with
    inv = fl32(1/s) gives |x - q s| <= s/2 + 2^-24 |x|.  q s is exact in fp32 (4 x 8 significant bits), and its
    one fp16 rounding adds <= 2^-11 |q s| (normal) or 2^-25 (subnormal), with |q s| <= |x| + s/2.  The step term
    uses (1 + 2^-7) where s needs only (1 + 2^-8).  The difference, absmax/14 * 2^-8 > 2^-12 s, covers
    2^-11 * s/2 and 2^-24 |x|.  So the bf16 bound holds with its re-rounding term 2^-7 |x| replaced by fp16's
    2^-11 |x| + 2^-25."""
    assert dtype in DTYPES, dtype
    if dtype == "bf16":
        return ko.q4_tolerance(x)
    G = ko.Q4_GROUP
    L, two, n, H, D = x.shape
    amax = np.abs(x.reshape(L, two, n, H, D // G, G)).max(axis=-1, keepdims=True)
    step = np.broadcast_to(amax / 7.0 * (1 + 2.0 ** -7), (L, two, n, H, D // G, G)).reshape(x.shape)
    return step / 2 + np.abs(x) * 2.0 ** -11 + 2.0 ** -25


# ---------------------------------------------------------------------------------------------
# MLA FP8 latent records (tests/mla_oracle.py fp8_*)
# ---------------------------------------------------------------------------------------------
def mla_fp8_pack_chunk(chunk_bits: np.ndarray, dtype: str = "bf16") -> np.ndarray:
    """(L, 1, n, 1, 576) 16-bit bit patterns of `dtype` -> (L, n, 656) uint8 records."""
    L, one, n, h, D = chunk_bits.shape
    assert one == 1 and h == 1 and D == mo.MLA_D
    bits = chunk_bits.reshape(L, n, D)
    amax_bits = mo._group_amax_bits(bits)                               # (L, n, 4): magnitude bits
    amax = bits_to_f32(amax_bits, dtype)
    zero = amax_bits == 0
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = np.where(zero, np.float32(1.0), np.float32(448.0) / amax).astype(np.float32)
        scale = np.where(zero, np.float32(1.0), amax / np.float32(448.0)).astype(np.float32)
    x = bits_to_f32(bits[..., :mo.MLA_LATENT], dtype).reshape(L, n, 4, mo.MLA_GROUP)
    codes = ko.f32_to_e4m3_satfinite((x * inv[..., None]).astype(np.float32)).reshape(L, n, mo.MLA_LATENT)
    rec = np.zeros((L, n, mo.MLA_RECORD), dtype=np.uint8)
    rec[..., :mo.MLA_SCALES_OFF] = codes
    rec[..., mo.MLA_SCALES_OFF:mo.MLA_ROPE_OFF] = np.ascontiguousarray(scale, dtype="<f4").view(np.uint8).reshape(L, n, 16)
    rec[..., mo.MLA_ROPE_OFF:] = np.ascontiguousarray(bits[..., mo.MLA_LATENT:], dtype="<u2").view(np.uint8).reshape(L, n, 128)
    return rec


def mla_fp8_unpack_chunk(records: np.ndarray, dtype: str = "bf16") -> np.ndarray:
    """(L, n, 656) records -> (L, 1, n, 1, 576) 16-bit bit patterns of `dtype`."""
    L, n, _ = records.shape
    scale = mo.record_scales(records)
    x = ko._E4M3_DEC[records[..., :mo.MLA_LATENT]].reshape(L, n, 4, mo.MLA_GROUP) * scale[..., None]
    out = np.empty((L, n, mo.MLA_D), dtype=np.uint16)
    out[..., :mo.MLA_LATENT] = f32_to_bits_rn(x.astype(np.float32), dtype).reshape(L, n, mo.MLA_LATENT)
    out[..., mo.MLA_LATENT:] = np.ascontiguousarray(records[..., mo.MLA_ROPE_OFF:]).view("<u2")
    return out[:, None, :, None, :]


def mla_fp8_tolerance(chunk_bits: np.ndarray, dtype: str = "bf16") -> np.ndarray:
    """Per-element bound on |x - decode(encode(x))| for (L, 1, n, 1, 576) bits of `dtype`: fp8_tolerance with the
    group's absmax (scale = absmax / 448) on the latent, 0 on the RoPE elements (copied exactly)."""
    L, _, n, _, D = chunk_bits.shape
    bits = chunk_bits.reshape(L, n, D)
    x = bits_to_f32(bits, dtype).astype(np.float64)
    scale = bits_to_f32(mo._group_amax_bits(bits), dtype).astype(np.float64) / 448.0
    per_elem = np.repeat(scale, mo.MLA_GROUP, axis=-1)
    tol = np.zeros_like(x)
    tol[..., :mo.MLA_LATENT] = fp8_tolerance(x[..., :mo.MLA_LATENT], per_elem, dtype)
    return tol.reshape(chunk_bits.shape)
