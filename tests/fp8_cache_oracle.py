"""CPU specification of the Q4 chunk format for fp8 KV caches (vLLM's --kv-cache-dtype fp8 / fp8_e4m3 / fp8_e5m2;
B200KV_DTYPE_E4M3 / B200KV_DTYPE_E5M2 on a 1-byte engine) — TEST INFRASTRUCTURE ONLY.

Extends oracle/kv_oracle.py, which specifies Q4 for bf16 caches (tests/fp16_oracle.py for fp16 ones).  The record
is the same: per token and plane [H*D/2 code bytes][H*D/32 bf16 scales], element 2i in the low nibble of byte i.
Only the two conversions differ, and here they are fp8 codes -> value and value -> fp8 codes.  The rules:

* decode: every code of the cache's type (e4m3fn or e5m2) is its exact value (torch.float8_e4m3fn /
  torch.float8_e5m2), NaN and e5m2's infinities included.  The kernels decode through f16, which holds every fp8
  value exactly.
* absmax is taken on the 7 magnitude bits (code & 0x7f).  Their integer order is magnitude order: the finite codes,
  then e5m2's inf (0x7c), then the NaN codes (e4m3fn 0x7f; e5m2 0x7d..0x7f).
* store: s = bf16_rn(fl32(absmax / 7)), 1 when absmax is 0; inv = fl32(1 / s); q = rint(x * inv) of the exact
  product, ties to even.  This is the 16-bit rule.  For finite groups |q| <= 7.
* load: q * s is exact in fp32 (4 x 8 significant bits), then one encode to the cache's type, round to nearest even,
  saturating to the largest finite code (cvt.rn.satfinite.e4m3x2.f32 / e5m2x2.f32).  NaN encodes to 0x7f.
* vLLM's per-layer k_scale / v_scale multiply the code's value when attention reads it, on the storing replica and on
  the loading one alike, so the format works on the code's value and never sees them.
* non-finite codes follow from IEEE arithmetic on the same steps, and the kernels produce the same bits:
  - a group holding a NaN code has absmax NaN, s = NaN (bf16 bits 0x7fff), inv = NaN, and every q is NaN.  The
    kernel rounds by fma(x, inv, 1.5 * 2^23) and keeps the low nibble: for NaN (0x7fffffff) that is 0xf, q = -1.
    Loaded, every element of the group is -1 * NaN -> NaN -> 0x7f.
  - an e5m2 group holding inf has s = inf (0x7f80) and inv = 0: finite elements get q = 0, infinite ones inf * 0 =
    NaN -> q = -1.  Loaded, 0 * inf is NaN (0x7f) and -1 * inf saturates to -57344 (0xfb).
  So a group with a non-finite code does not survive Q4; every finite group does within q4_fp8_tolerance.

The CUDA kernels kv_q4_store_fp8_kernel / kv_q4_load_fp8_kernel (production-stack_b200/csrc/b200kv_kernels.cuh)
follow this file bit for bit.
"""
from __future__ import annotations

import numpy as np
import torch

from oracle import kv_oracle as ko

FP8_TYPES = ("e4m3", "e5m2")
_TORCH = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}
MAX_FINITE_CODE = {"e4m3": 0x7E, "e5m2": 0x7B}
NAN_CODE = 0x7F
BF16_NAN = 0x7FFF     # what cvt.rn.bf16.f32 makes of a NaN


def decode_table(ft: str) -> np.ndarray:
    """(256,) float64: the value of every code of `ft`."""
    assert ft in FP8_TYPES, ft
    return torch.arange(256, dtype=torch.int32).to(torch.uint8).view(_TORCH[ft]).to(torch.float64).numpy()


_DEC = {ft: decode_table(ft) for ft in FP8_TYPES}


def codes_to_f64(codes: np.ndarray, ft: str) -> np.ndarray:
    return _DEC[ft][np.asarray(codes, dtype=np.uint8)]


def encode_rn_satfinite(x: np.ndarray, ft: str) -> np.ndarray:
    """Values (exact, float64) -> codes of `ft`: round to nearest, ties to the even code, |x| above the largest finite
    value (inf included) -> the largest finite code, NaN -> 0x7f, sign kept (also for a result that rounds to 0)."""
    x = np.asarray(x, dtype=np.float64)
    grid = _DEC[ft][:MAX_FINITE_CODE[ft] + 1]            # the non-negative finite values, ascending with the code
    nan = np.isnan(x)
    a = np.where(nan, 0.0, np.minimum(np.abs(x), grid[-1]))
    hi = np.minimum(np.searchsorted(grid, a, side="left"), len(grid) - 1)
    lo = np.maximum(hi - 1, 0)
    d_lo, d_hi = a - grid[lo], grid[hi] - a
    code = np.where(d_hi < d_lo, hi, np.where(d_lo < d_hi, lo, np.where(hi % 2 == 0, hi, lo)))
    code = code.astype(np.uint8) | np.where(np.signbit(x), np.uint8(0x80), np.uint8(0))
    return np.where(nan, np.uint8(NAN_CODE), code).astype(np.uint8)


def _bf16_bits_rn(x32: np.ndarray) -> np.ndarray:
    x32 = np.asarray(x32, dtype=np.float32)
    return np.where(np.isnan(x32), np.uint16(BF16_NAN), ko.f32_to_bf16_bits_rn(x32)).astype(np.uint16)


def group_scales(mag_codes: np.ndarray, ft: str) -> np.ndarray:
    """Magnitude codes (code & 0x7f) of the group maxima -> bf16 scale bits: bf16_rn(fl32(absmax / 7)), or 1.0."""
    amax = codes_to_f64(mag_codes, ft).astype(np.float32)
    with np.errstate(invalid="ignore", over="ignore"):
        a7 = (amax / np.float32(7.0)).astype(np.float32)
    return np.where(np.asarray(mag_codes) == 0, np.uint16(0x3F80), _bf16_bits_rn(a7)).astype(np.uint16)


def q4_pack_chunk(codes: np.ndarray, ft: str):
    """(L, 2, n, H, D) fp8 codes of `ft` -> (Q4 codes uint8 (L,2,n,H,D/2), scales uint16 bf16 bits (L,2,n,H,D/32)),
    the arrays oracle/kv_oracle.py q4_pack_chunk returns for a 16-bit cache."""
    G = ko.Q4_GROUP
    L, two, n, H, D = codes.shape
    assert D % G == 0
    c = np.asarray(codes, dtype=np.uint8).reshape(L, two, n, H, D // G, G)
    s_bits = group_scales((c & 0x7F).max(axis=-1), ft)
    s = ko.bf16_bits_to_f32(s_bits)
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = (np.float32(1.0) / s).astype(np.float32)
        p = codes_to_f64(c, ft) * inv[..., None].astype(np.float64)     # exact: 24 + 24 bits
    nan = np.isnan(p)
    q = np.where(nan, -1.0, np.rint(np.where(nan, 0.0, p)))
    assert np.all(np.abs(q) <= 7)
    nib = (q.astype(np.int8) & 0xF).astype(np.uint8).reshape(L, two, n, H, D)
    return (nib[..., 0::2] | (nib[..., 1::2] << 4)).astype(np.uint8), s_bits


def q4_values(qcodes: np.ndarray, scale_bits: np.ndarray) -> np.ndarray:
    """(L,2,n,H,D/2) Q4 codes + (L,2,n,H,D/32) bf16 scale bits -> q * s as float64 (exact, as in fp32)."""
    L, two, n, H, Dh = qcodes.shape
    lo = (qcodes & 0xF).astype(np.int8)
    hi = (qcodes >> 4).astype(np.int8)
    q = np.empty((L, two, n, H, 2 * Dh), dtype=np.float64)
    q[..., 0::2], q[..., 1::2] = np.where(lo > 7, lo - 16, lo), np.where(hi > 7, hi - 16, hi)
    s = ko.bf16_bits_to_f32(scale_bits).astype(np.float64)
    with np.errstate(invalid="ignore"):
        return (q.reshape(L, two, n, H, -1, ko.Q4_GROUP) * s[..., None]).reshape(L, two, n, H, 2 * Dh)


def q4_unpack_chunk(qcodes: np.ndarray, scale_bits: np.ndarray, ft: str) -> np.ndarray:
    """Inverse of q4_pack_chunk: (L,2,n,H,D) fp8 codes of `ft`, one RN satfinite encode of q * s."""
    return encode_rn_satfinite(q4_values(qcodes, scale_bits), ft)


def q4_fp8_tolerance(x: np.ndarray, ft: str) -> np.ndarray:
    """Bound on |x - x̂| for finite (L,2,n,H,D) values x: s/2 from Q4, plus one fp8 rounding of q * s, which is at
    most half the fp8 grid step at |q * s| <= |x| + s/2 (relative 2^-4 for e4m3, 2^-3 for e5m2, and the subnormal
    half-quantum 2^-10 / 2^-17 near 0).  s is the group's bf16 scale, so the bound holds exactly, not up to a factor:
    |x - q s| <= s/2 because inv = fl32(1/s) makes |x * inv - x / s| < 2^-23 * 7.5 < 1/2 - ... never move a rint."""
    G = ko.Q4_GROUP
    L, two, n, H, D = x.shape
    rel, sub = (2.0 ** -4, 2.0 ** -10) if ft == "e4m3" else (2.0 ** -3, 2.0 ** -17)
    amax = np.abs(x.reshape(L, two, n, H, D // G, G)).max(axis=-1)
    s = ko.bf16_bits_to_f32(_bf16_bits_rn((amax / 7.0).astype(np.float32))).astype(np.float64)
    s = np.where(amax == 0, 1.0, s)
    s = np.repeat(s, G, axis=-1).reshape(x.shape)
    y = np.abs(x) + s / 2
    return s / 2 + np.maximum(y * rel, sub)
