"""CPU specification of the MLA (multi-head latent attention) KV path — TEST INFRASTRUCTURE ONLY.

Extends oracle/kv_oracle.py to models with one latent plane per layer (DeepSeek-V2/V3, Kimi-K2):

* vLLM's MLA backends allocate one tensor per layer shaped (num_blocks, block_size, head_size) with
  strides (bs*D, D, 1) ([vllm-0.22] model_executor/layers/attention/mla_attention.py,
  MLACommonBackend.get_kv_cache_shape); head_size = kv_lora_rank 512 + qk_rope_head_dim 64 = 576.
* LMCache's MLA chunk is kv_shape = (num_layer, 1, chunk, 1, head_size)
  ([vllm-0.22] lmcache_integration/vllm_v1_adapter.py:463-477).  RAW chunks are that, token-major.
* The FP8 latent record (B200KV_LAYOUT_MLA + B200KV_FMT_FP8, include/b200kv.h) is the byte layout of
  vLLM's fp8_ds_mla entry ([vllm-0.22] v1/attention/backends/mla/flashmla_sparse.py:68-79), 656 bytes
  per (token, layer):
      [0, 512)    e4m3 codes of latent elements 0..511
      [512, 528)  4 fp32 scales; scale g covers elements [128g, 128g + 128)
      [528, 656)  RoPE elements 512..575, bf16 bits verbatim
  with this project's FP8 rule applied per group: scale = fl32(absmax / 448), inv = fl32(448 / absmax),
  code = e4m3_rn_satfinite(fl32(x * inv)), absmax == 0 -> scale = inv = 1; decode bf16_rn(e4m3 * scale).
  A chunk is L slabs of C records, rounded up to 256 bytes.
The CUDA kernels kv_mla_fp8_store_kernel / kv_mla_fp8_load_kernel follow this file bit for bit.
"""
from __future__ import annotations

import numpy as np

from oracle import kv_oracle as ko

MLA_D = 576
MLA_LATENT = 512
MLA_GROUP = 128
MLA_RECORD = 656
MLA_SCALES_OFF = 512
MLA_ROPE_OFF = 528


def chunk_bytes(n_layers: int, chunk_tokens: int, head_dim: int = MLA_D, elem_bytes: int = 2, fmt: str = "raw") -> int:
    if fmt == "raw":
        return n_layers * chunk_tokens * head_dim * elem_bytes
    assert fmt == "fp8" and head_dim == MLA_D and elem_bytes == 2
    return (n_layers * chunk_tokens * MLA_RECORD + 255) // 256 * 256


def gather_tokens(layers, slot_mapping) -> np.ndarray:
    """Paged latent planes (list of L arrays (NB, bs, D)) -> (L, 1, n, 1, D): layer.reshape(NB*bs, D)[slot_mapping]."""
    sm = np.asarray(slot_mapping, dtype=np.int64)
    out = [layer.reshape(-1, layer.shape[-1])[sm] for layer in layers]
    return np.stack(out, axis=0)[:, None, :, None, :]


def scatter_tokens(layers, chunk: np.ndarray, slot_mapping) -> None:
    """Inverse of gather_tokens, in place."""
    sm = np.asarray(slot_mapping, dtype=np.int64)
    for l, layer in enumerate(layers):
        flat = layer.reshape(-1, layer.shape[-1])
        assert np.shares_memory(flat, layer)
        flat[sm] = chunk[l, 0, :, 0, :]


def _group_amax_bits(bits: np.ndarray) -> np.ndarray:
    """(..., 576) bf16 bits -> (..., 4) bf16 bits of each latent group's absmax."""
    mag = (bits[..., :MLA_LATENT] & 0x7FFF).astype(np.uint16)
    return mag.reshape(*bits.shape[:-1], MLA_LATENT // MLA_GROUP, MLA_GROUP).max(axis=-1)


def fp8_pack_chunk(chunk_bits: np.ndarray) -> np.ndarray:
    """(L, 1, n, 1, 576) bf16 bit patterns (uint16) -> (L, n, 656) uint8 records."""
    L, one, n, h, D = chunk_bits.shape
    assert one == 1 and h == 1 and D == MLA_D
    bits = chunk_bits.reshape(L, n, D)
    amax_bits = _group_amax_bits(bits)                                  # (L, n, 4)
    amax = ko.bf16_bits_to_f32(amax_bits)
    zero = amax_bits == 0
    with np.errstate(divide="ignore", invalid="ignore"):
        inv = np.where(zero, np.float32(1.0), np.float32(448.0) / amax).astype(np.float32)
        scale = np.where(zero, np.float32(1.0), amax / np.float32(448.0)).astype(np.float32)
    x = ko.bf16_bits_to_f32(bits[..., :MLA_LATENT]).reshape(L, n, 4, MLA_GROUP)
    codes = ko.f32_to_e4m3_satfinite((x * inv[..., None]).astype(np.float32)).reshape(L, n, MLA_LATENT)
    rec = np.zeros((L, n, MLA_RECORD), dtype=np.uint8)
    rec[..., :MLA_SCALES_OFF] = codes
    rec[..., MLA_SCALES_OFF:MLA_ROPE_OFF] = np.ascontiguousarray(scale, dtype="<f4").view(np.uint8).reshape(L, n, 16)
    rec[..., MLA_ROPE_OFF:] = np.ascontiguousarray(bits[..., MLA_LATENT:], dtype="<u2").view(np.uint8).reshape(L, n, 128)
    return rec


def record_scales(records: np.ndarray) -> np.ndarray:
    """(L, n, 656) records -> (L, n, 4) fp32 scales."""
    return np.ascontiguousarray(records[..., MLA_SCALES_OFF:MLA_ROPE_OFF]).view("<f4").astype(np.float32)


def fp8_unpack_chunk(records: np.ndarray) -> np.ndarray:
    """(L, n, 656) records -> (L, 1, n, 1, 576) bf16 bit patterns."""
    L, n, _ = records.shape
    scale = record_scales(records)
    x = ko._E4M3_DEC[records[..., :MLA_LATENT]].reshape(L, n, 4, MLA_GROUP) * scale[..., None]
    out = np.empty((L, n, MLA_D), dtype=np.uint16)
    out[..., :MLA_LATENT] = ko.f32_to_bf16_bits_rn(x.astype(np.float32)).reshape(L, n, MLA_LATENT)
    out[..., MLA_LATENT:] = np.ascontiguousarray(records[..., MLA_ROPE_OFF:]).view("<u2")
    return out[:, None, :, None, :]


def fp8_tolerance(chunk_bits: np.ndarray) -> np.ndarray:
    """Per-element bound on |x - decode(encode(x))| for (L, 1, n, 1, 576) bf16 bits: oracle fp8_tolerance with the
    group's absmax (scale = absmax / 448) on the latent, 0 on the RoPE elements (copied exactly)."""
    L, _, n, _, D = chunk_bits.shape
    bits = chunk_bits.reshape(L, n, D)
    x = ko.bf16_bits_to_f32(bits).astype(np.float64)
    scale = ko.bf16_bits_to_f32(_group_amax_bits(bits)).astype(np.float64) / 448.0
    per_elem = np.repeat(scale, MLA_GROUP, axis=-1)
    tol = np.zeros_like(x)
    tol[..., :MLA_LATENT] = ko.fp8_tolerance(x[..., :MLA_LATENT], per_elem)
    return tol.reshape(chunk_bits.shape)
