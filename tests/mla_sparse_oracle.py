"""CPU specification of sparse-attention MLA caches (DeepSeek-V3.2) — TEST INFRASTRUCTURE ONLY.

Extends tests/mla_oracle.py (unchanged) with the indexer key cache that DeepSeek Sparse Attention keeps next to
each layer's latent:

* vLLM allocates one indexer cache per layer shaped (num_blocks, block_size, 132) uint8
  ([vllm-0.22] v1/attention/backends/mla/indexer.py, DeepseekV32IndexerBackend.get_kv_cache_shape; the layer is
  DeepseekV32IndexerCache, model_executor/models/deepseek_v2.py).  It is not token-major:
  indexer_k_quant_and_cache writes a block as [bs][128] e4m3 values followed by [bs][4] bytes, one fp32 scale per
  token.  Byte b of a block is value byte b % 128 of token b // 128 for b < bs*128, and scale byte of token
  (b - bs*128) // 4 after that.
* A chunk (b200kv_set_indexer, include/b200kv.h) is the engine's MLA chunk as before — RAW (L, 1, C, 1, D) slabs or
  L slabs of C 656-byte FP8 records — not rounded, followed by L indexer slabs.  Slab l is [C][128] values then
  [C][4] scales of layer l, mirroring the tile, so a whole block moves as two contiguous pieces on both sides.  The
  whole chunk is rounded up to 256 bytes.  Indexer bytes are copied verbatim in every format.
The CUDA kernel kv_indexer_copy_kernel follows this file bit for bit.
"""
from __future__ import annotations

import numpy as np

from tests import mla_oracle as mo

IDX_VALUE = 128
IDX_SCALE = 4
IDX_TOKEN = IDX_VALUE + IDX_SCALE


def latent_bytes(n_layers: int, chunk_tokens: int, head_dim: int = mo.MLA_D, elem_bytes: int = 2,
                 fmt: str = "raw") -> int:
    """The latent part of a chunk, not rounded."""
    if fmt == "raw":
        return n_layers * chunk_tokens * head_dim * elem_bytes
    assert fmt == "fp8" and head_dim == mo.MLA_D and elem_bytes == 2
    return n_layers * chunk_tokens * mo.MLA_RECORD


def chunk_bytes(n_layers: int, chunk_tokens: int, head_dim: int = mo.MLA_D, elem_bytes: int = 2,
                fmt: str = "raw") -> int:
    lat = latent_bytes(n_layers, chunk_tokens, head_dim, elem_bytes, fmt)
    return (lat + n_layers * chunk_tokens * IDX_TOKEN + 255) // 256 * 256


def token_bytes_of(plane: np.ndarray, slot: int) -> tuple[np.ndarray, np.ndarray]:
    """(values, scale bytes) of one token of an indexer plane (NB, bs, 132) uint8 — the per-token rule."""
    nb, bs, w = plane.shape
    blk = plane.reshape(nb, bs * w)[slot // bs]
    off = slot % bs
    return blk[off * IDX_VALUE:(off + 1) * IDX_VALUE], blk[bs * IDX_VALUE + off * IDX_SCALE:
                                                           bs * IDX_VALUE + (off + 1) * IDX_SCALE]


def gather_slabs(planes, slot_mapping, chunk_tokens: int) -> np.ndarray:
    """Indexer planes (L arrays (NB, bs, 132)) -> (L, C*132) slabs of one chunk holding tokens slot_mapping (<= C):
    [C][128] values then [C][4] scales; bytes of tokens past len(slot_mapping) are 0."""
    sm = np.asarray(slot_mapping, dtype=np.int64)
    C = chunk_tokens
    assert len(sm) <= C
    out = np.zeros((len(planes), C * IDX_TOKEN), dtype=np.uint8)
    for l, p in enumerate(planes):
        for t, s in enumerate(sm):
            v, sc = token_bytes_of(p, int(s))
            out[l, t * IDX_VALUE:(t + 1) * IDX_VALUE] = v
            out[l, C * IDX_VALUE + t * IDX_SCALE:C * IDX_VALUE + (t + 1) * IDX_SCALE] = sc
    return out


def scatter_slabs(planes, slabs: np.ndarray, slot_mapping, chunk_tokens: int) -> None:
    """Inverse of gather_slabs for the first len(slot_mapping) tokens, in place."""
    sm = np.asarray(slot_mapping, dtype=np.int64)
    C = chunk_tokens
    for l, p in enumerate(planes):
        for t, s in enumerate(sm):
            v, sc = token_bytes_of(p, int(s))
            v[:] = slabs[l, t * IDX_VALUE:(t + 1) * IDX_VALUE]
            sc[:] = slabs[l, C * IDX_VALUE + t * IDX_SCALE:C * IDX_VALUE + (t + 1) * IDX_SCALE]


def slab_tokens(slabs: np.ndarray, n: int, chunk_tokens: int) -> tuple[np.ndarray, np.ndarray]:
    """(L, C*132) slabs -> ((L, n, 128) values, (L, n, 4) scale bytes) of the first n tokens."""
    C = chunk_tokens
    return (slabs[:, :C * IDX_VALUE].reshape(-1, C, IDX_VALUE)[:, :n],
            slabs[:, C * IDX_VALUE:].reshape(-1, C, IDX_SCALE)[:, :n])


def split_chunk(buf: np.ndarray, n_layers: int, chunk_tokens: int, latent_token_bytes: int):
    """One chunk's bytes -> ((L, C, latent_token_bytes) latent slabs, (L, C*132) indexer slabs)."""
    lat = n_layers * chunk_tokens * latent_token_bytes
    return (buf[:lat].reshape(n_layers, chunk_tokens, latent_token_bytes),
            buf[lat:lat + n_layers * chunk_tokens * IDX_TOKEN].reshape(n_layers, chunk_tokens * IDX_TOKEN))


def pack_chunk(latent_layers, idx_planes, slot_mapping, chunk_tokens: int, fmt: str = "raw") -> np.ndarray:
    """The chunk of tokens slot_mapping (<= C) as the engine writes it, chunk_bytes long; bytes it does not write
    (tokens past len(slot_mapping), the rounding tail) are 0.  Latent part by tests/mla_oracle.py."""
    L, C, n = len(latent_layers), chunk_tokens, len(slot_mapping)
    lat = mo.gather_tokens(latent_layers, slot_mapping)                    # (L, 1, n, 1, D)
    if fmt == "fp8":
        rec = mo.fp8_pack_chunk(lat)                                        # (L, n, 656)
        tb = mo.MLA_RECORD
    else:
        rec = np.ascontiguousarray(lat.reshape(L, n, -1)).view(np.uint8).reshape(L, n, -1)
        tb = rec.shape[-1]
    out = np.zeros(chunk_bytes(L, C, tb if fmt == "raw" else mo.MLA_D, 1 if fmt == "raw" else 2, fmt), np.uint8)
    lat_view, idx_view = split_chunk(out, L, C, tb)
    lat_view[:, :n] = rec
    idx_view[:] = gather_slabs(idx_planes, slot_mapping, C)
    return out
