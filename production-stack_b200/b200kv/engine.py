"""Host-side engine: the Python face of libb200kv.so.

Mirrors the interface vLLM's vendored LMCache adapter drives (same names, argument meaning
and error behaviour) so the parity tests read like calls into the reference:

* ``KVEngine.store(tokens, mask, slot_mapping, offset)``      <- ``lmcache_engine.store(...)``
  (vllm/.../lmcache_integration/vllm_v1_adapter.py:1115-1123)
* ``KVEngine.retrieve(tokens, mask, slot_mapping) -> ret_mask`` <- ``lmcache_engine.retrieve(...)``
  (vllm_v1_adapter.py:882-889)
* ``KVPool.lookup_tokens(tokens)``                              <- ``lookup_client.lookup(...)``
  (vllm_v1_adapter.py:1187-1191)

``kvcaches`` is registered once (``register_kv_caches``, KVConnectorBase_V1 base.py:251) instead
of being passed on every call.  Nothing here computes on the CPU: the data path is the C ABI.
"""
from __future__ import annotations

import ctypes as C
import re
from dataclasses import dataclass

import numpy as np

from . import _lib
from ._lib import FMT_FP8, FMT_RAW, VARIANT_BULK, check, lib

DEFAULT_SEED = 0x6232303030304B56  # keys are namespaced further by KVGeometry.key_seed()
MLA_FP8_RECORD_BYTES = 656         # one (token, layer) of an MLA FP8 chunk (include/b200kv.h, B200KV_LAYOUT_MLA)
# DeepSeek-V3.2's indexer key cache: per token 128 e4m3 values then, after the block's values, one fp32 scale
# (vLLM's indexer_k_quant_and_cache; DeepseekV32IndexerCache has head_size 132)
INDEXER_VALUE_BYTES, INDEXER_SCALE_BYTES = 128, 4


def _as_i64(a) -> np.ndarray:
    arr = np.ascontiguousarray(np.asarray(a), dtype=np.int64)
    return arr


def _as_i32(a) -> np.ndarray:
    return np.ascontiguousarray(np.asarray(a), dtype=np.int32)


def _ptr(arr: np.ndarray, ctype):
    return arr.ctypes.data_as(C.POINTER(ctype))


def chunk_keys(tokens, chunk_tokens: int = 256, seed: int = DEFAULT_SEED,
               include_partial: bool = True) -> np.ndarray:
    """Prefix-chained XXH64 chunk keys (b200kv_chunk_keys)."""
    toks = _as_i32(tokens)
    n = len(toks)
    out = np.empty((n + chunk_tokens - 1) // chunk_tokens, dtype=np.uint64)
    cnt = C.c_int32(0)
    check(lib().b200kv_chunk_keys(_ptr(toks, C.c_int32), n, chunk_tokens, C.c_uint64(seed),
                                   1 if include_partial else 0, _ptr(out, C.c_uint64), C.byref(cnt)),
          "b200kv_chunk_keys")
    return out[:cnt.value]


def xxh64(data: bytes, seed: int = 0) -> int:
    buf = (C.c_char * len(data)).from_buffer_copy(data) if data else None
    return int(lib().b200kv_xxh64(C.cast(buf, C.c_void_p) if buf is not None else None, len(data),
                                  C.c_uint64(seed)))


# vLLM's 1-byte cache dtypes whose codes the Q4 kernels decode (vLLM allocates them as torch.uint8)
FP8_CACHE_DTYPES = {"fp8": _lib.DTYPE_E4M3, "fp8_e4m3": _lib.DTYPE_E4M3, "fp8_e5m2": _lib.DTYPE_E5M2}


def dtype_code(torch_dtype, cache_dtype: str | None = None) -> int | None:
    """torch dtype of a cache -> DTYPE_BF16 / DTYPE_FP16 / DTYPE_E4M3 / DTYPE_E5M2; None for every other type.
    vLLM allocates fp8 caches as torch.uint8, so for a uint8 tensor the fp8 flavour comes from vLLM's
    cache_config.cache_dtype (FP8_CACHE_DTYPES); without one, or for another 1-byte cache dtype, it is None."""
    name = str(torch_dtype)
    if name == "torch.uint8":
        return FP8_CACHE_DTYPES.get(str(cache_dtype)) if cache_dtype is not None else None
    return {"torch.bfloat16": _lib.DTYPE_BF16, "torch.float16": _lib.DTYPE_FP16,
            "torch.float8_e4m3fn": _lib.DTYPE_E4M3, "torch.float8_e5m2": _lib.DTYPE_E5M2}.get(name)


@dataclass(frozen=True)
class KVGeometry:
    """Model / cache geometry (LMCache's kv_shape = (L, 2, chunk, H, D),
    vllm_v1_adapter.py:471-477, plus vLLM's paged layout)."""
    n_layers: int
    n_kv_heads: int
    head_dim: int
    n_blocks: int
    block_tokens: int = 16
    chunk_tokens: int = 256
    elem_bytes: int = 2
    block_stride_bytes: int = 0   # 0 -> dense (block_tokens * H * D * elem)
    fmt: int = FMT_RAW
    layout: int = 0               # LAYOUT_NHD / LAYOUT_HND inside a block, or LAYOUT_MLA
    dtype: int = _lib.DTYPE_BF16  # element type of a 16-bit cache: DTYPE_BF16 or DTYPE_FP16 (b200kv_set_cache_dtype)
    # indexer planes of an MLA model with sparse attention (DeepSeek-V3.2; b200kv_set_indexer): bytes of a token's
    # values and of its scale in the split tile, and the planes' block stride (0 -> dense); 0 / 0 = none
    idx_value_bytes: int = 0
    idx_scale_bytes: int = 0
    idx_block_stride_bytes: int = 0
    # speculative decoding (MTP, EAGLE, EAGLE-3): how many of the n_layers are the drafter's, which vLLM puts in the
    # target's KV-cache group.  They are layers n_layers - draft_layers .. n_layers - 1, with the target's geometry.
    draft_layers: int = 0
    # fp8 type of a 1-byte cache (vLLM's --kv-cache-dtype fp8 / fp8_e4m3 / fp8_e5m2): DTYPE_E4M3 (the default, the
    # same value as DTYPE_BF16) or DTYPE_E5M2 (b200kv_set_cache_dtype)
    fp8_dtype: int = _lib.DTYPE_E4M3

    def __post_init__(self):
        if not 0 <= self.draft_layers < max(self.n_layers, 1):
            raise ValueError(f"{self.draft_layers} draft layers in a geometry of {self.n_layers} layers")

    @property
    def target_layers(self) -> int:
        """Layers of the target model: the engine's layers before the draft layers."""
        return self.n_layers - self.draft_layers

    @property
    def fp16(self) -> bool:
        return self.dtype == _lib.DTYPE_FP16

    @property
    def cache_dtype(self) -> int:
        """The element type the engine holds (b200kv_set_cache_dtype) and records in format tags and P/D documents:
        dtype on a 16-bit cache, fp8_dtype on a 1-byte one."""
        return self.fp8_dtype if self.elem_bytes == 1 and self.dtype == _lib.DTYPE_BF16 else self.dtype

    @property
    def e5m2(self) -> bool:
        return self.elem_bytes == 1 and self.cache_dtype == _lib.DTYPE_E5M2

    @property
    def dtype_name(self) -> str:
        if self.elem_bytes == 1:
            return "float8_e5m2" if self.e5m2 else "float8_e4m3fn"
        return "float16" if self.fp16 else "bfloat16"

    @property
    def fmt_tag(self) -> int:
        """The format tag the engine records with every chunk (pool_fmt in b200kv_engine.cu): format, tile order
        and cache element type, plus bit 24 with indexer planes.  bf16 tags are format | layout << 8, as before the
        element type was added."""
        return self.fmt | (self.layout << 8) | (self.cache_dtype << 16) | (_lib.FMT_TAG_INDEXED if self.indexed else 0)

    @property
    def token_bytes(self) -> int:
        return self.n_kv_heads * self.head_dim * self.elem_bytes

    @property
    def mla(self) -> bool:
        return self.layout == _lib.LAYOUT_MLA

    @property
    def indexed(self) -> bool:
        """An indexer plane per layer next to the latent one (MLA with sparse attention)."""
        return self.idx_value_bytes > 0

    @property
    def idx_token_bytes(self) -> int:
        return self.idx_value_bytes + self.idx_scale_bytes

    @property
    def idx_stride(self) -> int:
        return self.idx_block_stride_bytes or self.block_tokens * self.idx_token_bytes

    @property
    def planes(self) -> int:
        """Paged planes the engine moves: a K and a V plane per layer, or one latent plane (MLA)."""
        return self.n_layers * (1 if self.mla else 2)

    @property
    def n_descs(self) -> int:
        """IPC descriptors of the engine's cache (b200kv_export_ipc): one per paged plane and per indexer plane."""
        return self.planes + (self.n_layers if self.indexed else 0)

    @property
    def stride(self) -> int:
        return self.block_stride_bytes or self.block_tokens * self.token_bytes

    def key_seed(self, model: str = "", world_size: int = 1, rank: int = 0) -> int:
        """Namespace for chunk keys: same role as LMCache's CacheEngineKey(fmt, model, world_size,
        worker_id, ...) — chunks of different models / shards / formats never alias.  An MLA latent is
        the same on every tensor-parallel rank, so its namespace keeps only the pipeline stage
        (rank // world_size) of the rank: one stored copy serves every rank of the stage.  An fp16 cache
        appends "|fp16", so its chunks (RAW included) never alias a bf16 replica's; bf16 seeds are unchanged.  An
        e5m2 cache appends "|e5m2" likewise, and e4m3 seeds are unchanged.  A
        geometry with indexer planes appends "|idx<bytes per token>" (V3.2: "|idx132"); others are unchanged.
        Draft layers count in n_layers, so a speculative-decoding replica's chunks, which carry the drafter's planes,
        have a namespace of their own; a geometry without draft layers keeps its seed."""
        if self.mla:
            rank //= max(world_size, 1)
        tag = f"{model}|{world_size}|{rank}|{self.n_layers}|{self.n_kv_heads}|{self.head_dim}|" \
              f"{self.elem_bytes}|{self.chunk_tokens}|{self.fmt}|{self.layout}"
        if self.fp16:
            tag += "|fp16"
        if self.e5m2:
            tag += "|e5m2"
        if self.indexed:
            tag += f"|idx{self.idx_token_bytes}"
        return xxh64(tag.encode(), DEFAULT_SEED)

    def to_c(self, device: int, staging_bytes: int, owner: int, variant: int, stages: int,
             ctas_per_sm: int, numa_policy: int = 0) -> _lib.EngineConfig:
        return _lib.EngineConfig(device, self.n_layers, self.n_kv_heads, self.head_dim,
                                 self.elem_bytes, self.block_tokens, self.chunk_tokens, self.fmt,
                                 self.stride, self.n_blocks, staging_bytes, owner, variant, stages,
                                 ctas_per_sm, self.layout, numa_policy)

    @property
    def chunk_bytes(self) -> int:
        cfg = self.to_c(0, 0, 0, 0, 0, 0)
        if self.indexed:
            return check(int(lib().b200kv_engine_chunk_bytes_indexed(C.byref(cfg), self.idx_value_bytes,
                                                                      self.idx_scale_bytes)),
                         "b200kv_engine_chunk_bytes_indexed")
        return check(int(lib().b200kv_engine_chunk_bytes(C.byref(cfg))), "b200kv_engine_chunk_bytes")

    @property
    def payload_bytes_per_token(self) -> int:
        """Bytes one token occupies in a stored chunk (SURVEY.md §8d 'payload P')."""
        per = self.planes * self.token_bytes
        idx = self.n_layers * self.idx_token_bytes   # indexer planes travel verbatim in every format
        if self.fmt == FMT_RAW:
            return per + idx
        if self.fmt == FMT_FP8:
            return (self.n_layers * MLA_FP8_RECORD_BYTES + idx) if self.mla else per // 2
        return per * 9 // 32          # Q4: 4 bits + one bf16 scale per 32 elements = 4.5 bits per element


class KVPool:
    """Pinned-host chunk pool + index (CPU only; usable in the scheduler process)."""

    def __init__(self, name: str | None, pool_bytes: int = 0, slot_bytes: int = 0,
                 flags: int = _lib.POOL_CREATE_OR_ATTACH):
        self.name = name
        cfg = _lib.PoolConfig(name.encode() if name else None, pool_bytes, slot_bytes, flags, 0)
        h = C.c_void_p()
        check(lib().b200kv_pool_open(C.byref(cfg), C.byref(h)), f"b200kv_pool_open({name})")
        self._h = h

    @property
    def handle(self) -> C.c_void_p:
        if self._h is None:
            raise RuntimeError("pool is closed")
        return self._h

    def lookup(self, keys: np.ndarray, chunk_tokens: np.ndarray, lease_ms: int = 0) -> tuple[int, int]:
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        ct = _as_i32(chunk_tokens)
        hc, ht = C.c_int32(0), C.c_int64(0)
        check(lib().b200kv_pool_lookup(self.handle, _ptr(keys, C.c_uint64), _ptr(ct, C.c_int32),
                                        len(keys), lease_ms, C.byref(hc), C.byref(ht)),
              "b200kv_pool_lookup")
        return hc.value, ht.value

    def lookup_tokens(self, tokens, chunk_tokens: int, seed: int, lease_ms: int = 0,
                      include_partial: bool = True) -> int:
        """lookup_client.lookup(token_ids): tokens in the longest stored whole-chunk prefix."""
        toks = _as_i32(tokens)
        keys = chunk_keys(toks, chunk_tokens, seed, include_partial)
        if len(keys) == 0:
            return 0
        ct = np.minimum(chunk_tokens, len(toks) - np.arange(len(keys)) * chunk_tokens).astype(np.int32)
        return self.lookup(keys, ct, lease_ms)[1]

    def contains(self, keys, chunk_tokens=None, lease_ms: int = 0) -> np.ndarray:
        """Per-key membership (bool array), leasing what is present (b200kv_pool_contains)."""
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        out = np.zeros(len(keys), dtype=np.uint8)
        ct = None if chunk_tokens is None else np.ascontiguousarray(chunk_tokens, dtype=np.int32)
        check(lib().b200kv_pool_contains(self.handle, _ptr(keys, C.c_uint64), None if ct is None else _ptr(ct, C.c_int32),
                                         len(keys), lease_ms, out.ctypes.data_as(C.POINTER(C.c_uint8))),
              "b200kv_pool_contains")
        return out.astype(bool)

    def lookup_owner(self, keys: np.ndarray) -> tuple[int, np.ndarray]:
        keys = np.ascontiguousarray(keys, dtype=np.uint64)
        owners = np.zeros(len(keys), dtype=np.uint32)
        hc = C.c_int32(0)
        check(lib().b200kv_pool_lookup_owner(self.handle, _ptr(keys, C.c_uint64), len(keys),
                                              C.byref(hc), _ptr(owners, C.c_uint32)),
              "b200kv_pool_lookup_owner")
        return hc.value, owners[:hc.value]

    def reserve(self, key: int, n_tokens: int, fmt: int = FMT_RAW, owner: int = 0) -> int:
        slot = C.c_uint32(0)
        check(lib().b200kv_pool_reserve(self.handle, C.c_uint64(key), n_tokens, fmt, owner,
                                         C.byref(slot)), "b200kv_pool_reserve")
        return slot.value

    def commit(self, key: int):
        check(lib().b200kv_pool_commit(self.handle, C.c_uint64(key)), "b200kv_pool_commit")

    def abort(self, key: int):
        check(lib().b200kv_pool_abort(self.handle, C.c_uint64(key)), "b200kv_pool_abort")

    def acquire(self, key: int) -> tuple[int, int, int]:
        slot, n, fmt = C.c_uint32(0), C.c_int32(0), C.c_uint32(0)
        check(lib().b200kv_pool_acquire(self.handle, C.c_uint64(key), C.byref(slot), C.byref(n),
                                         C.byref(fmt)), "b200kv_pool_acquire")
        return slot.value, n.value, fmt.value

    def release(self, key: int):
        check(lib().b200kv_pool_release(self.handle, C.c_uint64(key)), "b200kv_pool_release")

    def slot_view(self, slot: int) -> np.ndarray:
        """uint8 view of one slot's payload (tests / CPU-side inspection)."""
        st = self.stats()
        p = lib().b200kv_pool_slot_ptr(self.handle, slot)
        if not p:
            raise IndexError(slot)
        return np.ctypeslib.as_array((C.c_uint8 * st["slot_bytes"]).from_address(p))

    def stats(self) -> dict:
        s = _lib.PoolStats()
        check(lib().b200kv_pool_get_stats(self.handle, C.byref(s)), "b200kv_pool_get_stats")
        return s.as_dict()

    def check(self) -> bool:
        """Index / LRU / free list consistent with the slot array (b200kv_pool_check)."""
        return lib().b200kv_pool_check(self.handle) == 0

    def clear(self) -> bool:
        rc = lib().b200kv_pool_clear(self.handle)
        if rc == _lib.EBUSY:
            return False
        check(rc, "b200kv_pool_clear")
        return True

    def close(self):
        if self._h is not None:
            lib().b200kv_pool_close(self._h)
            self._h = None

    @staticmethod
    def unlink(name: str):
        lib().b200kv_pool_unlink(name.encode())

    @staticmethod
    def sweep(prefix: str, min_age_s: int = 60) -> int:
        """Unlink the segments /dev/shm/<prefix>* that no live process holds (b200kv_pool_sweep)."""
        n = C.c_int32(0)
        check(lib().b200kv_pool_sweep(prefix.encode(), min_age_s, C.byref(n)), "b200kv_pool_sweep")
        return n.value

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass


DETACHED = "detached"   # stream value for asynchronous loads (B200KV_STREAM_DETACHED)


def _stream_ptr(stream) -> C.c_void_p:
    """torch.cuda.Stream | int | None(-> current torch stream) | DETACHED -> cudaStream_t."""
    if isinstance(stream, str) and stream == DETACHED:
        return C.c_void_p(2 ** 64 - 1)
    if stream is None:
        import torch
        stream = torch.cuda.current_stream()
    if hasattr(stream, "cuda_stream"):
        stream = stream.cuda_stream
    return C.c_void_p(int(stream))


def indexer_layout_of(t, block_tokens: int, token_bytes: int = INDEXER_VALUE_BYTES + INDEXER_SCALE_BYTES):
    """(ptr, block_stride_bytes, n_blocks) of one layer's indexer key cache: (NB, bs, 132) uint8 as vLLM's
    DeepseekV32IndexerBackend.get_kv_cache_shape allocates it, a block holding [bs][128] values then [bs][4] scales."""
    if t.dim() != 3 or t.element_size() != 1 or t.shape[1] != block_tokens or t.shape[2] != token_bytes:
        raise ValueError(f"indexer cache shape {tuple(t.shape)} / {t.dtype} is not (NB, {block_tokens}, {token_bytes}) bytes")
    if tuple(t.stride()[1:]) != (token_bytes, 1) or t.stride(0) < block_tokens * token_bytes:
        raise NotImplementedError("unsupported order inside an indexer block (strides %s)" % (tuple(t.stride()),))
    return t.data_ptr(), t.stride(0), t.shape[0]


def _layer_number(name: str):
    m = re.search(r"\.(\d+)\.", f".{name}.")
    return int(m.group(1)) if m else None


def split_indexer_caches(kv_caches, token_bytes: int = INDEXER_VALUE_BYTES + INDEXER_SCALE_BYTES):
    """kv_caches (dict name -> tensor, or a list) -> (latent tensors, indexer tensors), each in layer order.  vLLM
    puts a DeepSeek-V3.2's latent layers and its DeepseekV32IndexerCache layers in one KV-cache group, so
    register_kv_caches gets both.  An indexer cache is a rank-3 one-byte tensor of `token_bytes` per token (V3.2:
    132), which no latent cache is (576 elements, or 656 bytes with fp8_ds_mla).  With names, the split must
    also agree with them ("indexer" in a name), and the i-th latent and i-th indexer tensor must be the same
    layer.  Without any indexer tensor the second list is empty."""
    items = list(kv_caches.items()) if isinstance(kv_caches, dict) else [(None, t) for t in kv_caches]
    lat, idx = [], []
    for name, t in items:
        is_idx = t.dim() == 3 and t.element_size() == 1 and t.shape[-1] == token_bytes
        if name is not None and ("indexer" in name) != is_idx:
            raise ValueError(f"KV cache {name}: shape {tuple(t.shape)} / {t.dtype} contradicts its layer name")
        (idx if is_idx else lat).append((name, t))
    if idx:
        if len(idx) != len(lat):
            raise ValueError(f"{len(lat)} latent and {len(idx)} indexer caches: need one of each per layer")
        for (nl, _), (ni, _) in zip(lat, idx):
            if nl is not None and _layer_number(nl) != _layer_number(ni):
                raise ValueError(f"latent cache {nl} and indexer cache {ni} are not the same layer")
    return [t for _, t in lat], [t for _, t in idx]


def paged_layout_of(t, block_tokens: int, layout: str | None = None):
    """(k_ptr, v_ptr, block_stride_bytes, n_blocks, H, D, tile_layout) of one layer's paged KV tensor.
    FlashAttention (2, NB, bs, H, D) (vllm/v1/attention/backends/flash_attn.py:140-149) or
    FlashInfer (NB, 2, bs, H, D) (flashinfer.py:357-368); within a block the order must be NHD or HND.
    MLA (NB, bs, D) (MLACommonBackend.get_kv_cache_shape, model_executor/layers/attention/mla_attention.py):
    one latent plane, v_ptr None, H 1, LAYOUT_MLA."""
    es = t.element_size()
    if t.dim() == 3:
        nb, bs, d = t.shape
        if bs != block_tokens:
            raise ValueError(f"MLA KV cache shape {tuple(t.shape)} does not match block size {block_tokens}")
        if tuple(t.stride()[1:]) != (d, 1) or t.stride(0) < bs * d:
            raise NotImplementedError("unsupported order inside an MLA KV block (strides %s)" % (tuple(t.stride()),))
        return t.data_ptr(), None, t.stride(0) * es, nb, 1, d, _lib.LAYOUT_MLA
    if t.dim() != 5:
        raise NotImplementedError(f"unsupported KV cache rank {t.dim()} (packed layouts)")
    if layout is None:
        layout = "fa" if (t.shape[0] == 2 and t.shape[2] == block_tokens) else "fi"
    if layout == "fa":
        two, nb, bs, h, d = t.shape
        kv_stride, blk_stride = t.stride(0) * es, t.stride(1) * es
    else:
        nb, two, bs, h, d = t.shape
        blk_stride, kv_stride = t.stride(0) * es, t.stride(1) * es
    if two != 2 or bs != block_tokens:
        raise ValueError(f"KV cache shape {tuple(t.shape)} does not match block size {block_tokens}")
    inner = tuple(t.stride()[2:])
    if inner == (h * d, d, 1):
        tile_layout = _lib.LAYOUT_NHD
    elif inner == (d, bs * d, 1):
        tile_layout = _lib.LAYOUT_HND      # what vLLM's FlashInfer backend uses
    else:
        raise NotImplementedError("unsupported order inside a KV block (strides %s)" % (tuple(t.stride()),))
    return t.data_ptr(), t.data_ptr() + kv_stride, blk_stride, nb, h, d, tile_layout


class KVEngine:
    """Per-GPU engine (CUDA).  Raises B200KVError(-ENODEV) without a GPU, -ENOTSUP on one other than an H100 (sm_90)."""

    def __init__(self, geom: KVGeometry, pool: KVPool | None, device: int = 0,
                 staging_bytes: int = 1 << 30, owner: int = 0, variant: int = VARIANT_BULK,
                 stages: int = 0, ctas_per_sm: int = 0, key_seed: int | None = None,
                 numa_policy: int = _lib.NUMA_LOCAL):
        self.geom = geom
        self.pool = pool
        self.device = device
        self.key_seed = geom.key_seed() if key_seed is None else key_seed
        cfg = geom.to_c(device, staging_bytes, owner, variant, stages, ctas_per_sm, numa_policy)
        h = C.c_void_p()
        check(lib().b200kv_engine_create(C.byref(cfg), pool.handle if pool else None, C.byref(h)),
              "b200kv_engine_create")
        self._h = h
        self._kv_refs = None
        if geom.dtype != _lib.DTYPE_BF16:
            self.set_cache_dtype(geom.dtype)
        if geom.fp8_dtype != _lib.DTYPE_E4M3:
            self.set_cache_dtype(geom.fp8_dtype)    # -EINVAL unless the cache is 1-byte
        if geom.indexed:
            self.set_indexer(geom.idx_value_bytes, geom.idx_scale_bytes, geom.idx_stride)

    def set_cache_dtype(self, dtype: int):
        """b200kv_set_cache_dtype: legal before registration only (-EBUSY after)."""
        check(lib().b200kv_set_cache_dtype(self._h, dtype), "b200kv_set_cache_dtype")

    def set_indexer(self, value_bytes: int, scale_bytes: int, block_stride: int):
        """b200kv_set_indexer: an indexer plane per layer on an MLA engine; before registration only (-EBUSY after)."""
        check(lib().b200kv_set_indexer(self._h, value_bytes, scale_bytes, C.c_uint64(block_stride)),
              "b200kv_set_indexer")

    # ---- registration ---------------------------------------------------------------------
    def _plane_ptrs(self, k_ptrs, v_ptrs):
        """ctypes arrays of the K and V pointers; MLA takes one latent pointer per layer and v_ptrs None, or the
        indexer planes in v_ptrs when the geometry has them."""
        L = self.geom.n_layers
        if self.geom.mla and not self.geom.indexed:
            if len(k_ptrs) != L or v_ptrs is not None:
                raise ValueError("MLA: need one latent pointer per layer and no V pointers")
            return (C.c_void_p * L)(*[C.c_void_p(int(p)) for p in k_ptrs]), None
        if len(k_ptrs) != L or v_ptrs is None or len(v_ptrs) != L:
            raise ValueError("need one latent and one indexer pointer per layer" if self.geom.mla
                             else "need one K and one V pointer per layer")
        return ((C.c_void_p * L)(*[C.c_void_p(int(p)) for p in k_ptrs]),
                (C.c_void_p * L)(*[C.c_void_p(int(p)) for p in v_ptrs]))

    def register_kv_ptrs(self, k_ptrs, v_ptrs):
        ka, va = self._plane_ptrs(k_ptrs, v_ptrs)
        check(lib().b200kv_register_kv(self._h, ka, va), "b200kv_register_kv")

    def register_kv_caches(self, kv_caches, layout: str | None = None):
        """kv_caches: list (or dict) of per-layer torch tensors on this device.  With indexer planes, the latent and
        indexer caches of every layer (split_indexer_caches tells them apart)."""
        tensors = list(kv_caches.values()) if isinstance(kv_caches, dict) else list(kv_caches)
        # v_ptrs: the V planes, the indexer planes, or None (plain MLA); include/b200kv.h, "Planes and descriptors"
        lat, k_ptrs, v_ptrs = tensors, [], (None if self.geom.mla else [])
        if self.geom.indexed:
            lat, idx = split_indexer_caches(kv_caches, self.geom.idx_token_bytes)
            if not idx:
                raise ValueError("the engine has indexer planes but no indexer cache was given")
            v_ptrs = []
            for t in idx:
                ptr, stride, nb = indexer_layout_of(t, self.geom.block_tokens, self.geom.idx_token_bytes)
                if stride != self.geom.idx_stride or nb < self.geom.n_blocks:
                    raise ValueError("indexer cache tensor does not match the engine geometry")
                v_ptrs.append(ptr)
        for t in lat:
            k, v, stride, nb, h, d, tl = paged_layout_of(t, self.geom.block_tokens, layout)
            if stride != self.geom.stride or h != self.geom.n_kv_heads or d != self.geom.head_dim \
                    or nb < self.geom.n_blocks or t.element_size() != self.geom.elem_bytes \
                    or tl != self.geom.layout:
                raise ValueError("KV cache tensor does not match the engine geometry")
            code = dtype_code(t.dtype)
            if self.geom.fmt != FMT_RAW and code != self.geom.cache_dtype and not (code is None and str(t.dtype) == "torch.uint8"):
                # the lossy kernels decode the elements: fp16 bits read as bf16 (or the reverse) would be stored
                # and loaded as wrong values without any error.  A uint8 tensor (how vLLM allocates fp8 caches)
                # does not say which fp8 type it holds: the geometry does.
                raise ValueError(f"KV cache dtype {t.dtype} does not match the engine's cache dtype "
                                 f"({self.geom.dtype_name})")
            k_ptrs.append(k)
            if not self.geom.mla:
                v_ptrs.append(v)
        self._kv_refs = tensors   # keep the storage of every registered tensor alive
        self.register_kv_ptrs(k_ptrs, v_ptrs)

    # ---- LMCache-shaped data path ---------------------------------------------------------
    def _keys(self, tokens) -> np.ndarray:
        return chunk_keys(tokens, self.geom.chunk_tokens, self.key_seed, True)

    def store(self, tokens, mask=None, slot_mapping=None, offset: int = 0, stream=None,
              keys: np.ndarray | None = None) -> int:
        """Store tokens[offset:] (offset is chunk aligned, mask False exactly on [0, offset)).
        Returns a ticket (0 = nothing to do).  Failed / skipped chunks are future misses, never
        exceptions on the data path beyond argument errors."""
        C_ = self.geom.chunk_tokens
        n = len(tokens)
        if offset % C_:
            raise ValueError("offset must be chunk aligned (adapter :1084-1088)")
        if mask is not None and int(np.count_nonzero(~np.asarray(mask, dtype=bool))) != offset:
            raise ValueError("mask must be False exactly on the first `offset` tokens")
        if n <= offset:
            return 0
        sm = _as_i64(slot_mapping)
        if len(sm) != n:
            raise ValueError("slot_mapping and tokens differ in length")
        keys = self._keys(tokens) if keys is None else np.ascontiguousarray(keys, dtype=np.uint64)
        c0 = offset // C_
        sub_keys = np.ascontiguousarray(keys[c0:])
        sub_sm = np.ascontiguousarray(sm[offset:])
        ticket = C.c_uint64(0)
        check(lib().b200kv_store_async(self._h, _ptr(sub_keys, C.c_uint64), len(sub_keys),
                                        _ptr(sub_sm, C.c_int64), n - offset, _stream_ptr(stream),
                                        C.byref(ticket)), "b200kv_store_async")
        return ticket.value

    def retrieve(self, tokens, mask=None, slot_mapping=None, stream=None,
                 keys: np.ndarray | None = None, return_ticket: bool = False, layers_per_group: int = 0):
        """Load every stored chunk after the masked chunk-aligned prefix until the first miss;
        returns the bool mask of tokens that were scheduled to be written (ret_token_mask)."""
        C_ = self.geom.chunk_tokens
        n = len(tokens)
        skip = 0 if mask is None else int(np.count_nonzero(~np.asarray(mask, dtype=bool)))
        if skip % C_:
            raise ValueError("masked prefix must be chunk aligned (adapter :848-854)")
        ret = np.zeros(n, dtype=bool)
        if n == 0:
            return (ret, 0) if return_ticket else ret
        sm = _as_i64(slot_mapping)
        if len(sm) != n:
            raise ValueError("slot_mapping and tokens differ in length")
        keys = self._keys(tokens) if keys is None else np.ascontiguousarray(keys, dtype=np.uint64)
        ticket, loaded = C.c_uint64(0), C.c_int64(0)
        if layers_per_group > 0:   # lmcache_engine.retrieve_layer: the caller then waits per layer (wait_layer)
            check(lib().b200kv_load_layerwise_async(self._h, _ptr(keys, C.c_uint64), len(keys), _ptr(sm, C.c_int64), n,
                                                     skip // C_, layers_per_group, _stream_ptr(stream),
                                                     C.byref(ticket), C.byref(loaded)), "b200kv_load_layerwise_async")
        else:
            check(lib().b200kv_load_async(self._h, _ptr(keys, C.c_uint64), len(keys),
                                           _ptr(sm, C.c_int64), n, skip // C_, _stream_ptr(stream),
                                           C.byref(ticket), C.byref(loaded)), "b200kv_load_async")
        ret[skip:skip + loaded.value] = True
        return (ret, ticket.value) if return_ticket else ret

    # ---- one engine step in one op (b200kv_store_batch_async / b200kv_load_batch_async) -------------------
    def _batch_layout(self, reqs):
        """reqs: [(tokens, slot_mapping, first_chunk)] — chunks [first_chunk, ...) of each request take part.
        -> (keys, chunk_tokens, req_first_chunk, padded slot mapping): requests back to back, every request's
        last chunk padded to C entries."""
        C_ = self.geom.chunk_tokens
        keys, ct, first, sms = [], [], [0], []
        for tokens, sm, c0 in reqs:
            n = len(tokens)
            k = self._keys(tokens)[c0:]
            sm = _as_i64(sm)
            if len(sm) != n:
                raise ValueError("slot_mapping and tokens differ in length")
            part = sm[c0 * C_:]
            pad = len(k) * C_ - len(part)
            sms.append(part if pad == 0 else np.concatenate([part, np.full(pad, -1, dtype=np.int64)]))
            keys.append(k)
            ct.append(np.minimum(C_, n - (c0 + np.arange(len(k))) * C_).astype(np.int32))
            first.append(first[-1] + len(k))
        return (np.ascontiguousarray(np.concatenate(keys), dtype=np.uint64), np.ascontiguousarray(np.concatenate(ct)),
                np.asarray(first, dtype=np.int32), np.ascontiguousarray(np.concatenate(sms)))

    def store_batch(self, reqs, stream=None) -> int:
        """reqs: [(tokens, slot_mapping, offset)] with chunk-aligned offsets (tokens[offset:] are stored).  One
        ticket for all of them; 0 if nothing was to do."""
        C_ = self.geom.chunk_tokens
        todo = []
        for tokens, sm, offset in reqs:
            if offset % C_:
                raise ValueError("offset must be chunk aligned (adapter :1084-1088)")
            if len(tokens) > offset:
                todo.append((tokens, sm, offset // C_))
        if not todo:
            return 0
        keys, ct, _first, sm = self._batch_layout(todo)
        ticket = C.c_uint64(0)
        check(lib().b200kv_store_batch_async(self._h, _ptr(keys, C.c_uint64), _ptr(ct, C.c_int32), len(keys),
                                              _ptr(sm, C.c_int64), _stream_ptr(stream), C.byref(ticket)),
              "b200kv_store_batch_async")
        return ticket.value

    def retrieve_batch(self, reqs, stream=None, layers_per_group: int = 0):
        """reqs: [(tokens, slot_mapping, masked_tokens)] with chunk-aligned masked prefixes.  -> (tokens loaded
        per request (after its masked prefix), ticket)."""
        C_ = self.geom.chunk_tokens
        todo = []
        for tokens, sm, skip in reqs:
            if skip % C_:
                raise ValueError("masked prefix must be chunk aligned (adapter :848-854)")
            todo.append((tokens, sm, skip // C_))
        loaded = np.zeros(len(todo), dtype=np.int64)
        live = [i for i, (tokens, _, c0) in enumerate(todo) if len(tokens) > c0 * C_]
        if not live:
            return loaded, 0
        keys, ct, first, sm = self._batch_layout([todo[i] for i in live])
        got = np.zeros(len(live), dtype=np.int64)
        ticket = C.c_uint64(0)
        check(lib().b200kv_load_batch_async(self._h, _ptr(keys, C.c_uint64), _ptr(ct, C.c_int32), len(keys),
                                             _ptr(first, C.c_int32), len(live), _ptr(sm, C.c_int64), layers_per_group,
                                             _stream_ptr(stream), C.byref(ticket), _ptr(got, C.c_int64)),
              "b200kv_load_batch_async")
        loaded[live] = got
        return loaded, ticket.value

    def lookup(self, tokens, lease_ms: int = 0) -> int:
        if self.pool is None:
            return 0
        return self.pool.lookup_tokens(tokens, self.geom.chunk_tokens, self.key_seed, lease_ms)

    # ---- device-resident halves -----------------------------------------------------------
    def gather(self, slot_mapping, dev_chunks_ptr: int, stream=None):
        sm = _as_i64(slot_mapping)
        check(lib().b200kv_gather(self._h, _ptr(sm, C.c_int64), len(sm), C.c_void_p(dev_chunks_ptr),
                                   _stream_ptr(stream)), "b200kv_gather")

    def scatter(self, slot_mapping, dev_chunks_ptr: int, stream=None):
        sm = _as_i64(slot_mapping)
        check(lib().b200kv_scatter(self._h, _ptr(sm, C.c_int64), len(sm), C.c_void_p(dev_chunks_ptr),
                                    _stream_ptr(stream)), "b200kv_scatter")

    # ---- peers ----------------------------------------------------------------------------
    # ---- device chunk tier --------------------------------------------------------------------
    def tier_create(self, n_slots: int) -> int:
        base = C.c_uint64(0)
        check(lib().b200kv_tier_create(self._h, n_slots, C.byref(base)), "b200kv_tier_create")
        return base.value

    def tier_export(self) -> bytes:
        d = _lib.IpcDesc()
        check(lib().b200kv_tier_export(self._h, C.byref(d)), "b200kv_tier_export")
        return bytes(d)

    def tier_import(self, desc: bytes) -> int:
        d = _lib.IpcDesc.from_buffer_copy(desc)
        base = C.c_uint64(0)
        check(lib().b200kv_tier_import(self._h, C.byref(d), C.byref(base)), "b200kv_tier_import")
        return base.value

    def gather_chunks(self, slot_mapping, chunk_ptrs, stream=None):
        sm = _as_i64(slot_mapping)
        ptrs = np.ascontiguousarray(chunk_ptrs, dtype=np.uint64)
        check(lib().b200kv_gather_chunks(self._h, _ptr(sm, C.c_int64), len(sm), _ptr(ptrs, C.c_uint64),
                                         _stream_ptr(stream)), "b200kv_gather_chunks")

    def scatter_chunks(self, slot_mapping, chunk_ptrs, stream=None):
        sm = _as_i64(slot_mapping)
        ptrs = np.ascontiguousarray(chunk_ptrs, dtype=np.uint64)
        check(lib().b200kv_scatter_chunks(self._h, _ptr(sm, C.c_int64), len(sm), _ptr(ptrs, C.c_uint64),
                                          _stream_ptr(stream)), "b200kv_scatter_chunks")

    def export_ipc(self) -> bytes:
        n = self.geom.n_descs
        arr = (_lib.IpcDesc * n)()
        check(lib().b200kv_export_ipc(self._h, arr, n), "b200kv_export_ipc")
        return bytes(arr)

    def import_peer(self, peer_id: int, peer_device: int, descs: bytes,
                    peer_block_stride: int | None = None, peer_n_blocks: int | None = None, head_slice=None):
        """Map a peer's cache (b200kv_import_peer).  head_slice = (peer_heads, src_head0, dst_head0, n_heads): a peer
        of another tensor-parallel size, of which pulls move those heads only (b200kv_import_peer_sliced)."""
        n = self.geom.n_descs
        arr = (_lib.IpcDesc * n).from_buffer_copy(descs)
        stride, nb = peer_block_stride or self.geom.stride, peer_n_blocks or self.geom.n_blocks
        if head_slice is None:
            check(lib().b200kv_import_peer(self._h, peer_id, peer_device, arr, n, stride, nb), "b200kv_import_peer")
        else:
            check(lib().b200kv_import_peer_sliced(self._h, peer_id, peer_device, arr, n, stride, nb,
                                                   C.byref(_lib.HeadSlice(*head_slice))), "b200kv_import_peer_sliced")

    def import_peer_ptrs(self, peer_id: int, peer_device: int, k_ptrs, v_ptrs,
                         peer_block_stride: int | None = None, peer_n_blocks: int | None = None, head_slice=None):
        ka, va = self._plane_ptrs(k_ptrs, v_ptrs)
        stride, nb = peer_block_stride or self.geom.stride, peer_n_blocks or self.geom.n_blocks
        if head_slice is None:
            check(lib().b200kv_import_peer_ptrs(self._h, peer_id, peer_device, ka, va, stride, nb),
                  "b200kv_import_peer_ptrs")
        else:
            check(lib().b200kv_import_peer_ptrs_sliced(self._h, peer_id, peer_device, ka, va, stride, nb,
                                                        C.byref(_lib.HeadSlice(*head_slice))),
                  "b200kv_import_peer_ptrs_sliced")

    def peer_pull(self, peer_id: int, src_slots, dst_slots, stream=None) -> int:
        s, d = _as_i64(src_slots), _as_i64(dst_slots)
        if len(s) != len(d):
            raise ValueError("src_slots and dst_slots differ in length")
        ticket = C.c_uint64(0)
        check(lib().b200kv_peer_pull_async(self._h, peer_id, _ptr(s, C.c_int64), _ptr(d, C.c_int64),
                                            len(s), _stream_ptr(stream), C.byref(ticket)),
              "b200kv_peer_pull_async")
        return ticket.value

    # ---- completion / stats ---------------------------------------------------------------
    def poll(self, ticket: int) -> bool:
        done = C.c_int(0)
        check(lib().b200kv_poll(self._h, C.c_uint64(ticket), C.byref(done)), "b200kv_poll")
        return bool(done.value)

    def wait(self, ticket: int):
        check(lib().b200kv_wait(self._h, C.c_uint64(ticket)), "b200kv_wait")

    def wait_layer(self, ticket: int, layer: int, stream=None):
        """Make `stream` wait until layer `layer` of a layer-wise retrieve is in the pages."""
        check(lib().b200kv_wait_layer(self._h, C.c_uint64(ticket), layer, _stream_ptr(stream)), "b200kv_wait_layer")

    def wait_all(self):
        check(lib().b200kv_wait_all(self._h), "b200kv_wait_all")

    def stats(self) -> dict:
        s = _lib.EngineStats()
        check(lib().b200kv_engine_get_stats(self._h, C.byref(s)), "b200kv_engine_get_stats")
        return s.as_dict()

    def numa_placement(self) -> str:
        """Where the pool's host pages were put when this engine pinned them (text, for logs)."""
        buf = C.create_string_buffer(160)
        check(lib().b200kv_engine_numa_placement(self._h, buf, len(buf)), "b200kv_engine_numa_placement")
        return buf.value.decode()

    def last_kernel_ms(self, which: int) -> float:
        ms = C.c_float(0)
        check(lib().b200kv_last_kernel_ms(self._h, which, C.byref(ms)), "b200kv_last_kernel_ms")
        return ms.value

    def close(self):
        if self._h is not None:
            lib().b200kv_engine_destroy(self._h)
            self._h = None
            self._kv_refs = None

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass
