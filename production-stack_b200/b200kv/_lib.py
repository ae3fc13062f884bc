"""ctypes binding of libb200kv.so (include/b200kv.h).

The library is built in-tree by ``__graft_entry__.build()`` /
``production-stack_b200/csrc/Makefile``.  There is no Python or CPU fallback: if the shared
object is missing this module raises at import of the first symbol.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libb200kv.so")

FMT_RAW, FMT_FP8, FMT_Q4 = 0, 1, 2   # FMT_Q4: experimental (group-wise 4-bit)
VARIANT_BULK, VARIANT_LDG = 0, 1
LAYOUT_NHD, LAYOUT_HND, LAYOUT_MLA = 0, 1, 2   # LAYOUT_MLA: one latent plane per layer (DeepSeek-V2/V3, Kimi-K2)
DTYPE_BF16, DTYPE_FP16 = 0, 1                  # element type of the cache (b200kv_set_cache_dtype)
DTYPE_E4M3, DTYPE_E5M2 = 0, 2                  # ... of a 1-byte (fp8) cache: e4m3 is the default, value 0 as bf16
FMT_TAG_INDEXED = 1 << 24                      # format-tag bit of chunks with indexer planes (b200kv_set_indexer)
POOL_CREATE, POOL_ATTACH, POOL_CREATE_OR_ATTACH = 1, 2, 3
NUMA_LOCAL, NUMA_INTERLEAVE, NUMA_OFF = 0, 1, 2

OK, EINVAL, ENOMEM, ENODEV, ENOENT, EEXIST, ENOSPC, ENOTSUP, EBUSY = 0, -22, -12, -19, -2, -17, -28, -95, -16
EIO = -5


class PoolConfig(C.Structure):
    _fields_ = [("shm_name", C.c_char_p), ("pool_bytes", C.c_uint64), ("slot_bytes", C.c_uint64),
                ("flags", C.c_uint32), ("reserved", C.c_uint32)]


class PoolStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "n_slots", "n_used", "slot_bytes", "n_lookups", "n_lookup_chunks", "n_hit_chunks",
        "n_hit_tokens", "n_requested_tokens", "n_stored_chunks", "n_evicted_chunks",
        "n_dropped_chunks", "n_reclaimed_chunks", "n_recoveries")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class DiskStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "n_slots", "n_used", "slot_bytes", "n_put", "n_get", "n_get_miss", "n_corrupt", "n_evicted", "n_dropped",
        "bytes_written", "bytes_read", "hash_ns", "copy_ns", "io_ns", "n_restored")] + [
        ("direct_io", C.c_int32), ("last_errno", C.c_int32)]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class EngineConfig(C.Structure):
    _fields_ = [("device", C.c_int32), ("n_layers", C.c_int32), ("n_kv_heads", C.c_int32),
                ("head_dim", C.c_int32), ("elem_bytes", C.c_int32), ("block_tokens", C.c_int32),
                ("chunk_tokens", C.c_int32), ("format", C.c_int32),
                ("block_stride_bytes", C.c_uint64), ("n_blocks", C.c_uint64),
                ("staging_bytes", C.c_uint64), ("owner", C.c_uint32), ("variant", C.c_int32),
                ("stages", C.c_int32), ("ctas_per_sm", C.c_int32), ("kv_layout", C.c_int32),
                ("numa_policy", C.c_int32)]


class EngineStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "n_store_ops", "n_load_ops", "n_pull_ops", "n_stored_tokens", "n_loaded_tokens",
        "n_pulled_tokens", "n_kernel_launches", "h2d_bytes", "d2h_bytes", "p2p_bytes")]

    def as_dict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class IpcDesc(C.Structure):
    _fields_ = [("handle", C.c_uint8 * 64), ("offset", C.c_uint64), ("alloc_bytes", C.c_uint64)]


class HeadSlice(C.Structure):
    """b200kv_head_slice: heads [src_head0, src_head0 + n_heads) of a peer with peer_heads heads per token are this
    engine's heads [dst_head0, dst_head0 + n_heads)."""
    _fields_ = [("peer_heads", C.c_int32), ("src_head0", C.c_int32), ("dst_head0", C.c_int32), ("n_heads", C.c_int32)]


_P = C.c_void_p
_U64P = C.POINTER(C.c_uint64)
_I64P = C.POINTER(C.c_int64)
_I32P = C.POINTER(C.c_int32)
_U32P = C.POINTER(C.c_uint32)

# name -> (restype, argtypes); the list is also what tests/test_abi.py checks against the header
SIGNATURES = {
    "b200kv_abi_version": (C.c_int, []),
    "b200kv_strerror": (C.c_char_p, [C.c_int]),
    "b200kv_last_error": (C.c_char_p, []),
    "b200kv_xxh64": (C.c_uint64, [_P, C.c_size_t, C.c_uint64]),
    "b200kv_chunk_keys": (C.c_int, [_I32P, C.c_int64, C.c_int32, C.c_uint64, C.c_int, _U64P, _I32P]),
    "b200kv_pool_open": (C.c_int, [C.POINTER(PoolConfig), C.POINTER(_P)]),
    "b200kv_pool_close": (C.c_int, [_P]),
    "b200kv_pool_unlink": (C.c_int, [C.c_char_p]),
    "b200kv_pool_sweep": (C.c_int, [C.c_char_p, C.c_int32, _I32P]),
    "b200kv_pool_region": (C.c_int, [_P, C.POINTER(_P), _U64P]),
    "b200kv_pool_slot_ptr": (_P, [_P, C.c_uint32]),
    "b200kv_pool_lookup": (C.c_int, [_P, _U64P, _I32P, C.c_int32, C.c_uint32, _I32P, _I64P]),
    "b200kv_pool_contains": (C.c_int, [_P, _U64P, _I32P, C.c_int32, C.c_uint32, C.POINTER(C.c_uint8)]),
    "b200kv_pool_lookup_owner": (C.c_int, [_P, _U64P, C.c_int32, _I32P, _U32P]),
    "b200kv_pool_reserve": (C.c_int, [_P, C.c_uint64, C.c_int32, C.c_uint32, C.c_uint32, _U32P]),
    "b200kv_pool_commit": (C.c_int, [_P, C.c_uint64]),
    "b200kv_pool_abort": (C.c_int, [_P, C.c_uint64]),
    "b200kv_pool_acquire": (C.c_int, [_P, C.c_uint64, _U32P, _I32P, _U32P]),
    "b200kv_pool_release": (C.c_int, [_P, C.c_uint64]),
    "b200kv_pool_get_stats": (C.c_int, [_P, C.POINTER(PoolStats)]),
    "b200kv_pool_clear": (C.c_int, [_P]),
    "b200kv_pool_check": (C.c_int, [_P]),
    "b200kv_pool_place": (C.c_int, [_P, _U32P, _U64P, _I32P, _U32P, _U32P, C.c_int32]),
    "b200kv_pool_drop": (C.c_int, [_P, C.c_uint64]),
    "b200kv_engine_create": (C.c_int, [C.POINTER(EngineConfig), _P, C.POINTER(_P)]),
    "b200kv_engine_destroy": (C.c_int, [_P]),
    "b200kv_set_cache_dtype": (C.c_int, [_P, C.c_int32]),
    "b200kv_set_indexer": (C.c_int, [_P, C.c_int32, C.c_int32, C.c_uint64]),
    "b200kv_engine_numa_placement": (C.c_int, [_P, C.c_char_p, C.c_uint64]),
    "b200kv_engine_chunk_bytes": (C.c_int64, [C.POINTER(EngineConfig)]),
    "b200kv_engine_chunk_bytes_indexed": (C.c_int64, [C.POINTER(EngineConfig), C.c_int32, C.c_int32]),
    "b200kv_register_kv": (C.c_int, [_P, C.POINTER(_P), C.POINTER(_P)]),
    "b200kv_store_async": (C.c_int, [_P, _U64P, C.c_int32, _I64P, C.c_int64, _P, _U64P]),
    "b200kv_load_async": (C.c_int, [_P, _U64P, C.c_int32, _I64P, C.c_int64, C.c_int32, _P, _U64P, _I64P]),
    "b200kv_load_layerwise_async": (C.c_int, [_P, _U64P, C.c_int32, _I64P, C.c_int64, C.c_int32, C.c_int32, _P, _U64P, _I64P]),
    "b200kv_wait_layer": (C.c_int, [_P, C.c_uint64, C.c_int32, _P]),
    "b200kv_store_batch_async": (C.c_int, [_P, _U64P, _I32P, C.c_int32, _I64P, _P, _U64P]),
    "b200kv_load_batch_async": (C.c_int, [_P, _U64P, _I32P, C.c_int32, _I32P, C.c_int32, _I64P, C.c_int32, _P, _U64P, _I64P]),
    "b200kv_poll": (C.c_int, [_P, C.c_uint64, C.POINTER(C.c_int)]),
    "b200kv_wait": (C.c_int, [_P, C.c_uint64]),
    "b200kv_wait_all": (C.c_int, [_P]),
    "b200kv_gather": (C.c_int, [_P, _I64P, C.c_int64, _P, _P]),
    "b200kv_scatter": (C.c_int, [_P, _I64P, C.c_int64, _P, _P]),
    "b200kv_export_ipc": (C.c_int, [_P, C.POINTER(IpcDesc), C.c_int32]),
    "b200kv_import_peer": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(IpcDesc), C.c_int32, C.c_uint64, C.c_uint64]),
    "b200kv_import_peer_ptrs": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(_P), C.POINTER(_P), C.c_uint64, C.c_uint64]),
    "b200kv_import_peer_sliced": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(IpcDesc), C.c_int32, C.c_uint64,
                                            C.c_uint64, C.POINTER(HeadSlice)]),
    "b200kv_import_peer_ptrs_sliced": (C.c_int, [_P, C.c_int32, C.c_int32, C.POINTER(_P), C.POINTER(_P), C.c_uint64,
                                                 C.c_uint64, C.POINTER(HeadSlice)]),
    "b200kv_peer_pull_async": (C.c_int, [_P, C.c_int32, _I64P, _I64P, C.c_int64, _P, _U64P]),
    "b200kv_gather_chunks": (C.c_int, [_P, _I64P, C.c_int64, _U64P, _P]),
    "b200kv_scatter_chunks": (C.c_int, [_P, _I64P, C.c_int64, _U64P, _P]),
    "b200kv_tier_create": (C.c_int, [_P, C.c_uint32, _U64P]),
    "b200kv_tier_export": (C.c_int, [_P, C.POINTER(IpcDesc)]),
    "b200kv_tier_import": (C.c_int, [_P, C.POINTER(IpcDesc), _U64P]),
    "b200kv_engine_get_stats": (C.c_int, [_P, C.POINTER(EngineStats)]),
    "b200kv_last_kernel_ms": (C.c_int, [_P, C.c_int, C.POINTER(C.c_float)]),
    "b200kv_server_start": (C.c_int, [C.c_char_p, C.c_int, C.c_uint64, C.POINTER(_P)]),
    "b200kv_server_port": (C.c_int, [_P]),
    "b200kv_server_get_stats": (C.c_int, [_P, _U64P]),
    "b200kv_server_stop": (C.c_int, [_P]),
    "b200kv_remote_connect": (C.c_int, [C.c_char_p, C.c_int, C.c_int, C.POINTER(_P)]),
    "b200kv_remote_close": (C.c_int, [_P]),
    "b200kv_remote_ping": (C.c_int, [_P]),
    "b200kv_remote_exists": (C.c_int, [_P, _U64P, C.c_int32, _I32P]),
    "b200kv_remote_put": (C.c_int, [_P, _P, C.c_uint64, C.c_uint32]),
    "b200kv_remote_get": (C.c_int, [_P, _P, C.c_uint64, C.c_uint32]),
    "b200kv_remote_stats": (C.c_int, [_P, C.POINTER(PoolStats)]),
    "b200kv_remote_traffic": (C.c_int, [_P, _U64P, _U64P]),
    "b200kv_disk_open": (C.c_int, [C.c_char_p, C.c_uint64, C.c_uint64, C.POINTER(_P)]),
    "b200kv_disk_close": (C.c_int, [_P]),
    "b200kv_disk_put": (C.c_int, [_P, _P, C.c_uint64, C.c_uint32]),
    "b200kv_disk_get": (C.c_int, [_P, _P, C.c_uint64]),
    "b200kv_disk_lookup": (C.c_int, [_P, _U64P, C.c_int32, _I32P]),
    "b200kv_disk_get_stats": (C.c_int, [_P, C.POINTER(DiskStats)]),
    "b200kv_disk_clear": (C.c_int, [_P]),
}

_lib = None


class B200KVError(RuntimeError):
    def __init__(self, code: int, where: str):
        self.code = code
        detail = ""
        try:
            msg = lib().b200kv_strerror(code).decode()
            if code == ENODEV:
                detail = " — " + lib().b200kv_last_error().decode()
        except Exception:  # pragma: no cover
            msg = "?"
        super().__init__(f"{where} failed: {code} ({msg}){detail}")


def lib() -> C.CDLL:
    """Load libb200kv.so once.  Raises (no fallback) when it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; "
                "g.build()'` (or make -C production-stack_b200/csrc).  b200kv has no CPU fallback.")
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        if l.b200kv_abi_version() != 1:
            raise ImportError("libb200kv.so ABI version mismatch")
        _lib = l
    return _lib


def check(code: int, where: str) -> int:
    if code < 0:
        raise B200KVError(code, where)
    return code
