"""b200kv — H100-native KV-cache offload / cross-replica KV-transfer engine.

Drop-in for the vLLM KV-connector slot that vllm-project/production-stack fills with LMCache
(helm/templates/deployment-vllm-multi.yaml:194-207).  Python host code over the C ABI in
include/b200kv.h; hand-written sm_90a CUDA underneath; no CPU fallback.
"""
from ._lib import (DTYPE_BF16, DTYPE_FP16, FMT_FP8, FMT_Q4, FMT_RAW, VARIANT_BULK, VARIANT_LDG,  # noqa: F401
                   B200KVError, lib)
from .engine import KVEngine, KVGeometry, KVPool, chunk_keys, xxh64  # noqa: F401

__all__ = ["KVEngine", "KVGeometry", "KVPool", "chunk_keys", "xxh64", "B200KVError",
           "FMT_RAW", "FMT_FP8", "FMT_Q4", "DTYPE_BF16", "DTYPE_FP16", "VARIANT_BULK", "VARIANT_LDG", "lib"]
