"""Configuration surface: the env vars / JSON keys production-stack already emits for LMCache
(SURVEY.md Appendix A; helm/templates/deployment-vllm-multi.yaml:274-383,
operator/internal/controller/vllmruntime_controller.go:519-583) mapped onto this engine, so the
Helm chart and the operator stay byte-identical.  ``B200KV_*`` variables are this build's own.
"""
from __future__ import annotations

import logging
import os
import tempfile
from dataclasses import dataclass, field

from ._lib import FMT_FP8, FMT_Q4, FMT_RAW

logger = logging.getLogger("b200kv")

_TRUE = {"1", "true", "yes", "on"}

# accepted for compatibility but without effect here (out of scope rows of SURVEY.md Appendix A)
_IGNORED = ("LMCACHE_ENABLE_NIXL", "LMCACHE_NIXL_ROLE", "LMCACHE_USE_EXPERIMENTAL")


def _b(v: str | None, default: bool) -> bool:
    return default if v is None else v.strip().lower() in _TRUE


@dataclass
class B200KVConfig:
    chunk_size: int = 256                 # LMCACHE_CHUNK_SIZE
    local_cpu: bool = True                # LMCACHE_LOCAL_CPU
    max_local_cpu_size_gb: float = 5.0    # LMCACHE_MAX_LOCAL_CPU_SIZE (GB; tutorials use 20/30/60/120)
    fmt: int = FMT_RAW                    # LMCACHE_REMOTE_SERDE=cachegen or B200KV_FORMAT=fp8 -> FMT_FP8
    save_unfull_chunk: bool = True        # LMCACHE_SAVE_UNFULL_CHUNK
    save_decode_cache: bool = False       # LMCACHE_SAVE_DECODE_CACHE
    priority_limit: int | None = None     # LMCACHE_PRIORITY_LIMIT: requests with priority > limit are not saved
    instance_id: str = "b200kv_default_instance"   # LMCACHE_LMCACHE_INSTANCE_ID (pod name)
    enable_controller: bool = False       # LMCACHE_ENABLE_CONTROLLER
    controller_pull_url: str | None = None   # LMCACHE_CONTROLLER_PULL_URL  (router side binds)
    controller_reply_url: str | None = None  # LMCACHE_CONTROLLER_REPLY_URL
    worker_heartbeat_s: float = 10.0      # LMCACHE_LMCACHE_WORKER_HEARTBEAT_TIME
    advertise_ip: str | None = None       # B200KV_ADVERTISE_IP / LMCACHE_P2P_HOST: the address the router knows this
                                          # engine by (default: the pod's outbound IP)
    pool_name: str | None = None          # B200KV_POOL_NAME: POSIX shm name; shared => config 3
    staging_mb: int = 4096                # B200KV_STAGING_MB: device staging ring (half for stores, half for loads;
                                          # a layer-wise load needs all its chunks resident: 2 GiB = 8K tokens of Llama-3-8B)
    lookup_lease_ms: int = 30000          # B200KV_LOOKUP_LEASE_MS
    variant: int = 0                      # B200KV_VARIANT (0 bulk/TMA, 1 LDG)
    async_load: bool = False              # B200KV_ASYNC_LOAD=1: loads detached from the forward pass (costs one
                                          # extra scheduler step before the request can run)
    layerwise: bool = True                # B200KV_LAYERWISE / LMCACHE_USE_LAYERWISE: per-layer-group loads (default on:
                                          # layer l's attention starts once its group is in the pages; outputs identical)
    layer_group: int = 4                  # B200KV_LAYER_GROUP: layers per group
    device_tier_gb: float = 0.0           # B200KV_DEVICE_TIER_GB: HBM kept as a chunk cache peers can pull from (0 = off)
    remote_url: str | None = None         # LMCACHE_REMOTE_URL=lm://host:port: cache-server tier (b200kv/remote.py)
    remote_wait_ms: int = 2000            # B200KV_REMOTE_WAIT_MS: longest a request waits for its remote prefetch
    local_disk: str | None = None         # LMCACHE_LOCAL_DISK: file:///dir/, /dir, or True (a directory under $TMPDIR)
    max_local_disk_size: float = 0.0      # LMCACHE_MAX_LOCAL_DISK_SIZE (GB); the disk tier needs both (b200kv/disk.py)
    disk_wait_ms: int = 2000              # B200KV_DISK_WAIT_MS: longest a request waits for its disk prefetch
    extra: dict = field(default_factory=dict)

    @staticmethod
    def _file_overrides(path: str) -> dict:
        """LMCACHE_CONFIG_FILE: LMCache's YAML config (vllm/.../lmcache_integration/utils.py:47-62);
        its keys are the env names without the LMCACHE_ prefix, lower-cased."""
        import yaml
        with open(path) as f:
            doc = yaml.safe_load(f) or {}
        return {"LMCACHE_" + str(k).upper(): str(v) for k, v in doc.items() if v is not None}

    @staticmethod
    def from_env(env=None) -> "B200KVConfig":
        e = dict(os.environ if env is None else env)
        if e.get("LMCACHE_CONFIG_FILE"):
            # file first, explicit environment variables win
            e = {**B200KVConfig._file_overrides(e["LMCACHE_CONFIG_FILE"]), **e}
        c = B200KVConfig()
        c.chunk_size = int(e.get("LMCACHE_CHUNK_SIZE", c.chunk_size))
        c.local_cpu = _b(e.get("LMCACHE_LOCAL_CPU"), True)
        c.max_local_cpu_size_gb = float(e.get("LMCACHE_MAX_LOCAL_CPU_SIZE", c.max_local_cpu_size_gb))
        serde = (e.get("LMCACHE_REMOTE_SERDE") or "").lower()
        fmt = (e.get("B200KV_FORMAT") or ("fp8" if serde == "cachegen" else "raw")).lower()
        if fmt not in ("raw", "bf16", "naive", "fp8", "q4"):
            raise ValueError(f"B200KV_FORMAT={fmt!r}: expected raw|fp8|q4")
        c.fmt = {"fp8": FMT_FP8, "q4": FMT_Q4}.get(fmt, FMT_RAW)
        c.save_unfull_chunk = _b(e.get("LMCACHE_SAVE_UNFULL_CHUNK"), True)
        c.save_decode_cache = _b(e.get("LMCACHE_SAVE_DECODE_CACHE"), False)
        c.priority_limit = int(e["LMCACHE_PRIORITY_LIMIT"]) if e.get("LMCACHE_PRIORITY_LIMIT") not in (None, "") else None
        c.instance_id = e.get("LMCACHE_LMCACHE_INSTANCE_ID", c.instance_id)
        c.enable_controller = _b(e.get("LMCACHE_ENABLE_CONTROLLER"), False)
        c.controller_pull_url = e.get("LMCACHE_CONTROLLER_PULL_URL") or e.get("LMCACHE_CONTROLLER_URL")
        c.controller_reply_url = e.get("LMCACHE_CONTROLLER_REPLY_URL")
        c.worker_heartbeat_s = float(e.get("LMCACHE_LMCACHE_WORKER_HEARTBEAT_TIME", c.worker_heartbeat_s))
        c.advertise_ip = e.get("B200KV_ADVERTISE_IP") or e.get("LMCACHE_P2P_HOST") or None
        c.pool_name = e.get("B200KV_POOL_NAME") or None
        c.staging_mb = int(e.get("B200KV_STAGING_MB", c.staging_mb))
        c.lookup_lease_ms = int(e.get("B200KV_LOOKUP_LEASE_MS", c.lookup_lease_ms))
        c.variant = int(e.get("B200KV_VARIANT", 0))
        c.async_load = _b(e.get("B200KV_ASYNC_LOAD"), False)
        c.layerwise = _b(e.get("B200KV_LAYERWISE", e.get("LMCACHE_USE_LAYERWISE")), True)
        c.layer_group = max(1, int(e.get("B200KV_LAYER_GROUP", c.layer_group)))
        c.device_tier_gb = float(e.get("B200KV_DEVICE_TIER_GB", c.device_tier_gb))
        c.remote_url = e.get("LMCACHE_REMOTE_URL") or None
        c.remote_wait_ms = int(e.get("B200KV_REMOTE_WAIT_MS", c.remote_wait_ms))
        c.local_disk = e.get("LMCACHE_LOCAL_DISK") or None
        c.max_local_disk_size = float(e.get("LMCACHE_MAX_LOCAL_DISK_SIZE") or 0)
        c.disk_wait_ms = int(e.get("B200KV_DISK_WAIT_MS", c.disk_wait_ms))
        if c.max_local_disk_size > 0 and not _disk_path_given(c.local_disk):
            logger.warning("%s=%s is accepted for chart compatibility but has no effect in b200kv",
                           "LMCACHE_MAX_LOCAL_DISK_SIZE", e.get("LMCACHE_MAX_LOCAL_DISK_SIZE"))
        elif _disk_path_given(c.local_disk) and c.max_local_disk_size <= 0:
            logger.warning("LMCACHE_LOCAL_DISK=%s has no effect without LMCACHE_MAX_LOCAL_DISK_SIZE > 0", c.local_disk)
        for k in _IGNORED:
            if e.get(k) not in (None, "", "0", "False", "false"):
                logger.warning("%s=%s is accepted for chart compatibility but has no effect in b200kv", k, e.get(k))
        lvl = e.get("LMCACHE_LOG_LEVEL")
        if lvl:
            logger.setLevel(getattr(logging, lvl.upper(), logging.INFO))
        return c

    def apply_extra(self, extra: dict | None):
        """kv_connector_extra_config: `lmcache.<key>` / `b200kv.<key>` override the env
        (vllm/.../lmcache_integration/vllm_v1_adapter.py:588-600)."""
        for k, v in (extra or {}).items():
            for prefix in ("lmcache.", "b200kv."):
                if k.startswith(prefix):
                    name = k[len(prefix):]
                    if name == "format":
                        self.fmt = {"fp8": FMT_FP8, "q4": FMT_Q4}.get(str(v).lower(), FMT_RAW)
                    elif hasattr(self, name):
                        cur = getattr(self, name)
                        setattr(self, name, type(cur)(v) if cur is not None and not isinstance(cur, bool)
                                else (_b(str(v), False) if isinstance(cur, bool) else v))
                    else:
                        self.extra[name] = v
        return self

    @property
    def pool_bytes(self) -> int:
        return int(self.max_local_cpu_size_gb * (1 << 30))

    @property
    def disk_bytes(self) -> int:
        """LMCACHE_MAX_LOCAL_DISK_SIZE in bytes, GB read as GiB like LMCACHE_MAX_LOCAL_CPU_SIZE (pool_bytes)."""
        return int(self.max_local_disk_size * (1 << 30))

    def disk_dir(self) -> str | None:
        """The disk tier's directory, or None when the tier is off (it needs LMCACHE_LOCAL_DISK and a size > 0).
        `file:///dir/` and `/dir` name it; True / 1 (what the operator emits) means default_disk_dir()."""
        if self.max_local_disk_size <= 0 or not _disk_path_given(self.local_disk):
            return None
        v = str(self.local_disk).strip()
        if v.lower() in _TRUE:
            return default_disk_dir()
        if v.startswith("file://"):
            v = v[len("file://"):]
        if "://" in v or not v.startswith("/"):
            raise ValueError(f"LMCACHE_LOCAL_DISK={self.local_disk!r}: expected file:///dir/, /dir or True")
        return v


def default_disk_dir() -> str:
    """Where LMCACHE_LOCAL_DISK=True puts the disk tier: b200kv-disk under $TMPDIR (/tmp by default)."""
    return os.path.join(tempfile.gettempdir(), "b200kv-disk")


def _disk_path_given(v) -> bool:
    return v is not None and str(v).strip().lower() not in ("", "0", "false", "no", "off", "none")
