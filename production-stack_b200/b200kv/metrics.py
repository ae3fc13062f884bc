"""`lmcache:*` Prometheus series, from this engine's counters, through vLLM's connector-stats hooks
(KVConnectorBase_V1.get_kv_connector_stats / build_kv_connector_stats / build_prom_metrics,
vllm/.../v1/base.py:403,625-660).  Series names are the ones production-stack's Grafana dashboard
queries (helm/dashboards/lmcache-dashboard.json:204,295,389,453,517):

    lmcache:num_hit_tokens_total, lmcache:num_requested_tokens_total, lmcache:local_cache_usage,
    lmcache:retrieve_speed_{sum,count}   (+ store_speed, num_stored_tokens_total)

With the local-disk tier on (LMCACHE_LOCAL_DISK), this build's own b200kv:disk_* series as well: disk_usage (bytes),
disk_{fetched,written,skipped,corrupt}_chunks.
"""
from __future__ import annotations

from dataclasses import dataclass, field
from typing import Any

from vllm.distributed.kv_transfer.kv_connector.v1.metrics import KVConnectorPromMetrics, KVConnectorStats

_SUM_KEYS = ("num_hit_tokens", "num_requested_tokens", "num_stored_tokens", "num_loaded_tokens",
             "retrieve_seconds", "retrieve_calls", "retrieve_bytes", "store_bytes", "load_shortfalls",
             "num_foreign_loaded_tokens", "num_tier_local_tokens", "num_tier_peer_tokens",
             "disk_fetched_chunks", "disk_written_chunks", "disk_skipped_chunks", "disk_corrupt_chunks")
_DISK_COUNTERS = ("fetched", "written", "skipped", "corrupt")


@dataclass
class B200KVStats(KVConnectorStats):
    data: dict[str, Any] = field(default_factory=dict)

    def reset(self):
        self.data = {}

    def aggregate(self, other: "KVConnectorStats") -> "KVConnectorStats":
        for k in _SUM_KEYS:
            if k in other.data:
                self.data[k] = self.data.get(k, 0) + other.data[k]
        for k in ("local_cache_usage_bytes", "local_cache_capacity_bytes", "disk_usage_bytes"):
            if k in other.data:
                self.data[k] = other.data[k]  # gauges: last value wins
        return self

    def reduce(self) -> dict[str, int | float]:
        d = self.data
        out: dict[str, int | float] = {k: d[k] for k in ("num_hit_tokens", "num_requested_tokens", "num_stored_tokens",
                                                          "num_loaded_tokens", "num_foreign_loaded_tokens", "num_tier_local_tokens",
                                                          "num_tier_peer_tokens")
                                        + tuple(f"disk_{c}_chunks" for c in _DISK_COUNTERS) if k in d}
        if d.get("retrieve_seconds"):
            out["retrieve_GBps"] = round(d.get("retrieve_bytes", 0) / d["retrieve_seconds"] / 1e9, 2)
        if "local_cache_usage_bytes" in d:
            out["local_cache_usage_GB"] = round(d["local_cache_usage_bytes"] / 1e9, 2)
        return out

    def is_empty(self) -> bool:
        return not any(self.data.get(k) for k in _SUM_KEYS)


class B200KVPromMetrics(KVConnectorPromMetrics):
    def __init__(self, vllm_config, metric_types, labelnames, per_engine_labelvalues):
        super().__init__(vllm_config, metric_types, labelnames, per_engine_labelvalues)

        def per_engine(metric):
            return {idx: metric.labels(*vals) for idx, vals in per_engine_labelvalues.items()}

        c, g = self._counter_cls, self._gauge_cls
        self.hit = per_engine(c(name="lmcache:num_hit_tokens", documentation="tokens found in the KV pool by lookups",
                                labelnames=labelnames))
        self.req = per_engine(c(name="lmcache:num_requested_tokens", documentation="tokens looked up in the KV pool",
                                labelnames=labelnames))
        self.stored = per_engine(c(name="lmcache:num_stored_tokens", documentation="tokens stored to the KV pool",
                                   labelnames=labelnames))
        self.foreign = per_engine(c(name="b200kv:cross_replica_loaded_tokens",
                                    documentation="tokens loaded from chunks another replica stored (shared pool)",
                                    labelnames=labelnames))
        self.tier_local = per_engine(c(name="b200kv:device_tier_local_tokens",
                                       documentation="tokens loaded from this engine's device chunk tier (no PCIe)",
                                       labelnames=labelnames))
        self.tier_peer = per_engine(c(name="b200kv:device_tier_peer_tokens",
                                      documentation="tokens loaded from a peer replica's device chunk tier over NVLink",
                                      labelnames=labelnames))
        self.usage = per_engine(g(name="lmcache:local_cache_usage", documentation="bytes of pinned host pool in use",
                                  labelnames=labelnames, multiprocess_mode="mostrecent"))
        self.r_sum = per_engine(c(name="lmcache:retrieve_speed_sum", documentation="sum of retrieve speeds (tokens/s)",
                                  labelnames=labelnames))
        self.r_cnt = per_engine(c(name="lmcache:retrieve_speed_count", documentation="number of retrieve calls",
                                  labelnames=labelnames))
        self.disk = None
        if _disk_enabled(vllm_config):
            docs = {"fetched": "chunks read from the local disk tier into the pinned pool",
                    "written": "chunks written through to the local disk tier",
                    "skipped": "stored chunks not written to disk (queue full, no free disk slot, already evicted)",
                    "corrupt": "disk chunks that failed their checksum (never loaded)"}
            self.disk = {k: per_engine(c(name=f"b200kv:disk_{k}_chunks", documentation=docs[k], labelnames=labelnames))
                         for k in _DISK_COUNTERS}
            self.disk_usage = per_engine(g(name="b200kv:disk_usage", documentation="bytes of the local disk tier in use",
                                           labelnames=labelnames, multiprocess_mode="mostrecent"))

    def observe(self, transfer_stats_data: dict[str, Any], engine_idx: int = 0):
        d = transfer_stats_data
        self.hit[engine_idx].inc(d.get("num_hit_tokens", 0))
        self.req[engine_idx].inc(d.get("num_requested_tokens", 0))
        self.stored[engine_idx].inc(d.get("num_stored_tokens", 0))
        self.foreign[engine_idx].inc(d.get("num_foreign_loaded_tokens", 0))
        self.tier_local[engine_idx].inc(d.get("num_tier_local_tokens", 0))
        self.tier_peer[engine_idx].inc(d.get("num_tier_peer_tokens", 0))
        if "local_cache_usage_bytes" in d:
            self.usage[engine_idx].set(d["local_cache_usage_bytes"])
        if self.disk is not None:
            for k in _DISK_COUNTERS:
                self.disk[k][engine_idx].inc(d.get(f"disk_{k}_chunks", 0))
            if "disk_usage_bytes" in d:
                self.disk_usage[engine_idx].set(d["disk_usage_bytes"])
        if d.get("retrieve_calls") and d.get("retrieve_seconds"):
            self.r_sum[engine_idx].inc(d.get("num_loaded_tokens", 0) / d["retrieve_seconds"] * d["retrieve_calls"])
            self.r_cnt[engine_idx].inc(d["retrieve_calls"])


def _disk_enabled(vllm_config) -> bool:
    from .config import B200KVConfig
    try:
        ktc = vllm_config.kv_transfer_config
        return B200KVConfig.from_env().apply_extra(ktc.kv_connector_extra_config).disk_dir() is not None
    except Exception:
        return False
