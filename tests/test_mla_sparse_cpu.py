"""Sparse-attention MLA caches (DeepSeek-V3.2) without a GPU: layout detection on tensors built the way vLLM's
FlashMLASparseBackend and DeepseekV32IndexerBackend allocate them, the V3.2 chunk sizes through the C ABI and the
oracle (tests/mla_sparse_oracle.py), the split-tile piece builder of csrc/b200kv_runs.h against the oracle's
per-token rule, key seeds and format tags, the P/D check and the ABI's refusals."""
import ctypes
import importlib
import os
import subprocess
from types import SimpleNamespace as NS

import numpy as np
import pytest

from oracle import kv_oracle as ko
from tests import mla_sparse_oracle as so
from b200kv import _lib
from b200kv.engine import KVGeometry, indexer_layout_of, paged_layout_of, split_indexer_caches

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# DeepSeek-V3.2: 61 layers, a 576-element latent and a 132-byte indexer key per token and layer, chunk 256
V32 = dict(n_layers=61, n_kv_heads=1, head_dim=576, n_blocks=1, block_tokens=64, chunk_tokens=256, elem_bytes=2,
           layout=_lib.LAYOUT_MLA, idx_value_bytes=128, idx_scale_bytes=4)


def _alloc_like_vllm(backend, NB, bs, head_size, dtype, cache_dtype="auto"):
    import torch
    shape = backend.get_kv_cache_shape(NB, bs, 1, head_size, cache_dtype_str=cache_dtype)
    try:
        order = backend.get_kv_cache_stride_order()
    except (AttributeError, NotImplementedError):
        order = tuple(range(len(shape)))
    phys = tuple(shape[i] for i in order)
    inv = [order.index(i) for i in range(len(order))]
    return torch.zeros(phys, dtype=dtype).permute(*inv)


@pytest.mark.parametrize("bs", [64])
@pytest.mark.parametrize("cache_dtype", ["auto", "fp8_ds_mla"])
def test_layout_detection_on_tensors_built_like_vllms_sparse_backends(bs, cache_dtype):
    pytest.importorskip("vllm")
    import torch
    sparse = importlib.import_module("vllm.v1.attention.backends.mla.flashmla_sparse").FlashMLASparseBackend
    indexer = importlib.import_module("vllm.v1.attention.backends.mla.indexer").DeepseekV32IndexerBackend
    NB, L = 9, 3
    lat_dtype = torch.uint8 if cache_dtype == "fp8_ds_mla" else torch.bfloat16
    caches = {}
    for l in range(L):   # the model runner's order: a layer's attention, then its indexer
        caches[f"model.layers.{l}.self_attn.attn"] = _alloc_like_vllm(sparse, NB, bs, 576, lat_dtype, cache_dtype)
        caches[f"model.layers.{l}.self_attn.indexer.k_cache"] = _alloc_like_vllm(indexer, NB, bs, 132, torch.uint8)
    lat, idx = split_indexer_caches(caches)
    assert len(lat) == len(idx) == L
    k, v, stride, nb, h, d, tile = paged_layout_of(lat[0], bs)
    D, es = (656, 1) if cache_dtype == "fp8_ds_mla" else (576, 2)
    assert (v, nb, h, d, tile, stride) == (None, NB, 1, D, _lib.LAYOUT_MLA, bs * D * es)
    ptr, istride, inb = indexer_layout_of(idx[1], bs)
    assert (istride, inb) == (bs * 132, NB) and ptr == idx[1].data_ptr()
    # a name that contradicts the shape, or latent and indexer of different layers, is refused
    bad = dict(caches)
    bad["model.layers.0.self_attn.indexer.k_cache"] = caches["model.layers.0.self_attn.attn"]
    with pytest.raises(ValueError):
        split_indexer_caches(bad)
    swapped = {n: caches[n] for n in list(caches)[:2]}
    swapped["model.layers.1.self_attn.indexer.k_cache"] = swapped.pop("model.layers.0.self_attn.indexer.k_cache")
    with pytest.raises(ValueError, match="same layer"):
        split_indexer_caches(swapped)
    # plain MLA: no indexer caches
    assert split_indexer_caches([lat[0], lat[1]])[1] == []


def test_deepseek_v32_chunk_bytes():
    raw = KVGeometry(**V32)
    fp8 = KVGeometry(**V32, fmt=_lib.FMT_FP8)
    ds = KVGeometry(**{**V32, "head_dim": 656, "elem_bytes": 1})          # fp8_ds_mla: records stored RAW
    assert raw.chunk_bytes == 17_989_632 + 2_061_312 == 20_050_944 == so.chunk_bytes(61, 256)
    assert fp8.chunk_bytes == 10_244_096 + 2_061_312 == so.chunk_bytes(61, 256, fmt="fp8")
    assert ds.chunk_bytes == 12_305_408 == so.chunk_bytes(61, 256, 656, 1)
    assert raw.payload_bytes_per_token == 61 * (1152 + 132)
    assert fp8.payload_bytes_per_token == 61 * (656 + 132)
    # the whole chunk is rounded up, not its parts
    assert KVGeometry(**{**V32, "n_layers": 3, "chunk_tokens": 64}).chunk_bytes == (3 * 64 * 1152 + 3 * 64 * 132 + 255) // 256 * 256
    # without indexer planes nothing changes
    assert KVGeometry(**{**V32, "idx_value_bytes": 0, "idx_scale_bytes": 0}).chunk_bytes == 17_989_632


@pytest.mark.parametrize("change,code", [
    (dict(layout=_lib.LAYOUT_NHD, n_kv_heads=8, head_dim=128), _lib.EINVAL),   # indexer planes are MLA only
    (dict(idx_value_bytes=120), _lib.EINVAL),                                  # values in 16-byte vectors
    (dict(idx_scale_bytes=2), _lib.EINVAL),                                    # scales in 4-byte words
    (dict(layout=3), _lib.EINVAL),
    (dict(fmt=_lib.FMT_Q4), _lib.ENOTSUP),                                     # still no Q4 on MLA
])
def test_refused_geometries(change, code):
    from b200kv._lib import B200KVError
    with pytest.raises(B200KVError) as e:
        KVGeometry(**{**V32, **change}).chunk_bytes
    assert e.value.code == code


def test_abi_refusals_without_an_engine():
    l = _lib.lib()
    assert l.b200kv_set_indexer(None, 128, 4, 64 * 132) == _lib.EINVAL
    assert l.b200kv_engine_chunk_bytes_indexed(None, 128, 4) == _lib.EINVAL


# ---------------------------------------------------------------------------------------------------------------
# the split-tile piece builder (b200kv_runs.h) against the per-token rule
# ---------------------------------------------------------------------------------------------------------------
WRAPPER = r"""
#include <cstring>
#include "b200kv_runs.h"
using namespace b200kv;

static void move(const SplitPiece& p, const uint8_t* src, uint8_t* dst, int64_t* n_bulk) {
  std::memcpy(dst + p.dst, src + p.src, p.bytes);
  if (bulk_piece(p)) ++*n_bulk;
}

// store (mode 0) or load (mode 1) of L indexer planes (plane l at pages + l*plane_bytes) against chunks laid out
// as chunk c, layer l at chunks + (c*L + l)*slab; one table over `spans` as the engine builds it
extern "C" int apply_op(const int64_t* slots, const int64_t* spans, int64_t n_spans, int64_t max_slot, int32_t bs,
                        int32_t C, int32_t vb, int32_t sb, int mode, uint8_t* pages, uint64_t stride,
                        uint64_t plane_bytes, uint8_t* chunks, int32_t L, int64_t* n_val_bulk, int64_t* n_sc_bulk,
                        int64_t* n_runs) {
  std::vector<Span> sp;
  for (int64_t i = 0; i < n_spans; ++i) sp.push_back({spans[2 * i], spans[2 * i + 1]});
  OpTable t;
  const int rc = build_op_table(slots, sp.data(), sp.size(), max_slot, bs, C, false, false, &t);
  if (rc) return rc;
  const SplitTile tile{static_cast<uint32_t>(bs), static_cast<uint32_t>(C), static_cast<uint32_t>(vb),
                       static_cast<uint32_t>(sb), stride, stride};
  const uint64_t slab = static_cast<uint64_t>(C) * (vb + sb);
  *n_val_bulk = *n_sc_bulk = 0;
  *n_runs = static_cast<int64_t>(t.runs.size());
  for (const Run& r : t.runs) {
    SplitPiece v, s;
    split_run_pieces(tile, mode, r, &v, &s);
    for (int32_t l = 0; l < L; ++l) {
      uint8_t* pg = pages + l * plane_bytes;
      uint8_t* ch = chunks + (static_cast<uint64_t>(r.b / C) * L + l) * slab;
      move(v, mode == 0 ? pg : ch, mode == 0 ? ch : pg, n_val_bulk);
      move(s, mode == 0 ? pg : ch, mode == 0 ? ch : pg, n_sc_bulk);
    }
  }
  return 0;
}

extern "C" int apply_pull(const int64_t* src, const int64_t* dst, int64_t n, int64_t max_src, int64_t max_dst,
                          int32_t bs, int32_t vb, int32_t sb, const uint8_t* src_pages, uint64_t src_stride,
                          uint8_t* dst_pages, uint64_t dst_stride, int64_t* n_sc_bulk) {
  std::vector<Run> full, part;
  const int rc = build_pull_runs(src, dst, n, max_src, max_dst, bs, false, &full, &part);
  if (rc) return rc;
  const SplitTile tile{static_cast<uint32_t>(bs), 1, static_cast<uint32_t>(vb), static_cast<uint32_t>(sb), src_stride,
                       dst_stride};
  int64_t n_val = 0;
  *n_sc_bulk = 0;
  for (const Run& r : full) {
    SplitPiece v, s;
    split_run_pieces(tile, 2, r, &v, &s);
    move(v, src_pages, dst_pages, &n_val);
    move(s, src_pages, dst_pages, n_sc_bulk);
  }
  return 0;
}
"""


@pytest.fixture(scope="module")
def runs_lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("split")
    src, lib = d / "split_wrapper.cpp", d / "libsplitwrapper.so"
    src.write_text(WRAPPER)
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-shared", "-fPIC",
                    "-I", os.path.join(ROOT, "production-stack_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                    str(src), "-o", str(lib)], check=True)
    return ctypes.CDLL(str(lib))


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _mappings(rng, NB, bs, C):
    """name -> (slot_mapping with -1 padding, chunk spans [(tok_begin, n_tok)]) as the engine's ops see them."""
    out = {}
    n = 3 * C + 37
    out["block table, short last block"] = (ko.slot_mapping_from_blocks(rng.permutation(NB)[:(n + bs - 1) // bs], bs, n),
                                            [(c, min(C, n - c)) for c in range(0, n, C)])
    tok = rng.permutation(NB * bs)[:n].astype(np.int64)                  # token-granular: every token elsewhere
    out["token-granular"] = (tok, [(c, min(C, n - c)) for c in range(0, n, C)])
    shifted = (np.arange(n, dtype=np.int64) + 3) % (NB * bs)              # consecutive slots, blocks misaligned
    out["misaligned runs"] = (shifted, [(c, min(C, n - c)) for c in range(0, n, C)])
    # a batch: requests of 300, 64 and 200 tokens back to back, each request's tail padded to C
    perm, off, sm, spans = rng.permutation(NB), 0, [], []
    for r, m in enumerate((300, 64, 200)):
        nb = (m + bs - 1) // bs
        s = ko.slot_mapping_from_blocks(perm[off:off + nb], bs, m)
        off += nb
        for c in range(0, m, C):
            spans.append((len(sm) + 0, min(C, m - c)))
            part = s[c:c + C]
            sm.extend(part.tolist() + [-1] * (C - len(part)))
    out["partial chunks inside a batch"] = (np.asarray(sm, np.int64), spans)
    return out


@pytest.mark.parametrize("bs", [16, 64, 128])
def test_pieces_match_the_per_token_rule(runs_lib, bs):
    rng = np.random.default_rng(bs)
    L, C, NB = 2, 256, 2 * ((3 * 256 + 37 + bs - 1) // bs) + 5
    stride = bs * so.IDX_TOKEN + 16 * (bs == 16)            # a padded block stride is honoured too
    pages = [np.zeros((NB, stride), np.uint8) for _ in range(L)]
    for p in pages:
        p[:] = rng.integers(0, 256, p.shape, dtype=np.uint8)
    tiles = [p[:, :bs * so.IDX_TOKEN].reshape(NB, bs, so.IDX_TOKEN) for p in pages]   # the oracle's view
    flat = np.ascontiguousarray(np.stack(pages))
    slab = C * so.IDX_TOKEN
    for name, (sm, spans) in _mappings(rng, NB, bs, C).items():
        n_chunks = len(spans)
        chunks = np.zeros(n_chunks * L * slab, np.uint8)
        sp = np.ascontiguousarray(np.asarray(spans, np.int64).reshape(-1))
        nvb, nsb, nr = ctypes.c_int64(), ctypes.c_int64(), ctypes.c_int64()
        rc = runs_lib.apply_op(_p(sm), _p(sp), ctypes.c_int64(n_chunks), ctypes.c_int64(NB * bs), ctypes.c_int32(bs), ctypes.c_int32(C),
                               128, 4, 0, _p(flat), ctypes.c_uint64(stride), ctypes.c_uint64(NB * stride), _p(chunks),
                               ctypes.c_int32(L), ctypes.byref(nvb), ctypes.byref(nsb), ctypes.byref(nr))
        assert rc == 0, name
        assert nvb.value == nr.value * L, name                       # value pieces always go through the TMA engine
        got = chunks.reshape(n_chunks, L, slab)
        for c, (tb, n) in enumerate(spans):
            want = so.gather_slabs(tiles, sm[tb:tb + n], C)
            gv, gs = so.slab_tokens(got[c], n, C)
            wv, ws = so.slab_tokens(want, n, C)
            assert np.array_equal(gv, wv) and np.array_equal(gs, ws), (name, c)
        if name == "block table, short last block":
            # whole blocks: both pieces are 16-byte granular; only a short last block's scales may not be
            n_short = sum(1 for _, n in spans if n % bs and (n % bs) % 4)
            assert nsb.value >= (nr.value - n_short) * L, name
        # load the chunks into fresh pages: the mapped tokens take the chunk, every other byte stays
        fresh = np.ascontiguousarray(rng.integers(0, 256, flat.shape, dtype=np.uint8))
        expect = [f[:, :bs * so.IDX_TOKEN].reshape(NB, bs, so.IDX_TOKEN).copy() for f in fresh]
        expect_full = fresh.copy()
        for c, (tb, n) in enumerate(spans):
            so.scatter_slabs(expect, got[c], sm[tb:tb + n], C)
        for l in range(L):
            expect_full[l][:, :bs * so.IDX_TOKEN] = expect[l].reshape(NB, -1)
        rc = runs_lib.apply_op(_p(sm), _p(sp), ctypes.c_int64(n_chunks), ctypes.c_int64(NB * bs), ctypes.c_int32(bs), ctypes.c_int32(C),
                               128, 4, 1, _p(fresh), ctypes.c_uint64(stride), ctypes.c_uint64(NB * stride), _p(chunks),
                               ctypes.c_int32(L), ctypes.byref(nvb), ctypes.byref(nsb), ctypes.byref(nr))
        assert rc == 0 and np.array_equal(fresh, expect_full), name


@pytest.mark.parametrize("bs", [16, 64])
def test_pull_pieces_match_the_per_token_rule(runs_lib, bs):
    rng = np.random.default_rng(100 + bs)
    NB, n = 40, 500
    src_stride, dst_stride = bs * so.IDX_TOKEN, bs * so.IDX_TOKEN + 32
    src = np.ascontiguousarray(rng.integers(0, 256, (NB, src_stride), dtype=np.uint8))
    dst = np.ascontiguousarray(rng.integers(0, 256, (NB, dst_stride), dtype=np.uint8))
    nb = (n + bs - 1) // bs
    for s_map, d_map in [(ko.slot_mapping_from_blocks(rng.permutation(NB)[:nb], bs, n),
                          ko.slot_mapping_from_blocks(rng.permutation(NB)[:nb], bs, n)),
                         (rng.permutation(NB * bs)[:n].astype(np.int64), rng.permutation(NB * bs)[:n].astype(np.int64))]:
        out = dst.copy()
        nsb = ctypes.c_int64()
        rc = runs_lib.apply_pull(_p(s_map), _p(d_map), ctypes.c_int64(n), ctypes.c_int64(NB * bs), ctypes.c_int64(NB * bs),
                                 ctypes.c_int32(bs), 128, 4, _p(src), ctypes.c_uint64(src_stride), _p(out),
                                 ctypes.c_uint64(dst_stride), ctypes.byref(nsb))
        assert rc == 0
        expect = dst.copy()
        tiles_s = [src[:, :bs * so.IDX_TOKEN].reshape(NB, bs, so.IDX_TOKEN)]
        tiles_d = [expect[:, :bs * so.IDX_TOKEN].reshape(NB, bs, so.IDX_TOKEN)]
        so.scatter_slabs(tiles_d, so.gather_slabs(tiles_s, s_map[:256], 256), d_map[:256], 256)
        so.scatter_slabs(tiles_d, so.gather_slabs(tiles_s, s_map[256:], 256), d_map[256:], 256)
        assert np.array_equal(out, expect)


def test_out_of_range_slot_is_refused(runs_lib):
    sm = np.array([0, 1, 64 * 4], np.int64)
    sp = np.array([0, 3], np.int64)
    buf = np.zeros(4 * 64 * 132, np.uint8)
    ch = np.zeros(256 * 132, np.uint8)
    z = ctypes.c_int64()
    assert runs_lib.apply_op(_p(sm), _p(sp), ctypes.c_int64(1), ctypes.c_int64(4 * 64), ctypes.c_int32(64), ctypes.c_int32(256), 128, 4,
                             0, _p(buf), ctypes.c_uint64(64 * 132), ctypes.c_uint64(0), _p(ch), ctypes.c_int32(1), ctypes.byref(z),
                             ctypes.byref(z), ctypes.byref(z)) == _lib.EINVAL


# ---------------------------------------------------------------------------------------------------------------
# key seeds, format tags, vLLM configs, P/D
# ---------------------------------------------------------------------------------------------------------------
def test_key_seeds_and_format_tags():
    v32, v3 = KVGeometry(**V32), KVGeometry(**{**V32, "idx_value_bytes": 0, "idx_scale_bytes": 0})
    seeds = [v32.key_seed("deepseek-v3.2", 8, r) for r in range(8)]
    assert len(set(seeds)) == 1                                     # MLA's TP-rank rule is unchanged
    assert seeds[0] != v3.key_seed("deepseek-v3.2", 8, 0)          # "|idx132" keeps the namespaces apart
    assert v32.key_seed("deepseek-v3.2", 8, 8) != seeds[0]         # another pipeline stage
    assert v3.fmt_tag == _lib.LAYOUT_MLA << 8 and v32.fmt_tag == v3.fmt_tag | (1 << 24)
    f = KVGeometry(**V32, fmt=_lib.FMT_FP8)
    assert f.fmt_tag == _lib.FMT_FP8 | _lib.LAYOUT_MLA << 8 | 1 << 24
    # existing tags are unchanged: no bit 24 without indexer planes
    assert KVGeometry(32, 8, 128, 1).fmt_tag == 0


def _v32_vllm_config(cache_dtype="auto", sparse=True):
    import torch
    from vllm.config import KVTransferConfig
    ktc = KVTransferConfig(kv_connector="B200KVConnector", kv_connector_module_path="b200kv.connector",
                           kv_role="kv_both", engine_id="v32", kv_connector_extra_config={})
    hf = NS(index_topk=2048, index_head_dim=128, index_n_heads=64) if sparse else NS()
    mc = NS(model="synth-deepseek-v3.2", dtype=torch.bfloat16, use_mla=True, get_num_layers=lambda pc: 61,
            get_num_kv_heads=lambda pc: 1, get_head_size=lambda: 576, hf_config=hf, hf_text_config=hf)
    return NS(kv_transfer_config=ktc, model_config=mc, parallel_config=NS(tensor_parallel_size=1, rank=0),
              cache_config=NS(block_size=64, cache_dtype=cache_dtype))


@pytest.mark.parametrize("cache_dtype,fmt,want_fmt,want", [
    ("auto", _lib.FMT_RAW, _lib.FMT_RAW, 20_050_944),
    ("auto", _lib.FMT_FP8, _lib.FMT_FP8, 12_305_408),
    ("fp8_ds_mla", _lib.FMT_RAW, _lib.FMT_RAW, 12_305_408),
    ("fp8_ds_mla", _lib.FMT_FP8, _lib.FMT_RAW, 12_305_408)])    # the records are already FP8: stored RAW
def test_geometry_from_vllm_for_deepseek_v32(cache_dtype, fmt, want_fmt, want):
    pytest.importorskip("vllm")
    from b200kv.config import B200KVConfig
    from b200kv.connector import geometry_from_vllm
    cfg = B200KVConfig()
    cfg.fmt = fmt
    g = geometry_from_vllm(_v32_vllm_config(cache_dtype), cfg)
    assert g.indexed and (g.idx_value_bytes, g.idx_scale_bytes) == (128, 4) and g.fmt == want_fmt
    assert g.chunk_bytes == want
    assert not geometry_from_vllm(_v32_vllm_config(sparse=False), cfg).indexed     # DeepSeek-V3: no indexer
    cfg.fmt = _lib.FMT_Q4
    from b200kv._lib import B200KVError
    with pytest.raises(B200KVError):
        geometry_from_vllm(_v32_vllm_config(cache_dtype), cfg).chunk_bytes          # Q4 stays refused


class _PdEngine:
    def __init__(self, indexer):
        self.geom = NS(n_blocks=64, stride=64 * 1152, n_layers=2, n_kv_heads=1, head_dim=576, block_tokens=64,
                       elem_bytes=2, layout=_lib.LAYOUT_MLA, idx_token_bytes=indexer)

    def export_ipc(self):
        return b"\x07" * (72 * 4)

    def import_peer(self, pid, device, descs, stride, n_blocks):
        self.imported = (pid, device, len(descs), stride, n_blocks)


def test_pd_refuses_a_v32_producer_for_a_plain_mla_consumer(tmp_path, monkeypatch):
    import json
    from b200kv import pd
    monkeypatch.setattr(pd, "SHM_DIR", str(tmp_path))
    path = pd.publish_ipc("P-v32", _PdEngine(132), device=0)
    assert json.load(open(path))["indexer"] == 132
    with pytest.raises(ValueError, match="indexer"):
        pd.PeerResolver(_PdEngine(0)).resolve("P-v32")
    same = _PdEngine(132)
    assert pd.PeerResolver(same).resolve("P-v32") == 0 and same.imported[2] == 72 * 4
    # a document without the field was published by an engine without indexer planes
    doc = json.load(open(path))
    del doc["indexer"]
    json.dump(doc, open(path, "w"))
    with pytest.raises(ValueError, match="indexer"):
        pd.PeerResolver(_PdEngine(132)).resolve("P-v32")
    assert pd.PeerResolver(_PdEngine(0)).resolve("P-v32") == 0


# ---------------------------------------------------------------------------------------------------------------
# layer-wise loads against vLLM's DeepSeek-V3.2 layer order
# ---------------------------------------------------------------------------------------------------------------
class _StubEngine:
    """KVEngine's surface as register_kv_caches uses it (no CUDA)."""

    def __init__(self, geom, pool, **kw):
        self.geom, self.key_seed = geom, kw.get("key_seed")

    def numa_placement(self):
        return "stand-in"

    def register_kv_caches(self, kv_caches, layout=None):
        self.kv_caches = kv_caches

    def export_ipc(self):
        raise RuntimeError("no CUDA IPC on CPU")

    def wait_all(self):
        pass

    def close(self):
        pass


class _RecordingWorker:
    """WorkerState's load surface: one layer-wise load per step; every wait goes into the shared event log."""

    def __init__(self, log):
        self.log, self.layer_loads = log, []

    def start_load(self, metas, stream=None, layers_per_group=0):
        self.G = layers_per_group
        self.layer_loads = [(7, [0])] if layers_per_group else []
        self.log.append(("load", layers_per_group))

    def wait_layer(self, layer, stream=None):
        self.log.append(("wait", layer // self.G))       # the engine waits for the layer's whole group

    def save(self, metas, stream=None):
        pass


def _v32_worker(monkeypatch, L, G, sparse=True):
    import torch
    from vllm.distributed.kv_transfer.kv_connector.v1.base import KVConnectorRole
    import b200kv.connector as bc
    monkeypatch.setattr(bc, "KVEngine", _StubEngine)
    monkeypatch.setattr(torch.cuda, "current_stream", lambda *a, **k: None)
    monkeypatch.setenv("LMCACHE_MAX_LOCAL_CPU_SIZE", "0.05")
    monkeypatch.setenv("B200KV_LAYERWISE", "1")
    monkeypatch.setenv("B200KV_LAYER_GROUP", str(G))
    cfg = _v32_vllm_config(sparse=sparse)
    cfg.model_config.get_num_layers = lambda pc: L
    cfg.scheduler_config = NS(disable_hybrid_kv_cache_manager=False)
    cfg.kv_transfer_config.engine_id = f"v32-{os.getpid()}-{os.urandom(3).hex()}"
    w = bc.B200KVConnector(cfg, KVConnectorRole.WORKER, None)
    caches = {}
    for l in range(L):     # the model runner's order: a layer's attention, then its indexer
        caches[f"model.layers.{l}.self_attn.attn"] = torch.zeros((4, 64, 576), dtype=torch.bfloat16)
        if sparse:
            caches[f"model.layers.{l}.self_attn.indexer.k_cache"] = torch.zeros((4, 64, 132), dtype=torch.uint8)
    w.register_kv_caches(caches)
    log = []
    w._worker = _RecordingWorker(log)
    return w, log, bc


@pytest.mark.parametrize("G", [1, 2, 3, 5])
def test_layerwise_waits_cover_each_layer_before_its_indexer_reads(monkeypatch, G):
    """vLLM 0.22 runs layer l's indexer (which writes, then reads layer l's indexer keys) before layer l's attention,
    and only the attention calls wait_for_layer_load.  Simulating that order, every layer's group must have been
    waited for before its indexer runs — and its attention."""
    pytest.importorskip("vllm")
    L = 5
    w, log, bc = _v32_worker(monkeypatch, L, G)
    try:
        w.bind_connector_metadata(bc.B200KVConnectorMetadata())
        w.start_load_kv(NS(cudagraph_runtime_mode=NS(name="NONE")))
        for l in range(L):
            log.append(("indexer reads", l))
            w.wait_for_layer_load(f"model.layers.{l}.self_attn.indexer.k_cache")   # not a hook vLLM calls: a no-op
            w.wait_for_layer_load(f"model.layers.{l}.self_attn.attn")
            log.append(("attention", l))
        for l in range(L):
            for what in ("indexer reads", "attention"):
                at = log.index((what, l))
                assert ("wait", l // G) in log[:at], (G, l, what, log)
        assert log[0] == ("load", G)
        waits = [e for e in log if e[0] == "wait"]
        assert sorted(set(waits)) == [("wait", g) for g in range((L + G - 1) // G)]
    finally:
        w._worker = None
        w.shutdown()


def test_plain_mla_layerwise_waits_are_unchanged(monkeypatch):
    pytest.importorskip("vllm")
    w, log, bc = _v32_worker(monkeypatch, 4, 2, sparse=False)
    try:
        w.bind_connector_metadata(bc.B200KVConnectorMetadata())
        w.start_load_kv(NS(cudagraph_runtime_mode=NS(name="NONE")))
        for l in range(4):
            w.wait_for_layer_load(f"model.layers.{l}.self_attn.attn")
        assert log == [("load", 2), ("wait", 0), ("wait", 1)]      # in the hooks of layers 0 and 2 only
    finally:
        w._worker = None
        w.shutdown()
