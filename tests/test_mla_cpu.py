"""MLA (DeepSeek-V2/V3, Kimi-K2) support without a GPU: layout detection on tensors built the way vLLM's MLA
backends allocate them, chunk geometry through the C ABI, the FP8 latent record specification, the
tensor-parallel key namespace and store policy, and the P/D layout check."""
import importlib
from types import SimpleNamespace as NS

import numpy as np
import pytest

from tests import mla_oracle as mo
from b200kv import _lib
from b200kv.engine import KVGeometry, paged_layout_of

# DeepSeek-V3: 61 layers, one 576-element latent per token and layer, chunk 256
V3 = dict(n_layers=61, n_kv_heads=1, head_dim=576, n_blocks=1, block_tokens=64, chunk_tokens=256, elem_bytes=2,
          layout=_lib.LAYOUT_MLA)


def _mla_backends():
    out = []
    for mod, name in (("vllm.model_executor.layers.attention.mla_attention", "MLACommonBackend"),
                      ("vllm.v1.attention.backends.mla.flashmla", "FlashMLABackend"),
                      ("vllm.v1.attention.backends.mla.triton_mla", "TritonMLABackend"),
                      ("vllm.v1.attention.backends.mla.flashinfer_mla", "FlashInferMLABackend")):
        try:
            out.append(getattr(importlib.import_module(mod), name))
        except Exception:      # a backend module that cannot be imported without its GPU library
            continue
    return out


@pytest.mark.parametrize("bs", [16, 64, 128])
def test_layout_detection_on_tensors_built_like_vllms_mla_backends(bs):
    """The physical layout is whatever vLLM allocates: the backend's get_kv_cache_shape permuted by its
    get_kv_cache_stride_order, viewed back in logical order (as test_connector_cpu does for FlashAttention)."""
    pytest.importorskip("vllm")
    import torch
    backends = _mla_backends()
    assert backends, "vLLM's MLA backends could not be imported"
    NB, D = 7, 576
    for B in backends:
        shape = B.get_kv_cache_shape(NB, bs, 1, D)
        order = B.get_kv_cache_stride_order()
        phys = tuple(shape[i] for i in order)
        inv = [order.index(i) for i in range(len(order))]
        t = torch.arange(int(np.prod(shape)), dtype=torch.int32).to(torch.bfloat16).view(phys).permute(*inv)
        k, v, stride, nb, h, d, tile = paged_layout_of(t, bs)
        assert (v, nb, h, d, tile) == (None, NB, 1, D, _lib.LAYOUT_MLA), B.__name__
        assert stride == bs * D * 2
        for b, j, e in [(0, 0, 0), (3, 5, 511), (NB - 1, bs - 1, D - 1)]:
            assert k + b * stride + (j * D + e) * 2 == t[b, j, e].data_ptr()


def test_other_ranks_and_orders_still_raise():
    import torch
    t = torch.zeros(4, 16, 576, dtype=torch.bfloat16)
    with pytest.raises(NotImplementedError):
        paged_layout_of(t.transpose(1, 2).contiguous().transpose(1, 2), 16)    # (NB, bs, D) with D outer
    with pytest.raises(ValueError):
        paged_layout_of(t, 32)
    with pytest.raises(NotImplementedError):
        paged_layout_of(torch.zeros(2, 4, 16, 576), 16)


def test_deepseek_v3_chunk_bytes():
    raw = KVGeometry(**V3)
    fp8 = KVGeometry(**V3, fmt=_lib.FMT_FP8)
    assert raw.planes == 61 and raw.chunk_bytes == 17_989_632 == mo.chunk_bytes(61, 256)
    assert fp8.chunk_bytes == 10_244_096 == mo.chunk_bytes(61, 256, fmt="fp8")
    assert raw.payload_bytes_per_token == 70_272 and fp8.payload_bytes_per_token == 61 * 656
    # an fp8 (e4m3) cache is moved RAW at one byte per element
    assert KVGeometry(**{**V3, "elem_bytes": 1}).chunk_bytes == 61 * 256 * 576
    # K/V geometries are unchanged
    llama = KVGeometry(32, 8, 128, 1)
    assert llama.planes == 64 and llama.payload_bytes_per_token == 131_072


@pytest.mark.parametrize("change,code", [
    (dict(n_kv_heads=2), _lib.EINVAL),                           # the latent is per token, not per head
    (dict(fmt=_lib.FMT_Q4), _lib.ENOTSUP),                       # no Q4 on MLA
    (dict(fmt=_lib.FMT_FP8, head_dim=512), _lib.ENOTSUP),        # the record is defined for 512 + 64
    (dict(fmt=_lib.FMT_FP8, elem_bytes=1), _lib.ENOTSUP),        # FP8 needs a bf16 source
    (dict(layout=3), _lib.EINVAL),
])
def test_refused_geometries(change, code):
    from b200kv._lib import B200KVError
    with pytest.raises(B200KVError) as e:
        KVGeometry(**{**V3, **change}).chunk_bytes
    assert e.value.code == code


# ---------------------------------------------------------------------------------------------------------------
# FP8 latent record specification
# ---------------------------------------------------------------------------------------------------------------
def _bits(x):
    import torch
    return torch.as_tensor(np.asarray(x, np.float32)).bfloat16().view(torch.int16).numpy().view(np.uint16)


def test_record_layout_rope_verbatim_and_roundtrip_within_tolerance():
    rng = np.random.default_rng(0)
    x = rng.standard_normal((3, 1, 37, 1, 576)).astype(np.float32)
    x[..., :128] *= 40.0                                    # groups of very different ranges
    x[..., 384:512] *= 1e-3
    bits = _bits(x)
    rec = mo.fp8_pack_chunk(bits)
    assert rec.shape == (3, 37, 656)
    assert np.array_equal(rec[..., 528:].view("<u2"), bits[:, 0, :, 0, 512:])       # RoPE bytes verbatim
    s = mo.record_scales(rec)
    amax = np.abs(mo.ko.bf16_bits_to_f32(bits[:, 0, :, 0, :512])).reshape(3, 37, 4, 128).max(-1)
    assert np.array_equal(s, (amax / np.float32(448.0)).astype(np.float32))
    back = mo.fp8_unpack_chunk(rec)
    assert np.array_equal(back[..., 512:], bits[..., 512:])
    err = np.abs(mo.ko.bf16_bits_to_f32(back).astype(np.float64) - mo.ko.bf16_bits_to_f32(bits).astype(np.float64))
    assert (err <= mo.fp8_tolerance(bits)).all()
    assert (mo.fp8_tolerance(bits)[..., 512:] == 0).all()


def test_zero_group_has_scale_one_and_zero_codes():
    x = np.ones((1, 1, 2, 1, 576), np.float32)
    x[..., 128:256] = 0.0
    rec = mo.fp8_pack_chunk(_bits(x))
    assert (mo.record_scales(rec)[..., 1] == 1.0).all()
    assert (rec[..., 128:256] == 0).all()
    assert np.array_equal(mo.fp8_unpack_chunk(rec), _bits(x))      # 1.0 and 0.0 are exact


def test_group_absmax_maps_to_448_and_codes_saturate():
    x = np.zeros((1, 1, 1, 1, 576), np.float32)
    x[..., 0] = -3.0
    x[..., 1] = 1.5
    rec = mo.fp8_pack_chunk(_bits(x))
    assert rec[0, 0, 0] == 0xFE               # -448: the absmax element takes the largest finite code
    assert rec[0, 0, 1] == 0x76               # 1.5 * 448 / 3 = 224 = 1.75 * 2^7
    # a product just above 448 (inv rounded up) saturates to the finite maximum instead of NaN
    assert mo.ko.f32_to_e4m3_satfinite(np.float32([448.0 * (1 + 2 ** -20), 1e9]))[0] == 0x7E
    assert mo.ko.f32_to_e4m3_satfinite(np.float32([1e9]))[0] == 0x7E


# ---------------------------------------------------------------------------------------------------------------
# tensor parallelism: one namespace, one writer
# ---------------------------------------------------------------------------------------------------------------
def test_mla_key_seed_is_shared_by_tensor_parallel_ranks():
    mla = KVGeometry(**V3)
    kv = KVGeometry(61, 8, 128, 1)
    seeds = [mla.key_seed("deepseek-v3", 8, r) for r in range(8)]
    assert len(set(seeds)) == 1
    assert mla.key_seed("deepseek-v3", 8, 8) != seeds[0]                 # another pipeline stage
    assert mla.key_seed("deepseek-v3", 4, 0) != seeds[0]                 # world size stays in the namespace
    assert mla.key_seed("other", 8, 0) != seeds[0]
    assert len({kv.key_seed("llama", 8, r) for r in range(8)}) == 8     # K/V shards still differ per rank


class _RecordingEngine:
    def __init__(self):
        self.calls = []

    def store(self, *a, **kw):
        self.calls.append("store")
        return 1

    def store_batch(self, *a, **kw):
        self.calls.append("store_batch")
        return 1

    def _keys(self, tokens):
        return np.arange((len(tokens) + 63) // 64, dtype=np.uint64)


@pytest.mark.parametrize("stores", [False, True])
def test_only_the_storing_rank_issues_store_ops(stores):
    from b200kv.adapter import WorkerState
    eng = _RecordingEngine()
    w = WorkerState(eng, 16, 64, stores=stores)
    metas = [NS(save_spec=NS(can_save=True, skip_leading_tokens=0), token_ids=list(range(n)), is_last_prefill=True,
                slot_mapping=lambda bs, n=n: np.arange(n, dtype=np.int64), req_id=str(n)) for n in (100, 130)]
    w.save(metas)
    assert eng.calls == (["store_batch"] if stores else [])
    assert w.stats.num_stored_tokens == (230 if stores else 0)


def _fake_vllm_config(use_mla: bool, tp: int = 1):
    import torch
    from vllm.config import KVTransferConfig
    ktc = KVTransferConfig(kv_connector="B200KVConnector", kv_connector_module_path="b200kv.connector",
                           kv_role="kv_both", engine_id="mla", kv_connector_extra_config={})
    mc = NS(model="synth-deepseek", dtype=torch.bfloat16, use_mla=use_mla, get_num_layers=lambda pc: 61,
            get_num_kv_heads=lambda pc: 1 if use_mla else 8, get_head_size=lambda: 576 if use_mla else 128)
    return NS(kv_transfer_config=ktc, model_config=mc, parallel_config=NS(tensor_parallel_size=tp, rank=0),
              cache_config=NS(block_size=64, cache_dtype="auto"))


@pytest.mark.parametrize("fmt,want", [(_lib.FMT_RAW, 17_989_632), (_lib.FMT_FP8, 10_244_096)])
def test_geometry_from_vllm_for_an_mla_model(fmt, want):
    pytest.importorskip("vllm")
    from b200kv.config import B200KVConfig
    from b200kv.connector import geometry_from_vllm
    cfg = B200KVConfig()
    cfg.fmt = fmt
    g = geometry_from_vllm(_fake_vllm_config(True), cfg)
    assert (g.layout, g.n_kv_heads, g.head_dim, g.planes) == (_lib.LAYOUT_MLA, 1, 576, 61)
    assert g.chunk_bytes == want
    g2 = geometry_from_vllm(_fake_vllm_config(False), cfg)
    assert (g2.layout, g2.n_kv_heads, g2.planes) == (_lib.LAYOUT_NHD, 8, 122)


# ---------------------------------------------------------------------------------------------------------------
# disaggregated prefill: producer and consumer must agree on the layout
# ---------------------------------------------------------------------------------------------------------------
class _PdEngine:
    def __init__(self, layout):
        self.geom = NS(n_blocks=64, stride=64 * 1152, n_layers=2, n_kv_heads=1, head_dim=576, block_tokens=64,
                       elem_bytes=2, layout=layout)

    def export_ipc(self):
        return b"\x07" * (72 * 2)

    def import_peer(self, pid, device, descs, stride, n_blocks):
        self.imported = (pid, device, len(descs), stride, n_blocks)


def test_pd_layout_mismatch_is_refused(tmp_path, monkeypatch):
    from b200kv import pd
    monkeypatch.setattr(pd, "SHM_DIR", str(tmp_path))
    pd.publish_ipc("P-mla", _PdEngine(_lib.LAYOUT_MLA), device=0)
    with pytest.raises(ValueError, match="layout"):
        pd.PeerResolver(_PdEngine(_lib.LAYOUT_NHD)).resolve("P-mla")
    same = _PdEngine(_lib.LAYOUT_MLA)
    assert pd.PeerResolver(same).resolve("P-mla") == 0 and same.imported[2] == 72 * 2
