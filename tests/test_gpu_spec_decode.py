"""Engines with speculative-decoding draft layers on an H100 (-m gpu).  vLLM hands the connector the drafter's
attention layers in the target's KV-cache group; they keep the target's geometry and follow its layers, so an engine
of L target and D draft layers is an engine of L + D layers with the draft layers at L..L+D-1.  Here the caches come
named as vLLM names them (draft layers from num_hidden_layers upwards) in a shuffled dict, are ordered as
register_kv_caches orders them, and every path is bit-exact against the existing oracles with the draft layers as
layers L..L+D-1: pool store and load chunk-wise, layer-wise and batched, the device-resident gather (chunk bytes), the
device tier and the same-process peer pull.  K/V NHD and HND with L = 4, D = 1; MLA RAW and FP8, and MLA with
indexer planes (DeepSeek-V3.2's MTP layer has one), with L = 3, D = 1."""
import random

import numpy as np
import pytest

from oracle import kv_oracle as ko
from tests import mla_oracle as mo
from tests import test_gpu_mla_sparse as sp
from tests.test_gpu_kernels import bits_of, logical_bits, mk_host_layers, to_dev, to_dev_hnd

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from b200kv import FMT_FP8, FMT_RAW, KVEngine, KVGeometry, KVPool, _lib  # noqa: E402

H, HD, MLA_D = 8, 128, 576
CASES = {   # name: (kind, L, D, fmt)
    "kv-nhd": ("nhd", 4, 1, FMT_RAW),
    "kv-hnd": ("hnd", 4, 1, FMT_RAW),
    "mla-raw": ("mla", 3, 1, FMT_RAW),
    "mla-fp8": ("mla", 3, 1, FMT_FP8),
    "mla-indexed": ("idx", 3, 1, FMT_RAW),
}


def need_gpu():
    if not torch.cuda.is_available():
        pytest.fail("GPU tests selected but no CUDA device: the product has no CPU fallback")


class Case:
    """Host pages of L + D layers, their device caches in the order register_kv_caches gives them, the geometry,
    and the oracle's pages after a store from one slot mapping and a load into another."""

    def __init__(self, name, rng, NB, bs, C=256):
        self.kind, self.L, self.D, self.fmt = CASES[name]
        self.NB, self.bs, self.C = NB, bs, C
        n = self.L + self.D
        if self.kind in ("nhd", "hnd"):
            self.host = mk_host_layers(rng, n, NB, bs, H, HD)
            self.idx = []
        else:
            self.host, idx = sp.mk_host(rng, n, NB, bs)
            self.idx = idx if self.kind == "idx" else []
        self.geom = {"nhd": lambda: KVGeometry(n, H, HD, NB, bs, C, 2, 0, self.fmt, draft_layers=self.D),
                     "hnd": lambda: KVGeometry(n, H, HD, NB, bs, C, 2, 2 * bs * H * HD * 2, self.fmt, _lib.LAYOUT_HND,
                                               draft_layers=self.D),
                     "mla": lambda: KVGeometry(n, 1, MLA_D, NB, bs, C, 2, 0, self.fmt, _lib.LAYOUT_MLA,
                                               draft_layers=self.D),
                     "idx": lambda: KVGeometry(n, 1, MLA_D, NB, bs, C, 2, 0, self.fmt, _lib.LAYOUT_MLA,
                                               idx_value_bytes=128, idx_scale_bytes=4, draft_layers=self.D)}[self.kind]()

    def device(self, zero=False):
        """{vLLM name: tensor} in a shuffled order -> ordered by layer index as register_kv_caches does."""
        host = [np.zeros_like(h) for h in self.host] if zero else self.host
        idx = [np.zeros_like(h) for h in self.idx] if zero else self.idx
        if self.kind in ("nhd", "hnd"):
            lat = to_dev_hnd(host) if self.kind == "hnd" else to_dev(host)
        else:
            lat = [torch.from_numpy(h.view(np.int16)).view(torch.bfloat16).cuda() for h in host]
        items = [(f"model.layers.{l}.self_attn.attn", t) for l, t in enumerate(lat)]
        items += [(f"model.layers.{l}.self_attn.indexer.k_cache", torch.from_numpy(h.copy()).cuda())
                  for l, h in enumerate(idx)]
        random.Random(len(items)).shuffle(items)
        from b200kv.connector import _layer_index_of
        return dict(sorted(items, key=lambda kv: _layer_index_of(kv[0])))

    def registered(self, caches):
        return caches if self.idx else list(caches.values())

    def pages(self, caches):
        """Host copies in engine order: the paged planes of the L + D layers, then the indexer planes."""
        out, idx = [], []
        for name, t in caches.items():
            if "indexer" in name:
                idx.append(t.cpu().numpy())
            elif self.kind == "hnd":
                out.append(logical_bits(t))
            else:
                out.append(bits_of(t))
        return out + idx

    def expect(self, sm, dm, before=None):
        """The oracle's pages after storing sm's tokens and loading them at dm (into `before`, default zeros)."""
        if before is None:
            before = [np.zeros_like(h) for h in self.host + self.idx]
        if self.kind in ("nhd", "hnd"):
            want = [b.copy() for b in before]
            oe = ko.OracleEngine(self.C, "fp8" if self.fmt == FMT_FP8 else "raw")
            toks = np.arange(len(sm), dtype=np.int32)
            oe.store(toks, np.ones(len(sm), bool), self.host, sm)
            oe.retrieve(toks, np.ones(len(sm), bool), want, dm)
            return want
        n = len(self.host)
        if self.idx:
            el, ei = sp.expected_pages(self.fmt, self.host, self.idx, sm, dm, self.C, before[:n], before[n:])
            return el + ei
        want = [b.copy() for b in before]
        for c in range(0, len(sm), self.C):
            bits = mo.gather_tokens(self.host, sm[c:c + self.C])
            if self.fmt == FMT_FP8:
                bits = mo.fp8_unpack_chunk(mo.fp8_pack_chunk(bits))
            mo.scatter_tokens(want, bits, dm[c:c + self.C])
        return want

    def check_chunk(self, got, sm):
        """One chunk's bytes (valid tokens only) against the oracle's chunk layout."""
        g, n, C = self.geom, len(sm), self.C
        if self.kind == "idx":
            sp.check_chunk(got, g, self.host, self.idx, sm, self.fmt)
        elif self.kind == "mla":
            tb = mo.MLA_RECORD if self.fmt == FMT_FP8 else MLA_D * 2
            have = got[:g.n_layers * C * tb].reshape(g.n_layers, C, tb)[:, :n]
            bits = mo.gather_tokens(self.host, sm)
            want = mo.fp8_pack_chunk(bits) if self.fmt == FMT_FP8 else bits
            assert np.array_equal(have, want.view(np.uint8).reshape(g.n_layers, n, tb))
        elif self.kind == "nhd":
            tb = g.token_bytes
            want = ko.gather_tokens(self.host, sm)          # (L + D, 2, n, H, D)
            for plane in range(2 * g.n_layers):
                o = plane * C * tb
                assert np.array_equal(got[o:o + n * tb].view(np.uint16).reshape(n, H, HD),
                                      want[plane // 2, plane % 2]), plane
        # HND chunks keep whole tiles: their bytes are covered by the page round trips


def slots(rng, NB, bs, n):
    return ko.slot_mapping_from_blocks(rng.permutation(NB)[:(n + bs - 1) // bs], bs, n)


def assert_pages(case, caches, want, what):
    for i, (a, b) in enumerate(zip(case.pages(caches), want)):
        assert np.array_equal(a, b), f"{what}: plane {i} of {case.geom.n_layers} layers (draft from {case.L})"


@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("mode", ["chunk", "layer", "batch"])
def test_pool_store_and_load(name, mode):
    need_gpu()
    rng = np.random.default_rng(sum(map(ord, name + mode)))
    case = Case(name, rng, 64, 16 if name.startswith("kv") else 64)
    g, bs, C = case.geom, case.bs, case.C
    assert (g.n_layers, g.draft_layers, g.target_layers) == (case.L + case.D, case.D, case.L)
    pool = KVPool(None, 12 * g.chunk_bytes, g.chunk_bytes, 1)
    src = case.device()
    eng = KVEngine(g, pool, 0, staging_bytes=4 * g.chunk_bytes)
    eng.register_kv_caches(case.registered(src))
    lens = [2 * C + 70, C + 5] if mode == "batch" else [2 * C + 70]
    perm, off, reqs = rng.permutation(case.NB), 0, []
    for i, n in enumerate(lens):
        nb = (n + bs - 1) // bs
        reqs.append(((np.arange(n, dtype=np.int32) + 5000 * i) % 9000,
                     ko.slot_mapping_from_blocks(perm[off:off + nb], bs, n)))
        off += nb
    if mode == "batch":
        eng.wait(eng.store_batch([(t, s, 0) for t, s in reqs]))
    else:
        eng.wait(eng.store(reqs[0][0], None, reqs[0][1]))
    for t, _ in reqs:
        assert eng.lookup(t) == len(t)
    key = eng._keys(reqs[0][0])[1]
    slot, _n, tag = pool.acquire(key)
    assert tag == g.fmt_tag
    case.check_chunk(pool.slot_view(slot), reqs[0][1][C:2 * C])    # the pool's chunk has the draft planes too
    pool.release(key)
    dst = case.device(zero=True)
    eng2 = KVEngine(g, pool, 0, staging_bytes=4 * g.chunk_bytes)
    eng2.register_kv_caches(case.registered(dst))
    perm2, off, dms = np.random.default_rng(5).permutation(case.NB), 0, []
    for t, _ in reqs:
        nb = (len(t) + bs - 1) // bs
        dms.append(ko.slot_mapping_from_blocks(perm2[off:off + nb], bs, len(t)))
        off += nb
    if mode == "batch":
        loaded, ticket = eng2.retrieve_batch([(t, d, 0) for (t, _), d in zip(reqs, dms)])
        assert list(loaded) == lens
        eng2.wait(ticket)
    elif mode == "chunk":
        assert eng2.retrieve(reqs[0][0], None, dms[0]).all()
    else:
        # one group per target layer pair, the draft layer in a group of its own: after the waits the connector
        # issues in the last target layer's hook, the draft layer's pages are complete
        G = case.L if case.L % 2 else 2
        assert case.L % G == 0 and (case.L + case.D + G - 1) // G == case.L // G + 1
        from b200kv.connector import hook_waits
        s = torch.cuda.Stream()
        ret, ticket = eng2.retrieve(reqs[0][0], None, dms[0], stream=s, return_ticket=True, layers_per_group=G)
        assert ret.all() and ticket
        for l in range(case.L):
            for x in hook_waits(l, case.L, case.L + case.D, G, case.kind == "idx"):
                eng2.wait_layer(ticket, x, s)
        with torch.cuda.stream(s):
            seen = {k: t.clone() for k, t in dst.items()}
        s.synchronize()
        assert_pages(case, seen, case.expect(reqs[0][1], dms[0]), "after the last target layer's hook")
        eng2.wait(ticket)
    torch.cuda.synchronize()
    want = None
    for (t, sm), dm in zip(reqs, dms):
        want = case.expect(sm, dm, want)
    assert_pages(case, dst, want, mode)
    eng2.close()
    eng.close()
    pool.close()


@pytest.mark.parametrize("name", list(CASES))
def test_gather_device_tier_and_peer_pull(name):
    need_gpu()
    rng = np.random.default_rng(sum(map(ord, name)))
    case = Case(name, rng, 40, 16 if name.startswith("kv") else 64)
    g, C, n = case.geom, case.C, 600
    src = case.device()
    eng = KVEngine(g, None, 0, staging_bytes=0)
    eng.register_kv_caches(case.registered(src))
    sm, dm = slots(rng, case.NB, case.bs, n), slots(rng, case.NB, case.bs, n)
    n_chunks = (n + C - 1) // C
    # device-resident gather: chunk bytes
    buf = torch.zeros(n_chunks * g.chunk_bytes, dtype=torch.uint8, device="cuda:0")
    eng.gather(sm, buf.data_ptr())
    torch.cuda.synchronize()
    got = buf.cpu().numpy()
    for c in range(n_chunks):
        case.check_chunk(got[c * g.chunk_bytes:], sm[c * C:(c + 1) * C])
    # device tier: slots of the chunk size with the draft planes
    base = eng.tier_create(4)
    ptrs = [base + s * g.chunk_bytes for s in (2, 0, 3)]
    eng.gather_chunks(sm, ptrs)
    dst = case.device(zero=True)
    eng2 = KVEngine(g, None, 0, staging_bytes=0)
    eng2.register_kv_caches(case.registered(dst))
    eng2.scatter_chunks(dm, ptrs)
    torch.cuda.synchronize()
    assert_pages(case, dst, case.expect(sm, dm), "device tier")
    # same-process peer pull through the producer's plane pointers (descriptor order: one per plane, then indexer)
    local = case.device(zero=True)
    eng3 = KVEngine(g, None, 0, staging_bytes=0)
    eng3.register_kv_caches(case.registered(local))
    lat = [t for k, t in src.items() if "indexer" not in k]
    idx = [t for k, t in src.items() if "indexer" in k]
    if case.kind == "nhd":
        k_ptrs, v_ptrs = [t[0].data_ptr() for t in lat], [t[1].data_ptr() for t in lat]
    elif case.kind == "hnd":
        k_ptrs, v_ptrs = [t[:, 0].data_ptr() for t in lat], [t[:, 1].data_ptr() for t in lat]
    else:
        k_ptrs, v_ptrs = [t.data_ptr() for t in lat], ([t.data_ptr() for t in idx] if idx else None)
    eng3.import_peer_ptrs(1, 0, k_ptrs, v_ptrs)
    eng3.wait(eng3.peer_pull(1, sm, dm))
    torch.cuda.synchronize()
    # a pull copies verbatim: the source pages at sm land at dm in every plane, the draft layer's included
    want = [np.zeros_like(h) for h in case.host + case.idx]
    have = case.pages(src)
    for w_, h_ in zip(want, have):
        if w_.ndim == 5:                                  # K/V (2, NB, bs, H, D)
            w_.reshape(2, -1, H, HD)[:, dm] = h_.reshape(2, -1, H, HD)[:, sm]
        else:
            w_.reshape(-1, w_.shape[-1])[dm] = h_.reshape(-1, h_.shape[-1])[sm]
    if case.idx:       # indexer planes: a block is [bs][128] values then [bs][4] scales
        from tests import mla_sparse_oracle as so
        n_lat = len(case.host)
        want[n_lat:] = [np.zeros_like(h) for h in case.idx]
        so.scatter_slabs(want[n_lat:], so.gather_slabs(case.idx, sm, n), dm, n)
    assert_pages(case, local, want, "peer pull")
    for e in (eng3, eng2, eng):
        e.close()
