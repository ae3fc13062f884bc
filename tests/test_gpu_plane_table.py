"""The plane pointers of MLA engines on an H100 (-m gpu), plain and with DeepSeek-V3.2's indexer planes: a same-process
pull through b200kv_import_peer_ptrs is bit-exact against the oracles, and every malformed pointer set is refused
by registration and by the import alike, leaving the engine unregistered and the peer id free."""
import ctypes

import numpy as np
import pytest

from tests import test_gpu_mla as tm
from tests import test_gpu_mla_sparse as ts

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

from b200kv import FMT_RAW, KVEngine, _lib  # noqa: E402
from b200kv._lib import B200KVError  # noqa: E402

D = 576


def planes(indexed, rng, L, NB, bs):
    """(geometry, host latent pages, host indexer pages or None, device caches, latent ptrs, indexer ptrs or None)."""
    if indexed:
        lat, idx = ts.mk_host(rng, L, NB, bs)
        caches = ts.to_dev(lat, idx)
        k = [t.data_ptr() for n, t in caches.items() if "indexer" not in n]
        v = [t.data_ptr() for n, t in caches.items() if "indexer" in n]
        return ts.geom(L, NB, bs), lat, idx, caches, k, v
    lat = tm.mk_layers(rng, L, NB, bs)
    caches = tm.to_dev(lat)
    return tm.geom(L, NB, bs), lat, None, caches, [t.data_ptr() for t in caches], None


def ptr_array(ptrs):
    return None if ptrs is None else (ctypes.c_void_p * len(ptrs))(*[ctypes.c_void_p(p) for p in ptrs])


@pytest.mark.parametrize("indexed", [False, True])
def test_pull_through_import_peer_ptrs(indexed):
    tm.need_gpu()
    rng = np.random.default_rng(31 + indexed)
    L, NB, bs, C, n_tok = 3, 48, 64, 256, 1000
    g, lat, idx, remote, k, v = planes(indexed, rng, L, NB, bs)
    zl = [np.zeros_like(a) for a in lat]
    if indexed:
        zi = [np.zeros_like(b) for b in idx]
        local = ts.to_dev(zl, zi)
    else:
        local = tm.to_dev(zl)
    eng = KVEngine(g, None, 0, staging_bytes=0)
    eng.register_kv_caches(local)
    eng.import_peer_ptrs(1, 0, k, v)
    src, dst = ts.mapping(rng, NB, bs, n_tok), ts.mapping(rng, NB, bs, n_tok, "tokens")
    eng.wait(eng.peer_pull(1, src, dst))
    torch.cuda.synchronize()
    if indexed:
        el, ei = ts.expected_pages(FMT_RAW, lat, idx, src, dst, C, zl, zi)
        hl, hi = ts.host_of(local)
        got, want, per_tok = hl + hi, el + ei, L * (D * 2 + 132)
    else:
        got = [tm.host_of(t) for t in local]
        want, per_tok = tm._expected_pages(FMT_RAW, lat, src, dst, C, zl), L * D * 2
    for a, e in zip(got, want):
        assert np.array_equal(a, e)
    assert eng.stats()["p2p_bytes"] == n_tok * per_tok
    eng.close()


# (indexed engine, the valid (k_ptrs, v_ptrs) -> the refused ones)
FAULTS = {
    "indexed-v-null": (True, lambda k, v: (k, None)),
    "plain-v-set": (False, lambda k, v: (k, k)),
    "latent-misaligned": (True, lambda k, v: ([k[0] + 8] + k[1:], v)),
    "indexer-misaligned": (True, lambda k, v: (k, v[:-1] + [v[-1] + 4])),
    "latent-null": (False, lambda k, v: (k[:1] + [0] + k[2:], v)),
    "indexer-null": (True, lambda k, v: (k, [0] + v[1:])),
}


@pytest.mark.parametrize("fault", list(FAULTS))
def test_refused_plane_pointers(fault):
    tm.need_gpu()
    indexed, bend = FAULTS[fault]
    L, NB, bs = 3, 8, 64
    g, _, _, _caches, k, v = planes(indexed, np.random.default_rng(4), L, NB, bs)   # _caches: the planes' storage
    bk, bv = bend(k, v)
    lib = _lib.lib()
    eng = KVEngine(g, None, 0, staging_bytes=0)

    def planes_exported():
        """(offset, allocation size) of every exported descriptor: which plane each one points at."""
        return [(d.offset, d.alloc_bytes) for d in (_lib.IpcDesc * g.n_descs).from_buffer_copy(eng.export_ipc())]

    assert lib.b200kv_register_kv(eng._h, ptr_array(bk), ptr_array(bv)) == _lib.EINVAL
    descs = (_lib.IpcDesc * g.n_descs)()
    assert lib.b200kv_export_ipc(eng._h, descs, g.n_descs) == _lib.EINVAL      # still unregistered
    assert lib.b200kv_import_peer_ptrs(eng._h, 1, 0, ptr_array(bk), ptr_array(bv), g.stride, NB) == _lib.EINVAL
    with pytest.raises(B200KVError) as e:
        eng.peer_pull(1, [0], [0])
    assert e.value.code == _lib.ENOENT                                           # no peer was installed
    # the valid pointers register and import; a refused re-registration keeps the registration it had
    eng.register_kv_ptrs(k, v)
    before = planes_exported()
    assert lib.b200kv_register_kv(eng._h, ptr_array(bk), ptr_array(bv)) == _lib.EINVAL
    assert planes_exported() == before
    eng.import_peer_ptrs(1, 0, k, v)
    eng.wait(eng.peer_pull(1, np.arange(bs), np.arange(bs) + bs))
    eng.close()
