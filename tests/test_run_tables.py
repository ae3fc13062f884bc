"""Run tables (csrc/b200kv_runs.h) against the per-token rule they replace.

The header is host-only: it is compiled here with g++ behind a small extern "C" wrapper and called
through ctypes.  The reference below restates the per-token rule: token i extends the current run
when its slot follows the run's last slot, the slot does not start a vLLM block, the op-relative
index i - b_shift does not start a chunk and, for HND, does not start a tile; a pull run also needs
the destination slot to follow on and not start a block.  HND runs are split into whole aligned
tiles and the rest.  CPU only."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EINVAL = -22

WRAPPER = r"""
#include "b200kv_runs.h"
using b200kv::Run;

static void out(const std::vector<Run>& v, Run* dst, int64_t* n) {
  for (size_t i = 0; i < v.size(); ++i) dst[i] = v[i];
  *n = static_cast<int64_t>(v.size());
}

extern "C" int op_runs(const int64_t* slots, int64_t tok_begin, int64_t tok_end, int64_t b_shift, int64_t max_slot,
                       int32_t bs, int32_t C, int hnd, int split, Run* full, int64_t* n_full, Run* part,
                       int64_t* n_part) {
  std::vector<Run> f, p;
  const int rc = b200kv::build_runs(slots, tok_begin, tok_end, b_shift, max_slot, bs, C, hnd != 0, &f,
                                    split ? &p : nullptr);
  out(f, full, n_full);
  out(p, part, n_part);
  return rc;
}

extern "C" int op_table(const int64_t* slots, const int64_t* spans, int64_t n_spans, int64_t max_slot, int32_t bs,
                        int32_t C, int split, int hnd, Run* runs, int64_t* n_runs, uint32_t* full_off,
                        uint32_t* part_off) {
  std::vector<b200kv::Span> sp;
  for (int64_t i = 0; i < n_spans; ++i) sp.push_back({spans[2 * i], spans[2 * i + 1]});
  b200kv::OpTable t;
  const int rc = b200kv::build_op_table(slots, sp.data(), sp.size(), max_slot, bs, C, split != 0, hnd != 0, &t);
  out(t.runs, runs, n_runs);
  for (size_t i = 0; i < t.full_off.size(); ++i) full_off[i] = t.full_off[i];
  for (size_t i = 0; i < t.part_off.size(); ++i) part_off[i] = t.part_off[i];
  return rc;
}

extern "C" int table_layout(int64_t n_runs, int64_t n_chunks, uint64_t* l) {
  b200kv::TableLayout t;
  const int rc = b200kv::table_layout(static_cast<size_t>(n_runs), static_cast<size_t>(n_chunks), &t);
  l[0] = t.runs_off;
  l[1] = t.addrs_off;
  l[2] = t.offs_off;
  l[3] = t.bytes;
  return rc;
}

extern "C" int whole_block(const Run* runs, const uint32_t* full_off, int64_t n_chunks, int32_t bs, int32_t C) {
  b200kv::OpTable t;
  t.full_off.assign(full_off, full_off + n_chunks + 1);
  t.runs.assign(runs, runs + full_off[n_chunks]);
  return b200kv::whole_block_chunks(t, bs, C);
}

extern "C" int pull_runs(const int64_t* src, const int64_t* dst, int64_t n, int64_t max_src, int64_t max_dst,
                         int32_t bs, int hnd, Run* full, int64_t* n_full, Run* part, int64_t* n_part) {
  std::vector<Run> f, p;
  const int rc = b200kv::build_pull_runs(src, dst, n, max_src, max_dst, bs, hnd != 0, &f, &p);
  out(f, full, n_full);
  out(p, part, n_part);
  return rc;
}
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("runs")
    src, so = d / "runs_wrapper.cpp", d / "librunswrapper.so"
    src.write_text(WRAPPER)
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", "-shared", "-fPIC",
                    "-I", os.path.join(ROOT, "production-stack_b200", "csrc"), "-I", os.path.join(ROOT, "include"),
                    str(src), "-o", str(so)], check=True)
    return C.CDLL(str(so))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _call(fn, args, n):
    full, part = np.zeros((max(n, 1), 3), np.int32), np.zeros((max(n, 1), 3), np.int32)
    nf, npart = C.c_int64(-1), C.c_int64(-1)
    rc = fn(*args, _p(full), C.byref(nf), _p(part), C.byref(npart))
    if rc:
        return rc, None, None
    return rc, [tuple(r) for r in full[:nf.value]], [tuple(r) for r in part[:npart.value]]


def build(lib, slots, tb, te, b_shift, max_slot, bs, c, hnd, split=True):
    slots = np.ascontiguousarray(slots, np.int64)
    args = (_p(slots), C.c_int64(tb), C.c_int64(te), C.c_int64(b_shift), C.c_int64(max_slot), C.c_int32(bs),
            C.c_int32(c), C.c_int(hnd), C.c_int(split))
    return _call(lib.op_runs, args, te - tb)


def build_pull(lib, src, dst, max_src, max_dst, bs, hnd):
    src, dst = np.ascontiguousarray(src, np.int64), np.ascontiguousarray(dst, np.int64)
    args = (_p(src), _p(dst), C.c_int64(len(src)), C.c_int64(max_src), C.c_int64(max_dst), C.c_int32(bs), C.c_int(hnd))
    return _call(lib.pull_runs, args, len(src))


def _sink(bs, hnd, split):
    full, part = [], []

    def push(r):
        a, b, n = r
        whole = n == bs and a % bs == 0 and b % bs == 0
        (part if hnd and split and not whole else full).append(r)
    return full, part, push


def ref(slots, tb, te, b_shift, max_slot, bs, c, hnd, split=True):
    full, part, push = _sink(bs, hnd, split)
    cur = None
    for i in range(tb, te):
        s, j = int(slots[i]), i - b_shift
        if s < 0 or s >= max_slot:
            return EINVAL, None, None
        if (cur and s == cur[0] + cur[2] and s % bs and j % c and not (hnd and j % bs == 0)):
            cur[2] += 1
        else:
            if cur:
                push(tuple(cur))
            cur = [s, j, 1]
    if cur:
        push(tuple(cur))
    return 0, full, part


def ref_pull(src, dst, max_src, max_dst, bs, hnd):
    full, part, push = _sink(bs, hnd, True)
    cur = None
    for s, d in zip(map(int, src), map(int, dst)):
        if not (0 <= s < max_src and 0 <= d < max_dst):
            return EINVAL, None, None
        if cur and s == cur[0] + cur[2] and d == cur[1] + cur[2] and s % bs and d % bs:
            cur[2] += 1
        else:
            if cur:
                push(tuple(cur))
            cur = [s, d, 1]
    if cur:
        push(tuple(cur))
    return 0, full, part


def block_map(blocks, n_tok, bs, start=0):
    """vLLM slot mapping of tokens [start, start + n_tok) of a request with block table `blocks`."""
    i = np.arange(start, start + n_tok, dtype=np.int64)
    return np.asarray(blocks, np.int64)[i // bs] * bs + i % bs


def random_map(rng, n_tok, nb, bs):
    """A map made of pieces of every shape the builders meet: block tables entered mid-block, single
    tokens, runs of consecutive slots that cross block boundaries, and repeated slots."""
    parts, left = [], n_tok
    while left > 0:
        k = int(rng.integers(1, min(left, 3 * bs) + 1))
        kind = rng.integers(0, 4)
        if kind == 0:
            blocks = rng.permutation(nb)[:(k + 2 * bs) // bs + 1]
            parts.append(block_map(blocks, k, bs, start=int(rng.integers(0, bs))))
        elif kind == 1:
            parts.append(rng.integers(0, nb * bs, k))
        elif kind == 2:
            s0 = int(rng.integers(0, nb * bs - k))
            parts.append(np.arange(s0, s0 + k))
        else:
            parts.append(np.full(k, rng.integers(0, nb * bs)))
        left -= k
    return np.concatenate(parts).astype(np.int64)


# (bs, C): geometries make_geometry accepts, plus one whose chunk is not a whole number of blocks
# (make_geometry refuses it today; the HND tile rule must still follow the op-relative index)
GEOMS = [(16, 256), (16, 64), (8, 32), (16, 16), (16, 40)]


@pytest.mark.parametrize("hnd", [False, True])
@pytest.mark.parametrize("bs,c", GEOMS)
def test_random_maps_match_the_per_token_rule(lib, bs, c, hnd):
    rng = np.random.default_rng(bs * 1000 + c + hnd)
    nb = 64
    for _ in range(150):
        n = int(rng.integers(1, 5 * c))
        slots = random_map(rng, n, nb, bs)
        tb = int(rng.integers(0, n))
        te = int(rng.integers(tb + 1, n + 1))
        b_shift = int(rng.integers(-c, tb + 1))          # op-relative indices stay >= 0, as in the engine
        for split in (True, False):
            want = ref(slots, tb, te, b_shift, nb * bs, bs, c, hnd, split)
            assert build(lib, slots, tb, te, b_shift, nb * bs, bs, c, hnd, split) == want


@pytest.mark.parametrize("hnd", [False, True])
def test_batch_of_ragged_requests_matches_the_per_token_rule(lib, hnd):
    """Store / load batches: chunk k of the op holds the k-th chunk's slots at k*C, a request's last
    chunk is short, and chunk i of a staging batch is indexed from i*C (b_shift = k*C - i*C)."""
    bs, c, nb = 16, 64, 256
    rng = np.random.default_rng(7 + hnd)
    perm = rng.permutation(nb)
    sm, ntok, used = [], [], 0
    for n_req in (c + 5, 2 * c, 3 * c + 1, 17, c):
        nblk = (n_req + bs - 1) // bs
        req = block_map(perm[used:used + nblk], n_req, bs)
        used += nblk
        for k in range(0, n_req, c):
            t = req[k:k + c]
            sm.append(np.concatenate([t, np.full(c - len(t), -1)]))
            ntok.append(len(t))
    sm = np.concatenate(sm)
    for stage in (1, 3, len(ntok)):                      # staging batches of several sizes
        for b0 in range(0, len(ntok), stage):
            for i, k in enumerate(range(b0, min(b0 + stage, len(ntok)))):
                tb = k * c
                args = (sm, tb, tb + ntok[k], tb - i * c, nb * bs, bs, c, hnd)
                got = build(lib, *args)
                assert got[0] == 0 and got == ref(*args)


@pytest.mark.parametrize("hnd", [False, True])
def test_token_granular_and_shuffled_maps(lib, hnd):
    bs, c, nb = 16, 256, 512
    rng = np.random.default_rng(11)
    tokens = rng.permutation(nb * bs)[:3000]                          # every token its own slot
    shuffled = block_map(rng.permutation(nb)[:200], 3000, bs)         # whole blocks in random order
    mid = block_map(rng.permutation(nb)[:200], 3000, bs, start=5)     # a request entered mid-block
    for slots in (tokens, shuffled, mid):
        for b_shift in (0, -3, 7):
            tb = max(b_shift, 0)
            args = (slots, tb, len(slots), b_shift, nb * bs, bs, c, hnd)
            got = build(lib, *args)
            assert got[0] == 0 and got == ref(*args)


@pytest.mark.parametrize("hnd", [False, True])
def test_pull_runs_check_both_sides(lib, hnd):
    bs, nb_src, nb_dst = 16, 48, 64
    rng = np.random.default_rng(3 + hnd)
    for _ in range(200):
        n = int(rng.integers(1, 300))
        src = random_map(rng, n, nb_src, bs)
        dst = random_map(rng, n, nb_dst, bs) if rng.integers(0, 2) else \
            block_map(rng.permutation(nb_dst), n, bs, start=int(rng.integers(0, bs)))
        got = build_pull(lib, src, dst, nb_src * bs, nb_dst * bs, bs, hnd)
        assert got[0] == 0 and got == ref_pull(src, dst, nb_src * bs, nb_dst * bs, bs, hnd)
    # the source side follows on but the destination does not (and the other way round)
    src = np.arange(32, dtype=np.int64)
    dst = np.concatenate([np.arange(100, 108), np.arange(200, 224)]).astype(np.int64)
    for a, b in ((src, dst), (dst, src)):
        got = build_pull(lib, a, b, 4096, 4096, bs, hnd)
        assert got[0] == 0 and got == ref_pull(a, b, 4096, 4096, bs, hnd)


@pytest.mark.parametrize("bad", [-1, "max"])
@pytest.mark.parametrize("where", [0, "mid", "last"])
def test_out_of_range_slots_are_refused(lib, bad, where):
    bs, c, nb = 16, 64, 32
    max_slot = nb * bs
    slots = block_map(np.arange(nb), 200, bs)
    pos = {0: 0, "mid": 100, "last": 199}[where]
    slots[pos] = max_slot if bad == "max" else -1
    for hnd in (False, True):
        assert build(lib, slots, 0, 200, 0, max_slot, bs, c, hnd)[0] == EINVAL
    ok = block_map(np.arange(nb), 200, bs)
    assert build_pull(lib, slots, ok, max_slot, max_slot, bs, False)[0] == EINVAL
    assert build_pull(lib, ok, slots, max_slot, max_slot, bs, False)[0] == EINVAL
    # each side is checked against its own bound: slot 199 is past a bound of 199 on either side
    assert build_pull(lib, ok, ok, 199, max_slot, bs, False)[0] == EINVAL
    assert build_pull(lib, ok, ok, max_slot, 199, bs, False)[0] == EINVAL
    assert build_pull(lib, ok, ok, 200, 200, bs, False)[0] == 0
    for hnd in (False, True):       # a bound that is not a whole number of blocks
        assert build(lib, ok, 0, 200, 0, 199, bs, c, hnd)[0] == EINVAL
        assert build(lib, ok, 0, 199, 0, 199, bs, c, hnd) == ref(ok, 0, 199, 0, 199, bs, c, hnd)
    # slots that keep counting up past the bound: the first one past it starts a run of its own
    up = np.arange(max_slot - 20, max_slot + 5, dtype=np.int64)
    for hnd in (False, True):
        assert build(lib, up, 0, len(up), 0, max_slot, bs, c, hnd)[0] == EINVAL
        assert build(lib, up, 0, 20, 0, max_slot, bs, c, hnd) == ref(up, 0, 20, 0, max_slot, bs, c, hnd)
    assert build_pull(lib, up, up - 100, max_slot, max_slot, bs, False)[0] == EINVAL
    assert build_pull(lib, up - 100, up, max_slot, max_slot, bs, False)[0] == EINVAL
    # tokens outside [tok_begin, tok_end) are not read
    if where == "last":
        assert build(lib, slots, 0, 199, 0, max_slot, bs, c, False)[0] == 0


def test_bench_shape_gives_one_run_per_block(lib):
    """The device-resident step of bench.py: 16 sessions x 2048 tokens over shuffled 16-token blocks."""
    bs, c, nb, n = 16, 256, 8192, 16 * 2048
    perm = np.random.default_rng(1234).permutation(nb)
    slots = np.concatenate([block_map(perm[s * 128:(s + 1) * 128], 2048, bs) for s in range(16)])
    rc, full, part = build(lib, slots, 0, n, 0, nb * bs, bs, c, False)
    assert rc == 0 and part == [] and len(full) == 2048
    assert all(r[2] == 16 for r in full)
    assert [r[1] for r in full] == list(range(0, n, 16))
    assert [r[0] for r in full] == [int(slots[i]) for i in range(0, n, 16)]


def build_table(lib, slots, spans, max_slot, bs, c, split, hnd):
    slots = np.ascontiguousarray(slots, np.int64)
    sp = np.ascontiguousarray(np.asarray(spans, np.int64).reshape(-1, 2))
    n_tok = int(sp[:, 1].sum())
    runs = np.zeros((max(n_tok, 1), 3), np.int32)
    full_off, part_off = np.zeros(len(sp) + 1, np.uint32), np.zeros(len(sp) + 1, np.uint32)
    n = C.c_int64(-1)
    rc = lib.op_table(_p(slots), _p(sp), C.c_int64(len(sp)), C.c_int64(max_slot), C.c_int32(bs), C.c_int32(c),
                      C.c_int(split), C.c_int(hnd), _p(runs), C.byref(n), _p(full_off), _p(part_off))
    if rc:
        return rc, None, None, None
    return rc, [tuple(r) for r in runs[:n.value]], list(map(int, full_off)), list(map(int, part_off))


def ref_table(slots, spans, max_slot, bs, c, split, hnd):
    """Each span's runs from the per-token rule, chunk i indexed from i*C, regrouped: every chunk's full
    runs, chunk by chunk, then every chunk's partial runs."""
    full, part, full_off, part_off = [], [], [0], [0]
    for i, (tb, n) in enumerate(spans):
        rc, f, p = ref(slots, tb, tb + n, tb - i * c, max_slot, bs, c, hnd, split)
        if rc:
            return rc, None, None, None
        full += f
        part += p
        full_off.append(len(full))
        part_off.append(len(part))
    return 0, full + part, full_off, part_off


@pytest.mark.parametrize("hnd", [False, True])
@pytest.mark.parametrize("bs,c", GEOMS)
def test_op_table_regroups_the_runs_of_ragged_spans(lib, bs, c, hnd):
    """Store / load batches: any chunks of the op, each 1..C tokens, laid out as chunks 0, 1, ... of one table."""
    rng = np.random.default_rng(500 + bs * 100 + c + hnd)
    nb = 64
    for _ in range(60):
        n_op = int(rng.integers(1, 9))                      # chunks of the op, C slots apart
        slots = random_map(rng, n_op * c, nb, bs)
        picked = sorted(rng.choice(n_op, int(rng.integers(1, n_op + 1)), replace=False))
        spans = [(int(k) * c, int(rng.integers(1, c + 1))) for k in picked]
        for split in (True, False):
            want = ref_table(slots, spans, nb * bs, bs, c, split, hnd)
            assert want[0] == 0
            assert build_table(lib, slots, spans, nb * bs, bs, c, split, hnd) == want
    slots[0] = nb * bs                                       # a slot out of range refuses the table
    assert build_table(lib, slots, [(0, 1)], nb * bs, bs, c, True, hnd)[0] == EINVAL


@pytest.mark.parametrize("hnd", [False, True])
@pytest.mark.parametrize("bs,c", GEOMS)
def test_gather_spans_give_the_whole_op_runs(lib, bs, c, hnd):
    """Gather / scatter: spans [k*C, min((k+1)*C, n)) give exactly the runs of one build over the whole op, and,
    for the FP8 / Q4 table (no split), full_off is where each chunk's runs start by their op-relative index."""
    rng = np.random.default_rng(900 + bs * 100 + c + hnd)
    nb = 64
    for _ in range(60):
        n = int(rng.integers(1, 6 * c))
        slots = random_map(rng, n, nb, bs)
        spans = [(k, min(c, n - k)) for k in range(0, n, c)]
        for split in (True, False):
            rc, full, part = build(lib, slots, 0, n, 0, nb * bs, bs, c, hnd, split)
            got = build_table(lib, slots, spans, nb * bs, bs, c, split, hnd)
            assert rc == 0 and got[0] == 0 and got[1] == full + part
            if not split:
                offs, r = [], 0
                for k in range(len(spans)):
                    offs.append(r)
                    while r < len(full) and full[r][1] // c == k:
                        r += 1
                offs.append(r)
                assert got[2] == offs


def test_table_layout_and_its_cap(lib):
    def layout(n_runs, n_chunks):
        out = np.zeros(4, np.uint64)
        rc = lib.table_layout(C.c_int64(n_runs), C.c_int64(n_chunks), _p(out))
        return rc, list(map(int, out))

    def up16(x):
        return (x + 15) // 16 * 16

    for n_runs in (0, 1, 2, 5, 2048, 87378):
        for n_chunks in (1, 2, 3, 7, 128, 1000):
            runs, addrs, offs = up16(12 * n_runs), up16(8 * n_chunks), up16(4 * (n_chunks + 1))
            total = runs + addrs + offs
            assert layout(n_runs, n_chunks) == ((0 if total <= 1 << 20 else EINVAL), [0, runs, runs + addrs, total])
    assert layout(87378, 1) == (0, [0, 1048544, 1048560, 1 << 20])      # one chunk: exactly 1 MiB
    assert layout(87379, 1)[0] == EINVAL


def whole_block(lib, runs, full_off, bs, c):
    runs = np.ascontiguousarray(np.asarray(runs, np.int32).reshape(-1, 3))
    off = np.ascontiguousarray(full_off, np.uint32)
    return bool(lib.whole_block(_p(runs), _p(off), C.c_int64(len(off) - 1), C.c_int32(bs), C.c_int32(c)))


def ref_whole_block(runs, full_off, bs, c):
    """Chunk k's runs are its paged blocks in order: run j starts at op-relative token k*C + j*bs and at a block's
    first slot, and holds bs tokens, or the chunk's remaining tokens if it is the last run."""
    for k in range(len(full_off) - 1):
        rs = runs[full_off[k]:full_off[k + 1]]
        n = sum(r[2] for r in rs)
        if n == 0 or n > c or len(rs) != -(-n // bs):
            return False
        for j, (a, b, m) in enumerate(rs):
            if b != k * c + j * bs or a % bs or m != min(bs, n - j * bs):
                return False
    return True


def fp8_table(lib, slots, spans, nb, bs, c, hnd):
    """The table an FP8 op builds (no partial-tile split)."""
    rc, runs, full_off, _ = build_table(lib, slots, spans, nb * bs, bs, c, False, hnd)
    assert rc == 0
    return runs, full_off


@pytest.mark.parametrize("hnd", [False, True])
@pytest.mark.parametrize("bs,c", [(16, 256), (16, 64), (8, 32), (16, 16)])
def test_whole_block_chunks_accepts_block_tables(lib, bs, c, hnd):
    """Batches of requests over block tables: every request's last chunk is short and may end mid-block, and
    the next request's chunks follow it in the same table."""
    nb = 512
    rng = np.random.default_rng(40 + bs + c + hnd)
    perm = rng.permutation(nb)
    sm, spans, used = [], [], 0
    for n_req in (c + 5, 2 * c, 3 * c + 1, bs + 3, c, 1, 2 * c - 1):
        nblk = (n_req + bs - 1) // bs
        req = block_map(perm[used:used + nblk], n_req, bs)
        used += nblk
        for k in range(0, n_req, c):
            t = req[k:k + c]
            spans.append((len(sm) * c, len(t)))
            sm.append(np.concatenate([t, np.zeros(c - len(t), np.int64)]))
    sm = np.concatenate(sm)
    runs, full_off = fp8_table(lib, sm, spans, nb, bs, c, hnd)
    assert any(n % bs for _, n in spans) and any(n < c for _, n in spans[:-1])
    assert ref_whole_block(runs, full_off, bs, c)
    assert whole_block(lib, runs, full_off, bs, c)
    # gather-shaped: one request, chunks [k*C, (k+1)*C) of the op
    n = 5 * c + bs // 2
    slots = block_map(rng.permutation(nb)[:(n + bs - 1) // bs], n, bs)
    runs, full_off = fp8_table(lib, slots, [(k, min(c, n - k)) for k in range(0, n, c)], nb, bs, c, hnd)
    assert whole_block(lib, runs, full_off, bs, c)


@pytest.mark.parametrize("hnd", [False, True])
def test_whole_block_chunks_refuses_other_tables(lib, hnd):
    bs, c, nb = 16, 64, 256
    rng = np.random.default_rng(77 + hnd)
    n = 3 * c
    token_granular = rng.permutation(nb * bs)[:n]
    mid_block = block_map(rng.permutation(nb)[:20], n, bs, start=5)        # a request entered mid-block
    for slots in (token_granular, mid_block):
        runs, full_off = fp8_table(lib, slots, [(k, c) for k in range(0, n, c)], nb, bs, c, hnd)
        assert not ref_whole_block(runs, full_off, bs, c)
        assert not whole_block(lib, runs, full_off, bs, c)
    good = [(0, 0, 16), (32, 16, 16), (64, 32, 5)]                           # one chunk of 37 tokens
    assert whole_block(lib, good, [0, 3], bs, c)
    for bad in ([(0, 0, 16), (32, 16, 8), (64, 24, 13)],                     # a short run that is not the last
                [(0, 0, 16), (32, 32, 16), (64, 48, 5)],                     # run 1 skips block position 1
                [(0, 0, 16), (36, 16, 16), (64, 32, 5)],                     # run 1 starts mid-block
                [(0, 0, 16), (32, 16, 16), (64, 32, 5), (80, 37, 1)]):       # more runs than blocks
        assert not ref_whole_block(bad, [0, len(bad)], bs, c)
        assert not whole_block(lib, bad, [0, len(bad)], bs, c)
    assert not whole_block(lib, good + [(96, 64, 16)], [0, 3, 3], bs, c)     # an empty chunk
    assert whole_block(lib, good + [(96, 64, 16)], [0, 3, 4], bs, c)         # chunk 1 at token C


@pytest.mark.parametrize("hnd", [False, True])
def test_whole_block_chunks_matches_its_restatement(lib, hnd):
    bs, c, nb = 16, 64, 64
    rng = np.random.default_rng(300 + hnd)
    seen = set()
    for _ in range(300):
        n_op = int(rng.integers(1, 6))
        if rng.integers(0, 2):
            slots = random_map(rng, n_op * c, nb, bs)
        else:
            start = int(rng.integers(0, bs)) if rng.integers(0, 2) else 0
            slots = block_map(rng.permutation(nb), n_op * c, bs, start=start)
        spans = [(k * c, int(rng.integers(1, c + 1))) for k in range(n_op)]
        runs, full_off = fp8_table(lib, slots, spans, nb, bs, c, hnd)
        want = ref_whole_block(runs, full_off, bs, c)
        seen.add(want)
        assert whole_block(lib, runs, full_off, bs, c) == want
    assert seen == {False, True}
