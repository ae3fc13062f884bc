// b200kv_runs.h — run tables of the copy kernels, built on the host.
//
// Host-only (no CUDA header): the engine includes it through b200kv_kernels.cuh, and plain g++
// compiles it for the equivalence test (tests/test_run_tables.py).
//
// A run is a stretch of consecutive tokens that the kernels move as one contiguous byte range on
// each side.  The builders read the map once: at a run's first token they range-check its slot and
// compute the run's limit, then extend the run while the slots stay consecutive.  The limit keeps
// a run's slots below the bound its first slot was checked against, so checking the first slot of
// each run checks every slot of the map.
#pragma once

#include <stdint.h>

#include <algorithm>
#include <vector>

#include "b200kv.h"

namespace b200kv {

// One run = consecutive tokens that stay inside one vLLM block and one chunk.
//   store / load : a = paged slot (block*bs + off) ; b = op-relative token index
//   peer pull    : a = peer slot                   ; b = local slot
struct Run {
  int32_t a;
  int32_t b;
  int32_t n;
};

// true if slot s lies outside [0, bound)
inline bool out_of_range(int64_t s, int64_t bound) {
  return static_cast<uint64_t>(s) >= static_cast<uint64_t>(bound);
}

// length of the run of p[0, lim) that continues p[0] == s as s, s+1, s+2, ... (lim >= 1).  A whole
// block of a block table is the common case: it is recognised with one branch-free pass of subtracts
// and ORs over the window (which vectorises) before the scalar scan that finds where a run ends.
inline int64_t consecutive(const int64_t* p, int64_t s, int64_t lim) {
  if (lim == 1 || p[1] != s + 1) return 1;
  uint64_t diff = 0;
  for (int64_t k = 2; k < lim; ++k) diff |= static_cast<uint64_t>(p[k]) - static_cast<uint64_t>(s) - k;
  if (diff == 0) return lim;
  int64_t n = 2;
  while (p[n] == s + n) ++n;   // ends before lim: some slot of the window differs
  return n;
}

// tokens from x up to (excluding) the next multiple of m above x
inline int64_t tokens_to_boundary(int64_t x, int64_t m) {
  const int64_t r = x % m;
  return r < 0 ? -r : m - r;
}

// HND tiles: `full` takes runs that are one whole aligned block on both sides (a contiguous tile,
// moved by the bulk kernel exactly like NHD), `partial` the rest (moved per head by
// kv_hnd_partial_kernel).  NHD, or no `partial` list (the FP8 / Q4 kernels take one sorted list):
// everything goes to `full`.
inline void push_run(const Run& r, int32_t bs, bool hnd, std::vector<Run>* full, std::vector<Run>* partial) {
  if (!hnd || !partial) { full->push_back(r); return; }
  const bool whole = r.n == bs && (r.a % bs) == 0 && (r.b % bs) == 0;
  (whole ? full : partial)->push_back(r);
}

// Runs of slots[tok_begin, tok_end) (vllm_v1_adapter.py:368-375) for a store / load.  Token i has
// op-relative index i - b_shift.  A run never crosses a vLLM block on the slot side or a chunk (C
// tokens) on the op side; for HND it also stops at every op-side tile (bs tokens) boundary.  Returns
// B200KV_EINVAL if a slot lies outside [0, max_slot); the lists then hold an unspecified prefix.
inline int build_runs(const int64_t* slots, int64_t tok_begin, int64_t tok_end, int64_t b_shift, int64_t max_slot,
                      int32_t bs, int32_t C, bool hnd, std::vector<Run>* full, std::vector<Run>* partial) {
  // room left in the current chunk and tile on the op side; a run ends at or before both, so
  // subtracting its length and wrapping at zero keeps them exact
  int64_t chunk_room = tokens_to_boundary(tok_begin - b_shift, C);
  int64_t tile_room = tokens_to_boundary(tok_begin - b_shift, bs);
  for (int64_t i = tok_begin; i < tok_end;) {
    const int64_t s = slots[i];
    if (out_of_range(s, max_slot)) return B200KV_EINVAL;
    int64_t lim = std::min({static_cast<int64_t>(bs) - s % bs, max_slot - s, chunk_room, tok_end - i});
    if (hnd) lim = std::min(lim, tile_room);
    const int64_t n = consecutive(slots + i, s, lim);
    push_run(Run{static_cast<int32_t>(s), static_cast<int32_t>(i - b_shift), static_cast<int32_t>(n)}, bs, hnd,
             full, partial);
    i += n;
    chunk_room -= n;
    if (chunk_room == 0) chunk_room = C;
    if (hnd && (tile_room -= n) == 0) tile_room = bs;
  }
  return B200KV_OK;
}

// Runs of a peer pull: token i moves peer slot src[i] to local slot dst[i].  A run never crosses a
// vLLM block on either side.  Returns B200KV_EINVAL if a source slot lies outside [0, max_src) or a
// destination slot outside [0, max_dst); the lists then hold an unspecified prefix.
inline int build_pull_runs(const int64_t* src, const int64_t* dst, int64_t n_tokens, int64_t max_src,
                           int64_t max_dst, int32_t bs, bool hnd, std::vector<Run>* full,
                           std::vector<Run>* partial) {
  for (int64_t i = 0; i < n_tokens;) {
    const int64_t s = src[i], d = dst[i];
    if (out_of_range(s, max_src) || out_of_range(d, max_dst)) return B200KV_EINVAL;
    const int64_t lim = std::min({static_cast<int64_t>(bs) - s % bs, static_cast<int64_t>(bs) - d % bs, max_src - s,
                                  max_dst - d, n_tokens - i});
    int64_t n = 1;
    while (n < lim && src[i + n] == s + n && dst[i + n] == d + n) ++n;
    push_run(Run{static_cast<int32_t>(s), static_cast<int32_t>(d), static_cast<int32_t>(n)}, bs, hnd, full, partial);
    i += n;
  }
  return B200KV_OK;
}

// The run table of one op: the full runs of every chunk, chunk by chunk, then the partial runs of every
// chunk, chunk by chunk.  Chunk i's full runs are runs[full_off[i], full_off[i+1]) and its partial runs
// runs[n_full() + part_off[i], n_full() + part_off[i+1]).
struct OpTable {
  std::vector<Run> runs;
  std::vector<uint32_t> full_off{0};
  std::vector<uint32_t> part_off{0};
  uint32_t n_chunks() const { return static_cast<uint32_t>(full_off.size() - 1); }
  uint32_t n_full() const { return full_off.back(); }
};

// Chunk i of a table holds slots[tok_begin, tok_begin + n_tok) and starts at op-relative index i*C.
struct Span {
  int64_t tok_begin;
  int64_t n_tok;
};

// The table of an op over `spans`.  `split` (RAW) keeps HND partial-tile runs apart; without it every
// run is a full run.  Returns B200KV_EINVAL if a slot lies outside [0, max_slot).
inline int build_op_table(const int64_t* slots, const Span* spans, size_t n_spans, int64_t max_slot, int32_t bs,
                          int32_t C, bool split, bool hnd, OpTable* t) {
  *t = OpTable();
  std::vector<Run> partial;
  for (size_t i = 0; i < n_spans; ++i) {
    const int64_t tb = spans[i].tok_begin;
    const int rc = build_runs(slots, tb, tb + spans[i].n_tok, tb - static_cast<int64_t>(i) * C, max_slot, bs, C,
                              hnd, &t->runs, split ? &partial : nullptr);
    if (rc) return rc;
    t->full_off.push_back(static_cast<uint32_t>(t->runs.size()));
    t->part_off.push_back(static_cast<uint32_t>(partial.size()));
  }
  t->runs.insert(t->runs.end(), partial.begin(), partial.end());
  return B200KV_OK;
}

// True if every chunk of `t` is a sequence of whole, block-aligned runs, only the last one possibly short: run j
// of chunk c starts at op-relative token c*C + j*bs and at the first slot of a block.  Any vLLM block table gives
// such a table; the persistent FP8 store (kv_fp8_store3_kernel) takes no other.  Reads the full runs only.
inline bool whole_block_chunks(const OpTable& t, int32_t bs, int32_t C) {
  const uint32_t ubs = static_cast<uint32_t>(bs), uc = static_cast<uint32_t>(C);
  for (uint32_t c = 0; c < t.n_chunks(); ++c) {
    const uint32_t r0 = t.full_off[c], r1 = t.full_off[c + 1];
    uint32_t n_valid = 0;   // the chunk's tokens: its runs cover them
    for (uint32_t r = r0; r < r1; ++r) n_valid += static_cast<uint32_t>(t.runs[r].n);
    if (n_valid == 0 || n_valid > uc) return false;
    const uint32_t nb = (n_valid + ubs - 1) / ubs;
    if (r1 - r0 != nb) return false;
    for (uint32_t j = 0; j < nb; ++j) {
      const Run& run = t.runs[r0 + j];
      if (run.b != static_cast<int32_t>(c * uc + j * ubs) || static_cast<uint32_t>(run.a) % ubs != 0 ||
          static_cast<uint32_t>(run.n) != std::min(ubs, n_valid - j * ubs))
        return false;
    }
  }
  return true;
}

// ---- split tiles: the indexer key cache of DeepSeek-V3.2's sparse attention (b200kv_set_indexer) -----------------
// vLLM's indexer_k_quant_and_cache writes a block of bs tokens as [bs][vb] values followed by [bs][sb] scales (one
// fp32 per token), so a tile is not token-major.  A chunk's indexer slab of one layer mirrors the tile: [C][vb]
// values, then [C][sb] scales.  A run (consecutive tokens inside one block and one chunk) is therefore two
// contiguous pieces on each side, n*vb value bytes and n*sb scale bytes.  These helpers give the pieces of a run as
// offsets: relative to the plane's block 0 on a page side, to the layer's indexer slab of the run's chunk on the
// chunk side.  kv_indexer_copy_kernel calls the same code on the device.
#if defined(__CUDACC__)
#define B200KV_HD __host__ __device__ __forceinline__
#else
#define B200KV_HD inline
#endif

struct SplitTile {
  uint32_t bs, C, vb, sb;
  uint64_t a_stride;   // block stride of the pages at slot run.a: the local pages of a store / load, a pull's source
  uint64_t b_stride;   // a pull: block stride of the destination pages at slot run.b
};

struct SplitPiece {
  uint64_t src, dst;
  uint32_t bytes;
};

// value and scale offsets of slot `slot` inside pages of block stride `stride`
B200KV_HD void split_page_offsets(const SplitTile& t, uint64_t stride, uint32_t slot, uint64_t* v, uint64_t* s) {
  const uint32_t blk = slot / t.bs, off = slot - blk * t.bs;
  const uint64_t b = static_cast<uint64_t>(blk) * stride;
  *v = b + static_cast<uint64_t>(off) * t.vb;
  *s = b + static_cast<uint64_t>(t.bs) * t.vb + static_cast<uint64_t>(off) * t.sb;
}

// value and scale offsets of op-relative token `tok` inside its chunk's slab
B200KV_HD void split_chunk_offsets(const SplitTile& t, uint32_t tok, uint64_t* v, uint64_t* s) {
  const uint32_t ct = tok % t.C;
  *v = static_cast<uint64_t>(ct) * t.vb;
  *s = static_cast<uint64_t>(t.C) * t.vb + static_cast<uint64_t>(ct) * t.sb;
}

// The value piece and the scale piece of run r.  mode: 0 = store (pages at slot r.a -> chunk at op token r.b),
// 1 = load (the reverse), 2 = pull (source pages at slot r.a -> destination pages at slot r.b).
B200KV_HD void split_run_pieces(const SplitTile& t, int mode, const Run& r, SplitPiece* val, SplitPiece* sc) {
  uint64_t av, as, bv, bsc;   // side a: pages at slot r.a; side b: the chunk (or the destination pages) at r.b
  split_page_offsets(t, t.a_stride, static_cast<uint32_t>(r.a), &av, &as);
  if (mode == 2) split_page_offsets(t, t.b_stride, static_cast<uint32_t>(r.b), &bv, &bsc);
  else split_chunk_offsets(t, static_cast<uint32_t>(r.b), &bv, &bsc);
  const uint32_t nv = static_cast<uint32_t>(r.n) * t.vb, ns = static_cast<uint32_t>(r.n) * t.sb;
  if (mode == 1) {   // chunk -> pages
    *val = {bv, av, nv};
    *sc = {bsc, as, ns};
  } else {
    *val = {av, bv, nv};
    *sc = {as, bsc, ns};
  }
}

// A piece may go through the TMA engine when both ends and its size are 16-byte multiples (the bases of both sides
// are 16-byte aligned, so this holds for the offsets exactly when it holds for the addresses).  Value pieces always
// qualify (vb % 16 == 0); scale pieces do for whole blocks when bs % 4 == 0 and C % 4 == 0.
B200KV_HD bool bulk_piece(const SplitPiece& p) { return ((p.src | p.dst | p.bytes) & 15u) == 0; }

// Byte layout of a table as the kernels read it: the runs, the chunk addresses, then full_off (the FP8
// store kernels' per-chunk run offsets), each rounded up to 16 bytes.  A table over kTableBytes is refused.
constexpr size_t kTableBytes = 1u << 20;

struct TableLayout {
  size_t runs_off, addrs_off, offs_off, bytes;
};

inline int table_layout(size_t n_runs, size_t n_chunks, TableLayout* l) {
  const size_t runs_bytes = (n_runs * sizeof(Run) + 15) / 16 * 16;
  const size_t addrs_bytes = (n_chunks * 8 + 15) / 16 * 16;
  const size_t offs_bytes = ((n_chunks + 1) * 4 + 15) / 16 * 16;
  l->runs_off = 0;
  l->addrs_off = runs_bytes;
  l->offs_off = runs_bytes + addrs_bytes;
  l->bytes = runs_bytes + addrs_bytes + offs_bytes;
  return l->bytes > kTableBytes ? B200KV_EINVAL : B200KV_OK;
}

}  // namespace b200kv
