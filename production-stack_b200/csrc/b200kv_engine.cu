// b200kv_engine.cu — per-GPU runtime behind the C ABI (include/b200kv.h).
//
// Stands in for LMCacheEngine.store / .retrieve as driven by vLLM's adapter
// (vllm/.../lmcache_integration/vllm_v1_adapter.py:1115-1123 store, :882-889 retrieve) and for
// the NIXL peer channel (helm/templates/deployment-vllm-multi.yaml:296-324).
//
// Streams (all created on the engine's device):
//   s_gather   store kernels          (lowest priority: shares SMs with decode)
//   s_d2h      staging -> pinned pool (copy engine)
//   s_h2d      pinned pool -> staging (copy engine)
//   s_scatter  load / pull kernels    (highest priority: on the TTFT critical path)
// The caller's compute stream only ever waits for a *kernel* (gather done / scatter done),
// never for a PCIe transfer of a store.
#include <algorithm>
#include <atomic>
#include <cctype>
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include <cuda.h>
#include <cuda_runtime.h>

#include <sched.h>
#include <sys/syscall.h>
#include <unistd.h>

#include "b200kv.h"
#include "b200kv_kernels.cuh"

using namespace b200kv;

namespace {

thread_local char g_err[512] = {0};

void set_err(const char* what, cudaError_t e, int line) {
  std::snprintf(g_err, sizeof(g_err), "%s: %s (%s) at b200kv_engine.cu:%d", what,
                cudaGetErrorName(e), cudaGetErrorString(e), line);
}

#define CU_TRY(expr)                          \
  do {                                        \
    cudaError_t _e = (expr);                  \
    if (_e != cudaSuccess) {                  \
      set_err(#expr, _e, __LINE__);           \
      return B200KV_ENODEV;                   \
    }                                         \
  } while (0)

constexpr int kTableSlots = 16;
constexpr int kMaxPeers = 64;
constexpr uint32_t kStageMax = 32u << 10;

// kernel-time slots of b200kv_last_kernel_ms: stores and gathers, loads and scatters, peer pulls
enum TimingSlot { kTimeGather = 0, kTimeScatter = 1, kTimePull = 2, kTimingSlots = 3 };

struct StageSlot {
  cudaEvent_t free_ev = nullptr;  // recorded when the last consumer of this slot is done
  bool used = false;
};

struct TableSlot {
  uint8_t* host = nullptr;  // pinned
  uint8_t* dev = nullptr;
  cudaEvent_t ev = nullptr;  // H2D of the table finished (host side reusable)
  cudaEvent_t done_ev = nullptr;  // kernels reading the device table finished
  bool used = false;
};

struct Op {
  uint64_t id = 0;
  b200kv_pool* pool = nullptr;
  std::vector<uint64_t> commit_keys;   // store: commit after D2H
  std::vector<uint64_t> release_keys;  // load: unpin after scatter
  cudaEvent_t done = nullptr;
  std::atomic<int> host_done{0};
  // layer-wise loads: group_ev[g] fires when layers [g*G, (g+1)*G) of every chunk are in the pages
  std::vector<cudaEvent_t> group_ev;
  int layers_per_group = 0;
};

void destroy_op_events(Op* op) {
  if (op->done) cudaEventDestroy(op->done);
  op->done = nullptr;
  for (cudaEvent_t e : op->group_ev) cudaEventDestroy(e);
  op->group_ev.clear();
}

void CUDART_CB op_host_cb(void* p) {
  Op* op = static_cast<Op*>(p);
  if (op->pool) {
    for (uint64_t k : op->commit_keys) b200kv_pool_commit(op->pool, k);
    for (uint64_t k : op->release_keys) b200kv_pool_release(op->pool, k);
  }
  op->host_done.store(1, std::memory_order_release);
}

// Undoes what a store / load / pull had taken when it leaves early (argument the table cannot hold, a
// failed CUDA call): reserved-but-uncommitted pool slots are aborted (otherwise later stores of those keys
// see -EEXIST until the stale-writer reclaim), pinned chunks are released (otherwise they can never be
// evicted), and the op's events are destroyed.  The engine's streams are drained first, so no copy into
// or out of those slots is still in flight and no host callback enqueued for the op can still run.
struct OpGuard {
  b200kv_ctx* ctx;
  cudaStream_t s[4];
  std::unique_ptr<Op> op;
  std::vector<uint64_t> reserved;   // store: keys reserved in the pool, not yet handed to the commit callback
  bool cb_enqueued = false;         // the host callback owns commit / release from here on
  bool armed = true;
  OpGuard(b200kv_ctx* c, cudaStream_t a, cudaStream_t b, cudaStream_t d, cudaStream_t e) : ctx(c), s{a, b, d, e} {}
  ~OpGuard() {
    if (!armed || (!op && reserved.empty())) return;
    for (cudaStream_t st : s) if (st) cudaStreamSynchronize(st);
    cudaGetLastError();
    if (!cb_enqueued) {
      for (uint64_t k : reserved) b200kv_pool_abort(ctx_pool(), k);
      if (op) for (uint64_t k : op->release_keys) b200kv_pool_release(ctx_pool(), k);
    }
    if (op) destroy_op_events(op.get());
  }
  b200kv_pool* ctx_pool() const;
};

struct Peer {
  bool valid = false;
  int device = -1;
  uint64_t* d_bases = nullptr;       // the peer's base table, slots as ours (base_slot); indexer planes have our stride
  uint64_t block_stride = 0;
  uint64_t n_blocks = 0;
  std::vector<void*> opened;  // cudaIpcOpenMemHandle mappings to close
  // a peer of another tensor-parallel size (b200kv_import_peer_sliced): its planes hold slice.peer_heads heads per
  // token, and a pull moves slice.n_heads of them; pulls from it take kv_head_slice_pull_kernel
  bool sliced = false;
  b200kv_head_slice slice{};
};

struct Geometry {
  uint32_t L, H, D, elem, bs, C, planes;
  uint32_t planes_per_layer;  // 2 (K, V), or 1 (MLA latent)
  uint32_t n_bases;       // base-table slots, one per IPC descriptor: the planes, then L indexer planes (indexed)
  uint32_t token_bytes;   // H*D*elem
  uint64_t slab_bytes;    // C*token_bytes (RAW) or C*H*D (FP8)
  uint64_t chunk_bytes;
  uint64_t scales_off;    // FP8 K/V only
  uint64_t scales_bytes;  // bytes at scales_off (0: the format has no separate scales area)
  uint32_t fmt_token_bytes;
  bool hnd;               // [H][bs][D] inside a block (B200KV_LAYOUT_HND)
  bool mla;               // one latent plane per layer (B200KV_LAYOUT_MLA)
  uint32_t row_bytes;     // D*elem
  uint32_t dtype;         // B200KV_DTYPE_*: element type of the cache (b200kv_set_cache_dtype; bf16 by default)
  // indexer planes (MLA with sparse attention, b200kv_set_indexer): one split tile per block, [bs][idx_vb] values
  // then [bs][idx_sb] scales; in a chunk, L slabs of [C][idx_vb] + [C][idx_sb] after the latent part
  bool indexed;
  uint32_t idx_vb, idx_sb;
  uint64_t idx_stride;    // bytes between consecutive blocks of one indexer plane
  uint64_t idx_off;       // where the indexer slabs start inside a chunk
  uint64_t idx_slab;      // C * (idx_vb + idx_sb): one layer's indexer slab
};

int make_geometry(const b200kv_engine_config* c, Geometry* g) {
  if (c->n_layers <= 0 || c->n_kv_heads <= 0 || c->head_dim <= 0 || c->block_tokens <= 0 ||
      c->chunk_tokens <= 0 || c->chunk_tokens % c->block_tokens)
    return B200KV_EINVAL;
  if (c->elem_bytes != 1 && c->elem_bytes != 2 && c->elem_bytes != 4) return B200KV_EINVAL;
  g->L = c->n_layers;
  g->H = c->n_kv_heads;
  g->D = c->head_dim;
  g->elem = c->elem_bytes;
  g->bs = c->block_tokens;
  g->C = c->chunk_tokens;
  if (c->kv_layout != B200KV_LAYOUT_NHD && c->kv_layout != B200KV_LAYOUT_HND && c->kv_layout != B200KV_LAYOUT_MLA)
    return B200KV_EINVAL;
  g->hnd = c->kv_layout == B200KV_LAYOUT_HND;
  g->mla = c->kv_layout == B200KV_LAYOUT_MLA;
  if (g->mla && g->H != 1) return B200KV_EINVAL;  // the latent is per token, not per head
  g->planes_per_layer = g->mla ? 1u : 2u;
  g->planes = g->planes_per_layer * g->L;
  g->n_bases = g->planes;
  g->token_bytes = g->H * g->D * g->elem;
  g->row_bytes = g->D * g->elem;
  g->dtype = B200KV_DTYPE_BF16;
  g->scales_bytes = 0;
  g->indexed = false;
  g->idx_vb = g->idx_sb = 0;
  g->idx_stride = g->idx_off = g->idx_slab = 0;
  if (g->token_bytes % 16) return B200KV_EINVAL;  // 16-byte vectors / bulk-copy granularity
  if (g->hnd && g->row_bytes % 16) return B200KV_EINVAL;
  if (c->format == B200KV_FMT_RAW) {
    g->fmt_token_bytes = g->token_bytes;
    g->slab_bytes = static_cast<uint64_t>(g->C) * g->token_bytes;
    g->scales_off = 0;
    g->chunk_bytes = g->slab_bytes * g->planes;
  } else if (c->format == B200KV_FMT_FP8 && g->mla) {
    // per-token latent records (b200kv.h, B200KV_LAYOUT_MLA); the scales live inside each record
    if (g->elem != 2 || g->D != kMlaDim) return B200KV_ENOTSUP;
    g->fmt_token_bytes = kMlaRecordBytes;
    g->slab_bytes = static_cast<uint64_t>(g->C) * g->fmt_token_bytes;
    g->scales_off = 0;
    g->chunk_bytes = (g->slab_bytes * g->planes + 255) / 256 * 256;
  } else if (c->format == B200KV_FMT_FP8) {
    if (g->elem != 2) return B200KV_ENOTSUP;  // source must be bf16 or fp16
    if (g->hnd && (g->C / kCluster) % g->bs) return B200KV_ENOTSUP;  // a cluster window = whole tiles
    if (g->H > kMaxHeads) return B200KV_ENOTSUP;
    if (g->C % kCluster) return B200KV_EINVAL;
    if ((g->D * 2) % 16) return B200KV_EINVAL;
    g->fmt_token_bytes = g->token_bytes / 2;
    g->slab_bytes = static_cast<uint64_t>(g->C) * g->fmt_token_bytes;
    g->scales_off = g->slab_bytes * g->planes;
    g->scales_bytes = static_cast<uint64_t>(g->planes) * g->H * sizeof(float);
    g->chunk_bytes = (g->scales_off + g->scales_bytes + 255) / 256 * 256;
  } else if (c->format == B200KV_FMT_Q4) {
    if ((g->elem != 2 && g->elem != 1) || g->mla) return B200KV_ENOTSUP;   // 16-bit or fp8 pages
    if (g->D % 32) return B200KV_EINVAL;
    if (g->elem == 1 && (g->H * g->D) % 64) return B200KV_EINVAL;   // fp8 kernels: records 4-byte aligned
    g->fmt_token_bytes = g->H * g->D / 2 + g->H * (g->D / 32) * 2;   // one token record of one plane
    g->slab_bytes = static_cast<uint64_t>(g->C) * g->fmt_token_bytes;
    g->scales_off = 0;
    g->chunk_bytes = (g->slab_bytes * g->planes + 255) / 256 * 256;
  } else {
    return B200KV_EINVAL;
  }
  return B200KV_OK;
}

// Adds an indexer plane per layer to an MLA geometry (b200kv_set_indexer): the chunk becomes the latent part as
// before, unrounded, followed by L indexer slabs, and the whole is rounded up to 256 bytes.
int add_indexer(Geometry* g, int64_t value_bytes, int64_t scale_bytes, uint64_t block_stride) {
  if (!g->mla || g->scales_bytes) return B200KV_EINVAL;
  if (value_bytes <= 0 || value_bytes % 16 || value_bytes > (1 << 16) || scale_bytes <= 0 || scale_bytes % 4 ||
      scale_bytes > (1 << 16))
    return B200KV_EINVAL;
  const uint64_t tile = static_cast<uint64_t>(g->bs) * static_cast<uint64_t>(value_bytes + scale_bytes);
  if (block_stride < tile || block_stride % 16) return B200KV_EINVAL;
  const uint64_t slab = static_cast<uint64_t>(g->C) * static_cast<uint64_t>(value_bytes + scale_bytes);
  if (slab % 16) return B200KV_EINVAL;   // every slab starts on a 16-byte boundary (bulk copies)
  g->indexed = true;
  g->n_bases = g->planes + g->L;
  g->idx_vb = static_cast<uint32_t>(value_bytes);
  g->idx_sb = static_cast<uint32_t>(scale_bytes);
  g->idx_stride = block_stride;
  g->idx_off = g->slab_bytes * g->planes;
  g->idx_slab = slab;
  g->chunk_bytes = (g->idx_off + g->idx_slab * g->L + 255) / 256 * 256;
  return B200KV_OK;
}

// Base-table slot of plane (kind, l) as callers order planes (b200kv.h, "Planes and descriptors"; descriptor i is
// (i / L, i % L)): kernels index ppl*l + kind, and indexer planes follow at planes + l.  The only order conversion.
uint32_t base_slot(const Geometry& g, uint32_t kind, uint32_t l) {
  return kind < g.planes_per_layer ? g.planes_per_layer * l + kind : g.planes + l;
}

// (k_ptrs, v_ptrs) -> the full base table.  v_ptrs is given exactly when the engine has a second kind of plane, and
// every pointer is non-null and 16-byte aligned; otherwise -EINVAL.
int plane_bases(const Geometry& g, const void* const* k_ptrs, const void* const* v_ptrs, std::vector<uint64_t>* out) {
  const uint32_t kinds = g.n_bases / g.L;
  if (!k_ptrs || (kinds == 2) != (v_ptrs != nullptr)) return B200KV_EINVAL;
  out->assign(g.n_bases, 0);
  for (uint32_t kind = 0; kind < kinds; ++kind)
    for (uint32_t l = 0; l < g.L; ++l) {
      const uint64_t p = reinterpret_cast<uint64_t>((kind ? v_ptrs : k_ptrs)[l]);
      if (!p || p % 16) return B200KV_EINVAL;
      (*out)[base_slot(g, kind, l)] = p;
    }
  return B200KV_OK;
}

// The geometry kv_fp8_store3_kernel needs: a (chunk, head) unit of bf16 fits one consumer group's registers, a
// row is a whole number of 16-byte vectors that divides the group, one block's rows of a head fill whole 128-byte
// lines, a chunk has at most 256 blocks, and (HND) one step of the group's tokens is whole tiles.
bool fp8_store3_fits(const Geometry& g) {
  const uint32_t rv = g.row_bytes >> 4;
  return g.elem == 2 && static_cast<uint64_t>(g.C) * g.row_bytes <= kS3MaxUnitBytes && (g.row_bytes & 15) == 0 &&
         rv != 0 && kS3GroupThreads % rv == 0 && (static_cast<uint64_t>(g.bs) * g.row_bytes) % 128 == 0 &&
         g.C / g.bs <= 32 * 8 && !(g.hnd && (kS3GroupThreads / rv) % g.bs != 0);
}

}  // namespace

struct b200kv_ctx {
  b200kv_engine_config cfg{};
  Geometry g{};
  b200kv_pool* pool = nullptr;
  bool pool_registered = false;
  std::string numa_placement = "no pool";   // what place_pool_pages() did when this engine pinned the pool
  void* pool_base = nullptr;
  int sm_count = 132;
  std::mutex mu;

  cudaStream_t s_gather = nullptr, s_d2h = nullptr, s_h2d = nullptr, s_scatter = nullptr;
  cudaEvent_t fence = nullptr;          // stream_wait's event
  uint64_t* d_bases = nullptr;          // the base table, g.n_bases slots (base_slot)
  bool kv_registered = false;
  std::vector<uint64_t> h_bases;        // the registered base table on the host (export_ipc)

  uint8_t* d_staging = nullptr;
  std::vector<StageSlot> stage;
  // The ring is split in two halves — stores allocate from [0, n_store), loads from [n_store, n):
  // a TTFT-critical load must never queue behind the D2H of an unrelated store.
  uint32_t n_store_slots = 0, store_next = 0, load_next = 0;

  TableSlot tables[kTableSlots];
  uint32_t table_next = 0;

  Peer peers[kMaxPeers];

  uint64_t next_ticket = 1;
  std::map<uint64_t, std::unique_ptr<Op>> ops;

  // timing of the most recent kernel batch of each kind (CUDA events on the launching stream)
  struct Timing {
    std::vector<std::pair<cudaEvent_t, cudaEvent_t>> ev;
    size_t used = 0;
  } timing[kTimingSlots];

  b200kv_engine_stats stats{};

  // bulk-kernel launch shape
  int S = 2, LAG = 1, ctas_per_sm = 1;  // B200KV_STAGES / B200KV_LAG / B200KV_CTAS_PER_SM (tools/sweep.py)
  bool fp8_store3 = false;              // FP8 stores may take kv_fp8_store3_kernel: its geometry fits, and
                                        // B200KV_FP8_STORE (3 = that kernel, the default; 1 = cluster kernel) allows it
  void* d_tmaps = nullptr;              // one CUtensorMap per plane (NHD pages: strided [bs][D] boxes for the FP8 store)
  std::string tmap_status = "not built";
  uint32_t piece_tokens = 0, pieces = 0, stage_bytes = 0;

  void* tier_base = nullptr;            // device chunk tier (b200kv_tier_create)
  uint32_t tier_slots = 0;
  std::vector<void*> tier_imports;      // peers' tiers opened over CUDA IPC
};

b200kv_pool* OpGuard::ctx_pool() const { return ctx->pool; }

namespace {

struct DeviceGuard {
  int prev = -1;
  bool ok = false;
  explicit DeviceGuard(int dev) {
    if (cudaGetDevice(&prev) == cudaSuccess && cudaSetDevice(dev) == cudaSuccess) ok = true;
  }
  ~DeviceGuard() {
    if (prev >= 0) cudaSetDevice(prev);
  }
};

int env_int(const char* name, int dflt) {
  const char* v = std::getenv(name);
  return (v && *v) ? std::atoi(v) : dflt;
}

// ---- run tables: built by b200kv_runs.h, staged through the table ring --------------------------
int op_table(const b200kv_ctx* ctx, const int64_t* slots, const std::vector<Span>& spans, OpTable* t) {
  const Geometry& g = ctx->g;
  return build_op_table(slots, spans.data(), spans.size(), static_cast<int64_t>(ctx->cfg.n_blocks) * g.bs,
                        static_cast<int32_t>(g.bs), static_cast<int32_t>(g.C), ctx->cfg.format == B200KV_FMT_RAW,
                        g.hnd, t);
}

// a staged table: its ring slot and its arrays in device memory
struct TableView {
  TableSlot* slot;
  const Run* runs;
  const uint64_t* chunk_addrs;
  const uint32_t* full_off;
};

// Takes the next slot of the table ring, fills it with `t` and chunk_addrs[0, t.n_chunks()) and uploads it
// on `s`.  A table over kTableBytes is refused before anything is enqueued.
int stage_table(b200kv_ctx* ctx, const OpTable& t, const uint64_t* chunk_addrs, cudaStream_t s, TableView* tv) {
  const uint32_t n_chunks = t.n_chunks();
  TableLayout l;
  if (table_layout(t.runs.size(), n_chunks, &l)) return B200KV_EINVAL;  // op too large: caller must split
  TableSlot& ts = ctx->tables[ctx->table_next];
  ctx->table_next = (ctx->table_next + 1) % kTableSlots;
  if (ts.used) {  // host must not overwrite a table whose upload / readers are still in flight
    CU_TRY(cudaEventSynchronize(ts.ev));
    CU_TRY(cudaEventSynchronize(ts.done_ev));
  }
  std::memcpy(ts.host + l.runs_off, t.runs.data(), t.runs.size() * sizeof(Run));
  std::memcpy(ts.host + l.addrs_off, chunk_addrs, n_chunks * sizeof(uint64_t));
  std::memcpy(ts.host + l.offs_off, t.full_off.data(), (n_chunks + 1) * sizeof(uint32_t));
  CU_TRY(cudaMemcpyAsync(ts.dev, ts.host, l.bytes, cudaMemcpyHostToDevice, s));
  CU_TRY(cudaEventRecord(ts.ev, s));
  ts.used = true;
  ctx->stats.h2d_bytes += l.bytes;
  tv->slot = &ts;
  tv->runs = reinterpret_cast<const Run*>(ts.dev + l.runs_off);
  tv->chunk_addrs = reinterpret_cast<const uint64_t*>(ts.dev + l.addrs_off);
  tv->full_off = reinterpret_cast<const uint32_t*>(ts.dev + l.offs_off);
  return B200KV_OK;
}

// Makes `waiter` wait for the work enqueued on `signaller` so far.  cudaStreamWaitEvent takes the event's
// current record, so one event serves every wait made under ctx->mu.
int stream_wait(b200kv_ctx* ctx, cudaStream_t waiter, cudaStream_t signaller) {
  CU_TRY(cudaEventRecord(ctx->fence, signaller));
  CU_TRY(cudaStreamWaitEvent(waiter, ctx->fence, 0));
  return B200KV_OK;
}

// Every chunk holds 1..C tokens and every slot of chunk c, slot_mapping[c*C, c*C + chunk_tokens[c]), lies in
// [0, n_blocks*bs).  Ops check this before they reserve or pin anything, so a malformed mapping takes nothing.
int check_chunk_slots(const b200kv_ctx* ctx, const int64_t* slot_mapping, const int32_t* chunk_tokens,
                      int32_t n_chunks) {
  const int64_t max_slot = static_cast<int64_t>(ctx->cfg.n_blocks) * ctx->g.bs;
  for (int32_t c = 0; c < n_chunks; ++c) {
    if (chunk_tokens[c] <= 0 || chunk_tokens[c] > static_cast<int32_t>(ctx->g.C)) return B200KV_EINVAL;
    const int64_t* sm = slot_mapping + static_cast<int64_t>(c) * ctx->g.C;
    for (int32_t i = 0; i < chunk_tokens[c]; ++i)
      if (out_of_range(sm[i], max_slot)) return B200KV_EINVAL;
  }
  return B200KV_OK;
}

// ---- timing events -----------------------------------------------------------------------------
void timing_reset(b200kv_ctx* ctx, int which) { ctx->timing[which].used = 0; }

int timing_begin(b200kv_ctx* ctx, int which, cudaStream_t s) {
  auto& t = ctx->timing[which];
  if (t.used == t.ev.size()) {
    cudaEvent_t a, b;
    CU_TRY(cudaEventCreate(&a));
    CU_TRY(cudaEventCreate(&b));
    t.ev.emplace_back(a, b);
  }
  CU_TRY(cudaEventRecord(t.ev[t.used].first, s));
  return B200KV_OK;
}
int timing_end(b200kv_ctx* ctx, int which, cudaStream_t s) {
  auto& t = ctx->timing[which];
  CU_TRY(cudaEventRecord(t.ev[t.used].second, s));
  ++t.used;
  return B200KV_OK;
}

// ---- kernel launches ---------------------------------------------------------------------------
// the end of every launch: a launch error fails the op, and stats count the launches
int launched(b200kv_ctx* ctx) {
  CU_TRY(cudaGetLastError());
  ++ctx->stats.n_kernel_launches;
  return B200KV_OK;
}

typedef void (*BulkKernel)(KernelArgs, uint32_t);

// the bulk kernel built for a B200KV_STAGES / B200KV_LAG pair; null for a pair that is not built
template <int MODE>
BulkKernel bulk_kernel(int S, int LAG) {
  switch (S * 10 + LAG) {
    case 21: return kv_bulk_copy_kernel<MODE, 2, 1>;
    case 31: return kv_bulk_copy_kernel<MODE, 3, 1>;
    case 32: return kv_bulk_copy_kernel<MODE, 3, 2>;
    case 41: return kv_bulk_copy_kernel<MODE, 4, 1>;
    case 42: return kv_bulk_copy_kernel<MODE, 4, 2>;
    case 43: return kv_bulk_copy_kernel<MODE, 4, 3>;
    case 63: return kv_bulk_copy_kernel<MODE, 6, 3>;
    case 64: return kv_bulk_copy_kernel<MODE, 6, 4>;
    default: return nullptr;
  }
}

// format tag recorded with a chunk: a pool shared by engines of different tile order, codec, cache element type or
// indexer planes never hands one engine's bytes to another (bf16 engines keep the tags they had before the dtype
// field, engines without indexer planes the tags they had before bit 24)
uint32_t pool_fmt(const b200kv_ctx* ctx) {
  return static_cast<uint32_t>(ctx->cfg.format) | (static_cast<uint32_t>(ctx->cfg.kv_layout) << 8) |
         (ctx->g.dtype << 16) | (ctx->g.indexed ? 1u << 24 : 0u);
}

PagedSide local_side(const b200kv_ctx* ctx) {
  PagedSide s;
  s.bases = ctx->d_bases;
  s.block_stride = ctx->cfg.block_stride_bytes;
  s.block_tokens = ctx->g.bs;
  s.token_bytes = ctx->g.token_bytes;
  return s;
}

// The parameter block of a launch over runs [run_begin, ...) of the staged table `tv`, planes [plane_begin,
// plane_begin + n_planes) (n_planes == 0: every plane).  `peer` non-null is the pull source.  The launcher sets
// total_units.
KernelArgs kernel_args(const b200kv_ctx* ctx, const TableView& tv, size_t run_begin, uint32_t plane_begin,
                       uint32_t n_planes, const Peer* peer = nullptr) {
  const Geometry& g = ctx->g;
  KernelArgs a{};
  a.paged = local_side(ctx);
  a.peer = a.paged;
  if (peer) {
    a.peer.bases = peer->d_bases;
    a.peer.block_stride = peer->block_stride;
  }
  a.chunk.chunk_addrs = tv.chunk_addrs;
  a.chunk.slab_bytes = g.slab_bytes;
  a.chunk.scales_off = g.scales_off;
  a.chunk.chunk_tokens = g.C;
  a.chunk.token_bytes = g.fmt_token_bytes;
  a.runs = tv.runs + run_begin;
  a.chunk_run_off = tv.full_off;
  a.plane_begin = plane_begin;
  a.n_planes = n_planes ? n_planes : g.planes;
  a.n_heads = g.H;
  a.row_bytes = g.row_bytes;
  a.hnd = g.hnd ? 1u : 0u;
  a.pieces = ctx->pieces;
  a.piece_tokens = ctx->piece_tokens;
  return a;
}

// RAW: full runs [f0, f0 + nf) of the table go to the bulk (or LDG) kernel, HND partial-tile runs [p0, p0 + np)
// to kv_hnd_partial_kernel.  `peer` non-null selects the pull source.
template <int MODE>
int launch_copy_runs(b200kv_ctx* ctx, const TableView& tv, size_t f0, size_t nf, size_t p0, size_t np,
                     cudaStream_t s, const Peer* peer, uint32_t plane_begin, uint32_t n_planes) {
  if (nf) {
    KernelArgs a = kernel_args(ctx, tv, f0, plane_begin, n_planes, peer);
    a.total_units = static_cast<uint32_t>(nf) * a.n_planes * a.pieces;
    const bool ldg = ctx->cfg.variant == B200KV_VARIANT_LDG;
    const BulkKernel kernel = ldg ? nullptr : bulk_kernel<MODE>(ctx->S, ctx->LAG);
    if (!ldg && !kernel) return B200KV_EINVAL;
    const uint32_t grid = std::min(static_cast<uint32_t>(ctx->sm_count * (ldg ? 8 : ctx->ctas_per_sm)), a.total_units);
    if (grid) {
      if (ldg) kv_ldg_copy_kernel<MODE><<<grid, 256, 0, s>>>(a);
      else kernel<<<grid, 32, 256 + static_cast<size_t>(ctx->S) * ctx->stage_bytes, s>>>(a, ctx->stage_bytes);
      const int rc = launched(ctx);
      if (rc) return rc;
    }
  }
  if (np == 0) return B200KV_OK;
  KernelArgs a = kernel_args(ctx, tv, p0, plane_begin, n_planes, peer);
  a.total_units = static_cast<uint32_t>(np) * a.n_planes * a.n_heads;
  const uint32_t grid = std::min<uint32_t>(a.total_units, static_cast<uint32_t>(ctx->sm_count) * 16u);
  kv_hnd_partial_kernel<MODE><<<grid, 128, 0, s>>>(a);
  return launched(ctx);
}

// FP8 store of every chunk of the table; chunks of several requests may be partial anywhere.  The persistent
// kernel takes the table when the engine allows it (fp8_store3) and every chunk is whole, block-aligned runs; the
// cluster kernel takes every other table.  DT: the cache's element type (the lossy launchers are built per type).
template <int DT>
int launch_fp8_store(b200kv_ctx* ctx, const OpTable& t, const TableView& tv, cudaStream_t s) {
  const Geometry& g = ctx->g;
  KernelArgs a = kernel_args(ctx, tv, 0, 0, 0);
  if (ctx->fp8_store3 && (g.hnd || ctx->tmap_status == "ok") && whole_block_chunks(t, g.bs, g.C)) {
    a.total_units = t.n_chunks() * g.planes * g.H;
    const size_t smem = static_cast<size_t>(kS3Stages) * g.C * g.row_bytes;
    const uint32_t grid = std::min<uint32_t>(a.total_units, static_cast<uint32_t>(ctx->sm_count));
    if (grid == 0) return B200KV_OK;
    kv_fp8_store3_kernel<DT><<<grid, kS3Threads, smem, s>>>(a, g.hnd ? nullptr : ctx->d_tmaps);
    return launched(ctx);
  }
  const size_t smem = static_cast<size_t>(g.C / kCluster) * g.token_bytes;
  if (smem > 200 * 1024) return B200KV_ENOTSUP;
  const uint32_t grid = kCluster * t.n_chunks() * g.planes;
  if (grid == 0) return B200KV_OK;
  kv_fp8_store_kernel<DT><<<grid, kFp8Threads, smem, s>>>(a);
  return launched(ctx);
}

// FP8 load, Q4 store and Q4 load of runs [f0, f0 + nf): one unit per (run, plane).
template <int DT>
int launch_per_run(b200kv_ctx* ctx, CopyMode mode, const TableView& tv, size_t f0, size_t nf, cudaStream_t s,
                   uint32_t plane_begin, uint32_t n_planes) {
  const bool fp8 = ctx->cfg.format == B200KV_FMT_FP8;
  const size_t smem = fp8 ? static_cast<size_t>(ctx->g.bs) * ctx->g.fmt_token_bytes : 0;
  if (smem > 48 * 1024) return B200KV_ENOTSUP;
  KernelArgs a = kernel_args(ctx, tv, f0, plane_begin, n_planes);
  a.total_units = static_cast<uint32_t>(nf) * a.n_planes;
  const uint32_t grid = std::min<uint32_t>(a.total_units, static_cast<uint32_t>(ctx->sm_count) * 8u);
  if (grid == 0) return B200KV_OK;
  if (fp8) kv_fp8_load_kernel<DT><<<grid, kFp8Threads, smem, s>>>(a);
  else if (mode == kStore) kv_q4_store_kernel<DT><<<grid, 256, 0, s>>>(a);
  else kv_q4_load_kernel<DT><<<grid, 256, 0, s>>>(a);
  return launched(ctx);
}

// dynamic shared memory of kv_indexer_copy_kernel: the warps' mbarriers and stages
size_t indexer_smem_bytes(const Geometry& g) {
  return kIdxBarBytes + static_cast<size_t>(kIdxWarps) * ((static_cast<size_t>(g.bs) * (g.idx_vb + g.idx_sb) + 15) & ~15ull);
}

// Q4 store or load of fp8 pages, runs [f0, f0 + nf): one unit per (run, plane), as launch_per_run.
template <__nv_fp8_interpretation_t FT>
int launch_q4_fp8(b200kv_ctx* ctx, CopyMode mode, const TableView& tv, size_t f0, size_t nf, cudaStream_t s,
                  uint32_t plane_begin, uint32_t n_planes) {
  KernelArgs a = kernel_args(ctx, tv, f0, plane_begin, n_planes);
  a.total_units = static_cast<uint32_t>(nf) * a.n_planes;
  const uint32_t grid = std::min<uint32_t>(a.total_units, static_cast<uint32_t>(ctx->sm_count) * 8u);
  if (grid == 0) return B200KV_OK;
  if (mode == kStore) kv_q4_store_fp8_kernel<FT><<<grid, 256, 0, s>>>(a);
  else kv_q4_load_fp8_kernel<FT><<<grid, 256, 0, s>>>(a);
  return launched(ctx);
}

// FP8 latent records of an MLA engine, either direction, runs [f0, f0 + nf): one warp per (run, plane) unit.
template <int DT>
int launch_mla_fp8(b200kv_ctx* ctx, CopyMode mode, const TableView& tv, size_t f0, size_t nf, cudaStream_t s,
                   uint32_t plane_begin, uint32_t n_planes) {
  KernelArgs a = kernel_args(ctx, tv, f0, plane_begin, n_planes);
  a.total_units = static_cast<uint32_t>(nf) * a.n_planes;
  constexpr uint32_t warps = kMlaThreads / 32;
  const uint32_t grid = std::min<uint32_t>((a.total_units + warps - 1) / warps, static_cast<uint32_t>(ctx->sm_count) * 8u);
  if (grid == 0) return B200KV_OK;
  if (mode == kStore) kv_mla_fp8_store_kernel<DT><<<grid, kMlaThreads, 0, s>>>(a);
  else kv_mla_fp8_load_kernel<DT><<<grid, kMlaThreads, 0, s>>>(a);
  return launched(ctx);
}

// The lossy launches of one cache element type.
template <int DT>
int launch_lossy(b200kv_ctx* ctx, CopyMode mode, const OpTable& t, const TableView& tv, size_t f0, size_t nf,
                 cudaStream_t s, uint32_t pb, uint32_t np) {
  if (ctx->cfg.format == B200KV_FMT_FP8 && ctx->g.mla) return launch_mla_fp8<DT>(ctx, mode, tv, f0, nf, s, pb, np);
  if (ctx->cfg.format == B200KV_FMT_FP8 && mode == kStore) return launch_fp8_store<DT>(ctx, t, tv, s);
  return launch_per_run<DT>(ctx, mode, tv, f0, nf, s, pb, np);
}

// The indexer planes of layers [pb, pb + np) (np == 0: every layer) of runs [f0, f0 + nf), verbatim in every
// direction.  KernelArgs carry the indexer side in the fields kv_indexer_copy_kernel names.
int launch_indexer(b200kv_ctx* ctx, CopyMode mode, const TableView& tv, size_t f0, size_t nf, cudaStream_t s,
                   uint32_t pb, uint32_t np, const Peer* peer) {
  const Geometry& g = ctx->g;
  KernelArgs a = kernel_args(ctx, tv, f0, pb, np, peer);
  a.paged.bases = ctx->d_bases + g.planes;
  a.paged.block_stride = g.idx_stride;
  a.paged.token_bytes = g.idx_vb;
  a.peer = a.paged;
  if (peer) a.peer.bases = peer->d_bases + g.planes;
  a.chunk.slab_bytes = g.idx_slab;
  a.chunk.scales_off = g.idx_off;
  a.chunk.token_bytes = g.idx_vb;
  a.row_bytes = g.idx_sb;
  a.total_units = static_cast<uint32_t>(nf) * a.n_planes;
  const uint32_t grid = std::min<uint32_t>((a.total_units + kIdxWarps - 1) / kIdxWarps,
                                           static_cast<uint32_t>(ctx->sm_count) * 8u);
  if (grid == 0) return B200KV_OK;
  const size_t smem = indexer_smem_bytes(g);
  switch (mode) {
    case kStore: kv_indexer_copy_kernel<kStore><<<grid, kIdxWarps * 32, smem, s>>>(a); break;
    case kLoad: kv_indexer_copy_kernel<kLoad><<<grid, kIdxWarps * 32, smem, s>>>(a); break;
    default: kv_indexer_copy_kernel<kPull><<<grid, kIdxWarps * 32, smem, s>>>(a); break;
  }
  return launched(ctx);
}

// Launches the kernels that move chunks [c0, c1) of table t, planes [pb, pb + np) (np == 0: every plane), in
// direction `mode`, and then, on an engine with indexer planes, the indexer planes of the same layers.
int launch_planes(b200kv_ctx* ctx, CopyMode mode, const OpTable& t, const TableView& tv, uint32_t c0, uint32_t c1,
                  cudaStream_t s, uint32_t pb, uint32_t np, const Peer* peer);

// A pull from a sliced peer: every run of the table (full, then partial) through kv_head_slice_pull_kernel, the
// slice in the KernelArgs fields the kernel names.  Sliced peers exist on K/V engines only, so there are no
// indexer planes.
int launch_slice_pull(b200kv_ctx* ctx, const OpTable& t, const TableView& tv, cudaStream_t s, const Peer& peer) {
  const Geometry& g = ctx->g;
  KernelArgs a = kernel_args(ctx, tv, 0, 0, 0, &peer);
  a.peer.token_bytes = static_cast<uint32_t>(peer.slice.peer_heads) * g.row_bytes;
  a.chunk.chunk_tokens = static_cast<uint32_t>(peer.slice.n_heads);
  a.chunk.slab_bytes = static_cast<uint64_t>(peer.slice.src_head0);
  a.chunk.scales_off = static_cast<uint64_t>(peer.slice.dst_head0);
  a.total_units = static_cast<uint32_t>(t.runs.size()) * a.n_planes;
  const uint32_t grid = std::min<uint32_t>(a.total_units, static_cast<uint32_t>(ctx->sm_count) * 8u);
  if (grid == 0) return B200KV_OK;
  kv_head_slice_pull_kernel<<<grid, kSliceThreads, 0, s>>>(a);
  return launched(ctx);
}

int launch_op(b200kv_ctx* ctx, CopyMode mode, const OpTable& t, const TableView& tv, uint32_t c0, uint32_t c1,
              cudaStream_t s, uint32_t pb = 0, uint32_t np = 0, const Peer* peer = nullptr) {
  if (peer && peer->sliced) return launch_slice_pull(ctx, t, tv, s, *peer);
  const int rc = launch_planes(ctx, mode, t, tv, c0, c1, s, pb, np, peer);
  if (rc || !ctx->g.indexed) return rc;
  const size_t f0 = t.full_off[c0], nf = t.full_off[c1] - f0;   // MLA tables have full runs only
  return launch_indexer(ctx, mode, tv, f0, nf, s, pb, np, peer);
}

// The latent (or K and V) planes of launch_op.  A pull copies pages to pages whatever the chunk format.  The FP8
// store of a K/V engine always takes the whole table.
int launch_planes(b200kv_ctx* ctx, CopyMode mode, const OpTable& t, const TableView& tv, uint32_t c0, uint32_t c1,
                  cudaStream_t s, uint32_t pb, uint32_t np, const Peer* peer) {
  const size_t f0 = t.full_off[c0], nf = t.full_off[c1] - f0;
  const int fmt = mode == kPull ? B200KV_FMT_RAW : ctx->cfg.format;
  if (fmt != B200KV_FMT_RAW && ctx->g.elem == 1)   // Q4, the one lossy format of fp8 pages (make_geometry)
    return ctx->g.dtype == B200KV_DTYPE_E5M2 ? launch_q4_fp8<__NV_E5M2>(ctx, mode, tv, f0, nf, s, pb, np)
                                             : launch_q4_fp8<__NV_E4M3>(ctx, mode, tv, f0, nf, s, pb, np);
  if (fmt != B200KV_FMT_RAW)
    return ctx->g.dtype == B200KV_DTYPE_FP16 ? launch_lossy<kFp16>(ctx, mode, t, tv, f0, nf, s, pb, np)
                                             : launch_lossy<kBf16>(ctx, mode, t, tv, f0, nf, s, pb, np);
  const size_t p0 = t.n_full() + t.part_off[c0], n_part = t.part_off[c1] - t.part_off[c0];
  switch (mode) {
    case kStore: return launch_copy_runs<kStore>(ctx, tv, f0, nf, p0, n_part, s, peer, pb, np);
    case kLoad: return launch_copy_runs<kLoad>(ctx, tv, f0, nf, p0, n_part, s, peer, pb, np);
    default: return launch_copy_runs<kPull>(ctx, tv, f0, nf, p0, n_part, s, peer, pb, np);
  }
}

// Planes [pb, pb + np) of one chunk between the pinned pool and staging; np == 0 moves the whole chunk, as
// one copy of chunk_bytes when the chunk is full.  Partial chunks move only their tokens.  The FP8 scales
// travel with a whole chunk, and with a plane range when `with_scales` (the first group of a layer-wise load).
// Indexer slabs travel with their layers.
int copy_chunk_planes(b200kv_ctx* ctx, void* dst, const void* src, uint32_t n_tok, cudaMemcpyKind kind,
                      cudaStream_t s, uint32_t pb = 0, uint32_t np = 0, bool with_scales = true) {
  const Geometry& g = ctx->g;
  const bool whole = np == 0 && n_tok == g.C;
  if (np == 0) np = g.planes;
  uint8_t* d = static_cast<uint8_t*>(dst) + static_cast<uint64_t>(pb) * g.slab_bytes;
  const uint8_t* sp = static_cast<const uint8_t*>(src) + static_cast<uint64_t>(pb) * g.slab_bytes;
  uint64_t moved;
  if (n_tok == g.C) {
    moved = whole ? g.chunk_bytes : static_cast<uint64_t>(np) * g.slab_bytes;
    CU_TRY(cudaMemcpyAsync(d, sp, moved, kind, s));
  } else {
    // HND keeps whole tiles: a ragged tail still occupies its last tile across all heads
    const uint32_t tok_span = (g.hnd && ctx->cfg.format != B200KV_FMT_Q4) ? (n_tok + g.bs - 1) / g.bs * g.bs : n_tok;
    const size_t width = static_cast<size_t>(tok_span) * g.fmt_token_bytes;
    CU_TRY(cudaMemcpy2DAsync(d, g.slab_bytes, sp, g.slab_bytes, width, np, kind, s));
    moved = width * np;
  }
  if (with_scales && !whole && g.scales_bytes) {
    CU_TRY(cudaMemcpyAsync(static_cast<uint8_t*>(dst) + g.scales_off, static_cast<const uint8_t*>(src) + g.scales_off,
                           g.scales_bytes, kind, s));
    moved += g.scales_bytes;
  }
  if (g.indexed && !whole) {   // the indexer slabs of the same layers (MLA: plane == layer)
    uint8_t* di = static_cast<uint8_t*>(dst) + g.idx_off + static_cast<uint64_t>(pb) * g.idx_slab;
    const uint8_t* si = static_cast<const uint8_t*>(src) + g.idx_off + static_cast<uint64_t>(pb) * g.idx_slab;
    if (n_tok == g.C) {
      CU_TRY(cudaMemcpyAsync(di, si, static_cast<uint64_t>(np) * g.idx_slab, kind, s));
      moved += static_cast<uint64_t>(np) * g.idx_slab;
    } else {   // the values of the chunk's tokens, then their scales
      const uint64_t sc = static_cast<uint64_t>(g.C) * g.idx_vb;
      CU_TRY(cudaMemcpy2DAsync(di, g.idx_slab, si, g.idx_slab, static_cast<size_t>(n_tok) * g.idx_vb, np, kind, s));
      CU_TRY(cudaMemcpy2DAsync(di + sc, g.idx_slab, si + sc, g.idx_slab, static_cast<size_t>(n_tok) * g.idx_sb, np,
                               kind, s));
      moved += static_cast<uint64_t>(n_tok) * (g.idx_vb + g.idx_sb) * np;
    }
  }
  if (kind == cudaMemcpyDeviceToHost) ctx->stats.d2h_bytes += moved;
  else ctx->stats.h2d_bytes += moved;
  return B200KV_OK;
}

void reap(b200kv_ctx* ctx) {
  for (auto it = ctx->ops.begin(); it != ctx->ops.end();) {
    Op* op = it->second.get();
    if (cudaEventQuery(op->done) == cudaSuccess && op->host_done.load(std::memory_order_acquire)) {
      destroy_op_events(op);
      it = ctx->ops.erase(it);
    } else {
      ++it;
    }
  }
}

}  // namespace

// ================================================================================================
// C ABI
// ================================================================================================
extern "C" int b200kv_abi_version(void) { return B200KV_ABI_VERSION; }

extern "C" const char* b200kv_last_error(void) { return g_err; }

extern "C" const char* b200kv_strerror(int err) {
  switch (err) {
    case B200KV_OK: return "ok";
    case B200KV_EINVAL: return "invalid argument";
    case B200KV_ENOMEM: return "out of memory";
    case B200KV_ENODEV: return "CUDA device unavailable or CUDA call failed";
    case B200KV_ENOENT: return "not found";
    case B200KV_EEXIST: return "already exists";
    case B200KV_ENOSPC: return "pool full";
    case B200KV_ENOTSUP: return "not supported";
    case B200KV_EBUSY: return "busy";
    default: return std::strerror(-err);
  }
}

extern "C" int64_t b200kv_engine_chunk_bytes(const b200kv_engine_config* cfg) {
  if (!cfg) return B200KV_EINVAL;
  Geometry g;
  const int rc = make_geometry(cfg, &g);
  if (rc) return rc;
  return static_cast<int64_t>(g.chunk_bytes);
}

extern "C" int64_t b200kv_engine_chunk_bytes_indexed(const b200kv_engine_config* cfg, int32_t value_bytes,
                                                    int32_t scale_bytes) {
  if (!cfg) return B200KV_EINVAL;
  Geometry g;
  int rc = make_geometry(cfg, &g);
  if (rc) return rc;
  // the block stride does not enter the chunk: pass the smallest legal one
  rc = add_indexer(&g, value_bytes, scale_bytes,
                   (static_cast<uint64_t>(g.bs) * static_cast<uint64_t>(std::max(value_bytes + scale_bytes, 0)) + 15) / 16 * 16);
  if (rc) return rc;
  return static_cast<int64_t>(g.chunk_bytes);
}

static int engine_create_impl(const b200kv_engine_config* cfg, b200kv_pool* pool, b200kv_ctx** out);

extern "C" int b200kv_engine_destroy(b200kv_ctx* ctx);

extern "C" int b200kv_engine_numa_placement(b200kv_ctx* ctx, char* buf, uint64_t n) {
  if (!ctx || !buf || n == 0) return B200KV_EINVAL;
  std::snprintf(buf, n, "%s", ctx->numa_placement.c_str());
  return B200KV_OK;
}

// ---- host-page placement of the pinned pool --------------------------------------------------
// On a two-socket HGX box every DMA of a GPU whose pool pages sit on the other socket crosses the
// inter-socket link twice as slowly as the PCIe link it came over.  The pages of the pool segment are
// physically allocated when the first engine pins them (cudaHostRegister faults them in), so the
// policy is applied to the mapping right before that: mbind() on the shared mapping (shmem keeps the
// policy with the object, so later attachers inherit it).  Where mbind is filtered (containers without
// CAP_SYS_NICE) the fallback for NUMA_LOCAL is to run the pinning call on the node's CPUs.
static int gpu_numa_node(int device) {
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof(bus), device) != cudaSuccess) return -1;
  for (char* p = bus; *p; ++p) *p = static_cast<char>(std::tolower(*p));
  char path[128];
  std::snprintf(path, sizeof(path), "/sys/bus/pci/devices/%s/numa_node", bus);
  FILE* f = std::fopen(path, "r");
  if (!f) return -1;
  int node = -1;
  if (std::fscanf(f, "%d", &node) != 1) node = -1;
  std::fclose(f);
  return node;
}

static int online_numa_nodes(unsigned long* mask, int* max_node) {
  *mask = 0;
  *max_node = -1;
  FILE* f = std::fopen("/sys/devices/system/node/online", "r");
  if (!f) return -1;
  char buf[128] = {0};
  if (!std::fgets(buf, sizeof(buf), f)) { std::fclose(f); return -1; }
  std::fclose(f);
  for (char* p = buf; *p && *p != '\n';) {       // "0-1" or "0,2-3"
    char* e = nullptr;
    long a = std::strtol(p, &e, 10), b = a;
    if (e == p) break;
    if (*e == '-') { p = e + 1; b = std::strtol(p, &e, 10); }
    for (long n = a; n <= b && n < 64; ++n) { *mask |= 1ul << n; *max_node = std::max<int>(*max_node, static_cast<int>(n)); }
    p = (*e == ',') ? e + 1 : e;
  }
  return *max_node >= 0 ? 0 : -1;
}

struct NumaPinScope {       // restores the thread's CPU affinity if the fallback narrowed it
  cpu_set_t saved;
  bool narrowed = false;
  ~NumaPinScope() { if (narrowed) sched_setaffinity(0, sizeof(saved), &saved); }
};

// returns a short description for the log / stats ("mbind preferred node 1", "affinity node 0", ...)
static std::string place_pool_pages(void* base, uint64_t bytes, int device, int policy, NumaPinScope* scope) {
  const char* e = std::getenv("B200KV_POOL_NUMA");       // local | interleave | off overrides the config
  if (e) policy = !std::strcmp(e, "interleave") ? B200KV_NUMA_INTERLEAVE : !std::strcmp(e, "off") ? B200KV_NUMA_OFF : B200KV_NUMA_LOCAL;
  if (policy == B200KV_NUMA_OFF) return "first touch (off)";
  unsigned long online = 0;
  int max_node = -1;
  if (online_numa_nodes(&online, &max_node) != 0 || max_node == 0) return "single NUMA node";
  constexpr int kPreferred = 1, kInterleave = 3;    // MPOL_* of <linux/mempolicy.h>
  if (policy == B200KV_NUMA_INTERLEAVE) {
    const long rc = syscall(SYS_mbind, base, static_cast<unsigned long>(bytes), kInterleave, &online, 65ul, 0u);
    return rc == 0 ? "mbind interleave over online nodes" : std::string("mbind refused (") + std::strerror(errno) + "): first touch";
  }
  const int node = gpu_numa_node(device);
  if (node < 0 || node > max_node) return "GPU NUMA node unknown: first touch";
  unsigned long mask = 1ul << node;
  if (syscall(SYS_mbind, base, static_cast<unsigned long>(bytes), kPreferred, &mask, 65ul, 0u) == 0)
    return "mbind preferred node " + std::to_string(node);
  const int mbind_errno = errno;
  // fallback: fault the pages in from a CPU of that node
  char path[96];
  std::snprintf(path, sizeof(path), "/sys/devices/system/node/node%d/cpulist", node);
  FILE* f = std::fopen(path, "r");
  cpu_set_t want;
  CPU_ZERO(&want);
  if (f) {
    char buf[512] = {0};
    if (std::fgets(buf, sizeof(buf), f)) {
      for (char* p = buf; *p && *p != '\n';) {
        char* q = nullptr;
        long a = std::strtol(p, &q, 10), b = a;
        if (q == p) break;
        if (*q == '-') { p = q + 1; b = std::strtol(p, &q, 10); }
        for (long c = a; c <= b && c < CPU_SETSIZE; ++c) CPU_SET(static_cast<int>(c), &want);
        p = (*q == ',') ? q + 1 : q;
      }
    }
    std::fclose(f);
  }
  if (CPU_COUNT(&want) > 0 && sched_getaffinity(0, sizeof(scope->saved), &scope->saved) == 0) {
    cpu_set_t both;
    CPU_AND(&both, &want, &scope->saved);
    if (CPU_COUNT(&both) > 0 && sched_setaffinity(0, sizeof(both), &both) == 0) {
      scope->narrowed = true;
      return std::string("mbind refused (") + std::strerror(mbind_errno) + "): pinned from the CPUs of node " + std::to_string(node);
    }
  }
  return std::string("mbind refused (") + std::strerror(mbind_errno) + "): first touch";
}

extern "C" int b200kv_engine_create(const b200kv_engine_config* cfg, b200kv_pool* pool,
                                    b200kv_ctx** out) {
  if (!cfg || !out) return B200KV_EINVAL;
  *out = nullptr;
  b200kv_ctx* ctx = nullptr;
  const int rc = engine_create_impl(cfg, pool, &ctx);
  if (rc != B200KV_OK) {
    if (ctx) b200kv_engine_destroy(ctx);  // releases whatever had been created (streams, buffers, pinning)
    return rc;
  }
  *out = ctx;
  return B200KV_OK;
}

// The staging ring: as many chunk_bytes slots as staging_bytes holds.  The new ring is built completely before it
// replaces the engine's current one (b200kv_set_indexer re-cuts the ring for its larger chunk before any op has used
// it), so a refusal or a failed allocation leaves the engine with the ring it had.
static int make_staging(b200kv_ctx* ctx, uint64_t chunk_bytes) {
  const uint64_t n_stage = ctx->cfg.staging_bytes / chunk_bytes;
  if (ctx->pool && n_stage < 2) return B200KV_EINVAL;  // store/load need one staging chunk each
  uint8_t* buf = nullptr;
  std::vector<StageSlot> ring(n_stage);
  if (n_stage > 0) {
    cudaError_t e = cudaMalloc(&buf, n_stage * chunk_bytes);
    for (size_t i = 0; e == cudaSuccess && i < ring.size(); ++i)
      e = cudaEventCreateWithFlags(&ring[i].free_ev, cudaEventDisableTiming);
    if (e != cudaSuccess) {
      set_err("staging ring", e, __LINE__);
      for (auto& r : ring)
        if (r.free_ev) cudaEventDestroy(r.free_ev);
      if (buf) cudaFree(buf);
      return B200KV_ENODEV;
    }
  }
  for (auto& r : ctx->stage)
    if (r.free_ev) cudaEventDestroy(r.free_ev);
  if (ctx->d_staging) cudaFree(ctx->d_staging);
  ctx->d_staging = buf;
  ctx->stage = std::move(ring);
  ctx->n_store_slots = static_cast<uint32_t>(n_stage / 2);
  ctx->store_next = ctx->load_next = 0;
  return B200KV_OK;
}

static int engine_create_impl(const b200kv_engine_config* cfg, b200kv_pool* pool, b200kv_ctx** out) {
  Geometry g;
  int rc = make_geometry(cfg, &g);
  if (rc) return rc;
  if (cfg->block_stride_bytes < static_cast<uint64_t>(g.bs) * g.token_bytes ||
      cfg->block_stride_bytes % 16 || cfg->n_blocks == 0 ||
      cfg->n_blocks * g.bs > 0x7fffffffull)
    return B200KV_EINVAL;

  int n_dev = 0;
  if (cudaGetDeviceCount(&n_dev) != cudaSuccess || n_dev == 0) {
    std::snprintf(g_err, sizeof(g_err),
                  "no CUDA device: libb200kv has no CPU fallback (the oracle/ directory is test "
                  "infrastructure only)");
    return B200KV_ENODEV;
  }
  if (cfg->device < 0 || cfg->device >= n_dev) return B200KV_EINVAL;
  DeviceGuard dg(cfg->device);
  if (!dg.ok) return B200KV_ENODEV;

  cudaDeviceProp prop;
  CU_TRY(cudaGetDeviceProperties(&prop, cfg->device));
  if (prop.major != 9 || prop.minor != 0) {
    std::snprintf(g_err, sizeof(g_err), "device %d is sm_%d%d; this library is built for sm_90a only",
                  cfg->device, prop.major, prop.minor);
    return B200KV_ENOTSUP;
  }

  b200kv_ctx* ctx = new (std::nothrow) b200kv_ctx();
  if (!ctx) return B200KV_ENOMEM;
  *out = ctx;  // from here on the caller destroys it on failure
  ctx->cfg = *cfg;
  ctx->g = g;
  ctx->pool = pool;
  ctx->sm_count = prop.multiProcessorCount;

  // launch shape of the bulk kernel
  ctx->S = cfg->stages > 0 ? cfg->stages : env_int("B200KV_STAGES", 2);
  ctx->LAG = env_int("B200KV_LAG", ctx->S / 2);
  ctx->ctas_per_sm = cfg->ctas_per_sm > 0 ? cfg->ctas_per_sm : env_int("B200KV_CTAS_PER_SM", 1);
  ctx->fp8_store3 = cfg->format == B200KV_FMT_FP8 && !g.mla && env_int("B200KV_FP8_STORE", 3) == 3 &&
                    fp8_store3_fits(g);
  const uint32_t stage_max = static_cast<uint32_t>(env_int("B200KV_STAGE_KB", 32)) << 10;
  if (g.token_bytes > stage_max || stage_max > kStageMax * 2) return B200KV_ENOTSUP;
  ctx->piece_tokens = std::min<uint32_t>(g.bs, stage_max / g.token_bytes);
  ctx->pieces = (g.bs + ctx->piece_tokens - 1) / ctx->piece_tokens;
  ctx->stage_bytes = ctx->piece_tokens * g.token_bytes;
  if (256 + static_cast<size_t>(ctx->S) * ctx->stage_bytes > 227u * 1024) return B200KV_EINVAL;

  int lo_pri = 0, hi_pri = 0;
  CU_TRY(cudaDeviceGetStreamPriorityRange(&lo_pri, &hi_pri));
  CU_TRY(cudaStreamCreateWithPriority(&ctx->s_gather, cudaStreamNonBlocking, lo_pri));
  CU_TRY(cudaStreamCreateWithPriority(&ctx->s_d2h, cudaStreamNonBlocking, lo_pri));
  CU_TRY(cudaStreamCreateWithPriority(&ctx->s_h2d, cudaStreamNonBlocking, hi_pri));
  CU_TRY(cudaStreamCreateWithPriority(&ctx->s_scatter, cudaStreamNonBlocking, hi_pri));
  CU_TRY(cudaEventCreateWithFlags(&ctx->fence, cudaEventDisableTiming));

  // dynamic shared memory past 48 KiB, set on this device for the kernels this engine can launch; a
  // B200KV_STAGES / B200KV_LAG pair that is not built fails at launch instead
  if (cfg->variant != B200KV_VARIANT_LDG) {
    for (BulkKernel k : {bulk_kernel<kStore>(ctx->S, ctx->LAG), bulk_kernel<kLoad>(ctx->S, ctx->LAG),
                         bulk_kernel<kPull>(ctx->S, ctx->LAG)})
      if (k) CU_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
  }
  if (cfg->format == B200KV_FMT_FP8 && !g.mla) {   // both element types: b200kv_set_cache_dtype comes later
    CU_TRY(cudaFuncSetAttribute(kv_fp8_store3_kernel<kBf16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                kS3Stages * kS3MaxUnitBytes));
    CU_TRY(cudaFuncSetAttribute(kv_fp8_store_kernel<kBf16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    CU_TRY(cudaFuncSetAttribute(kv_fp8_store3_kernel<kFp16>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                kS3Stages * kS3MaxUnitBytes));
    CU_TRY(cudaFuncSetAttribute(kv_fp8_store_kernel<kFp16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  }

  // 2*L slots, the most any geometry uses, so b200kv_set_indexer has nothing to allocate
  CU_TRY(cudaMalloc(&ctx->d_bases, sizeof(uint64_t) * 2 * g.L));

  rc = make_staging(ctx, g.chunk_bytes);
  if (rc) return rc;
  for (auto& t : ctx->tables) {
    CU_TRY(cudaHostAlloc(&t.host, kTableBytes, cudaHostAllocDefault));
    CU_TRY(cudaMalloc(&t.dev, kTableBytes));
    CU_TRY(cudaEventCreateWithFlags(&t.ev, cudaEventDisableTiming));
    CU_TRY(cudaEventCreateWithFlags(&t.done_ev, cudaEventDisableTiming));
  }

  if (pool) {
    void* base = nullptr;
    uint64_t bytes = 0;
    rc = b200kv_pool_region(pool, &base, &bytes);
    if (rc) return rc;
    b200kv_pool_stats ps;
    b200kv_pool_get_stats(pool, &ps);
    if (ps.slot_bytes < g.chunk_bytes) return B200KV_EINVAL;
    // Pin the (possibly shared) pool for this process so D2H/H2D run at full PCIe speed and
    // asynchronously.  Portable: every replica on the box registers the same segment.
    NumaPinScope numa_scope;
    ctx->numa_placement = place_pool_pages(base, bytes, cfg->device, cfg->numa_policy, &numa_scope);
    if (env_int("B200KV_VERBOSE", 0)) std::fprintf(stderr, "b200kv: pool pages: %s\n", ctx->numa_placement.c_str());
    const cudaError_t re = cudaHostRegister(base, bytes, cudaHostRegisterPortable);
    if (re == cudaSuccess) {
      ctx->pool_registered = true;
      ctx->pool_base = base;
    } else if (re == cudaErrorHostMemoryAlreadyRegistered) {
      cudaGetLastError();  // another engine of this process (e.g. a second GPU) pinned it already
    } else {
      set_err("cudaHostRegister(pool)", re, __LINE__);
      return B200KV_ENODEV;
    }
  }
  return B200KV_OK;
}

extern "C" int b200kv_wait_all(b200kv_ctx* ctx);

extern "C" int b200kv_engine_destroy(b200kv_ctx* ctx) {
  if (!ctx) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  b200kv_wait_all(ctx);
  cudaDeviceSynchronize();
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    reap(ctx);
    for (auto& kv : ctx->ops) destroy_op_events(kv.second.get());
    ctx->ops.clear();
  }
  if (ctx->pool_registered) cudaHostUnregister(ctx->pool_base);
  for (auto& p : ctx->peers) {
    if (!p.valid) continue;
    for (void* m : p.opened) cudaIpcCloseMemHandle(m);
    cudaFree(p.d_bases);
  }
  for (auto& t : ctx->tables) {
    if (t.host) cudaFreeHost(t.host);
    if (t.dev) cudaFree(t.dev);
    if (t.ev) cudaEventDestroy(t.ev);
    if (t.done_ev) cudaEventDestroy(t.done_ev);
  }
  for (auto& s : ctx->stage)
    if (s.free_ev) cudaEventDestroy(s.free_ev);
  for (auto& t : ctx->timing)
    for (auto& e : t.ev) {
      cudaEventDestroy(e.first);
      cudaEventDestroy(e.second);
    }
  if (ctx->d_staging) cudaFree(ctx->d_staging);
  for (void* m : ctx->tier_imports) cudaIpcCloseMemHandle(m);
  if (ctx->tier_base) cudaFree(ctx->tier_base);
  if (ctx->d_bases) cudaFree(ctx->d_bases);
  if (ctx->d_tmaps) cudaFree(ctx->d_tmaps);
  if (ctx->fence) cudaEventDestroy(ctx->fence);
  for (cudaStream_t s : {ctx->s_gather, ctx->s_d2h, ctx->s_h2d, ctx->s_scatter})
    if (s) cudaStreamDestroy(s);
  delete ctx;
  return B200KV_OK;
}

// One 4-D tensor map per plane over NHD pages, so that TMA can fetch "the bs rows of head h in block b" — a
// [bs][D] box whose rows are a token apart — as ONE copy (SASS UTMALDG).  Dimensions are ordered by ascending
// stride: {D, H, bs, NB}, box {D, 1, bs, 1}, which lands as [bs][D] in shared memory.  HND pages need no map:
// those rows are contiguous and a plain bulk copy fetches them.  Failure is not fatal: the FP8 store then runs
// its cluster kernel.
static void build_tensor_maps(b200kv_ctx* ctx, const std::vector<uint64_t>& bases) {
  const Geometry& g = ctx->g;
  if (ctx->cfg.format != B200KV_FMT_FP8 || g.elem != 2 || g.hnd || g.mla) { ctx->tmap_status = "not needed"; return; }
  typedef CUresult (*EncodeFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                               const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                               CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q) != cudaSuccess || !fn ||
      q != cudaDriverEntryPointSuccess) {
    cudaGetLastError();
    ctx->tmap_status = "cuTensorMapEncodeTiled unavailable";
    return;
  }
  if (g.D > 256 || g.bs > 256) { ctx->tmap_status = "box too large"; return; }
  std::vector<CUtensorMap> maps(g.planes);
  const cuuint64_t row = static_cast<cuuint64_t>(g.D) * g.elem, tok = g.token_bytes, blk = ctx->cfg.block_stride_bytes;
  for (uint32_t pl = 0; pl < g.planes; ++pl) {
    const cuuint64_t dims[4] = {g.D, g.H, g.bs, ctx->cfg.n_blocks}, strides[3] = {row, tok, blk};
    const cuuint32_t box[4] = {g.D, 1, g.bs, 1}, estr[4] = {1, 1, 1, 1};
    const CUresult r = reinterpret_cast<EncodeFn>(fn)(&maps[pl], CU_TENSOR_MAP_DATA_TYPE_UINT16, 4,
                                                      reinterpret_cast<void*>(bases[pl]), dims, strides, box, estr,
                                                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                                                      CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) {
      ctx->tmap_status = "cuTensorMapEncodeTiled failed (" + std::to_string(static_cast<int>(r)) + ")";
      return;
    }
  }
  if (!ctx->d_tmaps && cudaMalloc(&ctx->d_tmaps, sizeof(CUtensorMap) * g.planes) != cudaSuccess) {
    cudaGetLastError();
    ctx->d_tmaps = nullptr;
    ctx->tmap_status = "cudaMalloc failed";
    return;
  }
  if (cudaMemcpy(ctx->d_tmaps, maps.data(), sizeof(CUtensorMap) * g.planes, cudaMemcpyHostToDevice) != cudaSuccess) {
    cudaGetLastError();
    cudaFree(ctx->d_tmaps);
    ctx->d_tmaps = nullptr;
    ctx->tmap_status = "cudaMemcpy failed";
    return;
  }
  ctx->tmap_status = "ok";
}

extern "C" int b200kv_set_cache_dtype(b200kv_ctx* ctx, int32_t dtype) {
  if (!ctx || (dtype != B200KV_DTYPE_BF16 && dtype != B200KV_DTYPE_FP16 && dtype != B200KV_DTYPE_E5M2))
    return B200KV_EINVAL;
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ctx->kv_registered) return B200KV_EBUSY;   // chunks already stored or moved under the old type
  if (dtype == B200KV_DTYPE_FP16 && ctx->g.elem != 2) return B200KV_EINVAL;
  if (dtype == B200KV_DTYPE_E5M2 && ctx->g.elem != 1) return B200KV_EINVAL;
  ctx->g.dtype = static_cast<uint32_t>(dtype);
  return B200KV_OK;
}

extern "C" int b200kv_set_indexer(b200kv_ctx* ctx, int32_t value_bytes, int32_t scale_bytes,
                                  uint64_t block_stride_bytes) {
  if (!ctx) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ctx->kv_registered || ctx->tier_base) return B200KV_EBUSY;   // pages or tier slots sized without the planes
  if (!ctx->g.mla) return B200KV_EINVAL;
  Geometry g;
  int rc = make_geometry(&ctx->cfg, &g);
  if (rc) return rc;
  g.dtype = ctx->g.dtype;
  rc = add_indexer(&g, value_bytes, scale_bytes, block_stride_bytes);
  if (rc) return rc;
  // everything that can refuse is checked before the staging ring is rebuilt
  if (indexer_smem_bytes(g) > 227u * 1024) return B200KV_ENOTSUP;
  const uint64_t n_stage = ctx->cfg.staging_bytes / g.chunk_bytes;
  if (ctx->pool) {
    b200kv_pool_stats ps;
    b200kv_pool_get_stats(ctx->pool, &ps);
    if (ps.slot_bytes < g.chunk_bytes || n_stage < 2) return B200KV_EINVAL;
  }
  typedef void (*IndexerKernel)(KernelArgs);
  for (IndexerKernel k : {kv_indexer_copy_kernel<kStore>, kv_indexer_copy_kernel<kLoad>, kv_indexer_copy_kernel<kPull>})
    CU_TRY(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(indexer_smem_bytes(g))));
  rc = make_staging(ctx, g.chunk_bytes);   // the engine keeps its geometry and ring if this fails
  if (rc) return rc;
  ctx->g = g;
  return B200KV_OK;
}

extern "C" int b200kv_register_kv(b200kv_ctx* ctx, const void* const* k_ptrs,
                                  const void* const* v_ptrs) {
  if (!ctx) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  // the Q4 kernels of fp8 pages decode e4m3 or e5m2 codes: no other type may reach them
  if (ctx->cfg.format == B200KV_FMT_Q4 && ctx->g.elem == 1 && ctx->g.dtype != B200KV_DTYPE_E4M3 &&
      ctx->g.dtype != B200KV_DTYPE_E5M2)
    return B200KV_EINVAL;
  std::vector<uint64_t> h;
  const int rc = plane_bases(ctx->g, k_ptrs, v_ptrs, &h);
  if (rc) return rc;
  CU_TRY(cudaMemcpy(ctx->d_bases, h.data(), sizeof(uint64_t) * h.size(), cudaMemcpyHostToDevice));
  ctx->h_bases = std::move(h);
  build_tensor_maps(ctx, ctx->h_bases);
  if (env_int("B200KV_VERBOSE", 0)) std::fprintf(stderr, "b200kv: tensor maps: %s\n", ctx->tmap_status.c_str());
  ctx->kv_registered = true;
  return B200KV_OK;
}

// ------------------------------------------------------------------------------------------------
// device-resident gather / scatter
// ------------------------------------------------------------------------------------------------
static int gather_scatter(b200kv_ctx* ctx, const int64_t* slots, int64_t n_tokens, void* dev_chunks,
                          void* stream, bool is_gather, const uint64_t* chunk_ptrs = nullptr) {
  if (!ctx || !slots || n_tokens <= 0 || (!dev_chunks && !chunk_ptrs)) return B200KV_EINVAL;
  if (!ctx->kv_registered) return B200KV_EINVAL;
  if (reinterpret_cast<uint64_t>(dev_chunks) % 16) return B200KV_EINVAL;
  if (chunk_ptrs) {
    const int64_t n = (n_tokens + ctx->g.C - 1) / ctx->g.C;
    for (int64_t c = 0; c < n; ++c)
      if (!chunk_ptrs[c] || chunk_ptrs[c] % 16) return B200KV_EINVAL;
  }
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  const Geometry& g = ctx->g;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const uint32_t n_chunks = static_cast<uint32_t>((n_tokens + g.C - 1) / g.C);

  std::vector<Span> spans(n_chunks);
  std::vector<uint64_t> addrs(n_chunks);
  for (uint32_t c = 0; c < n_chunks; ++c) {
    const int64_t tb = static_cast<int64_t>(c) * g.C;
    spans[c] = {tb, std::min<int64_t>(g.C, n_tokens - tb)};
    addrs[c] = chunk_ptrs ? chunk_ptrs[c]
                          : reinterpret_cast<uint64_t>(dev_chunks) + static_cast<uint64_t>(c) * g.chunk_bytes;
  }
  OpTable table;
  int rc = op_table(ctx, slots, spans, &table);
  if (rc) return rc;
  TableView tv;
  rc = stage_table(ctx, table, addrs.data(), s, &tv);
  if (rc) return rc;

  const int which = is_gather ? kTimeGather : kTimeScatter;
  timing_reset(ctx, which);
  rc = timing_begin(ctx, which, s);
  if (rc) return rc;
  rc = launch_op(ctx, is_gather ? kStore : kLoad, table, tv, 0, n_chunks, s);
  if (rc) return rc;
  rc = timing_end(ctx, which, s);
  if (rc) return rc;
  CU_TRY(cudaEventRecord(tv.slot->done_ev, s));
  if (is_gather) ctx->stats.n_stored_tokens += n_tokens; else ctx->stats.n_loaded_tokens += n_tokens;
  return B200KV_OK;
}

extern "C" int b200kv_gather(b200kv_ctx* ctx, const int64_t* slot_mapping, int64_t n_tokens,
                             void* dev_chunks, void* stream) {
  return gather_scatter(ctx, slot_mapping, n_tokens, dev_chunks, stream, true);
}

extern "C" int b200kv_scatter(b200kv_ctx* ctx, const int64_t* slot_mapping, int64_t n_tokens,
                              const void* dev_chunks, void* stream) {
  return gather_scatter(ctx, slot_mapping, n_tokens, const_cast<void*>(dev_chunks), stream, false);
}

extern "C" int b200kv_gather_chunks(b200kv_ctx* ctx, const int64_t* slot_mapping, int64_t n_tokens,
                                    const uint64_t* chunk_ptrs, void* stream) {
  return gather_scatter(ctx, slot_mapping, n_tokens, nullptr, stream, true, chunk_ptrs);
}

extern "C" int b200kv_scatter_chunks(b200kv_ctx* ctx, const int64_t* slot_mapping, int64_t n_tokens,
                                     const uint64_t* chunk_ptrs, void* stream) {
  return gather_scatter(ctx, slot_mapping, n_tokens, nullptr, stream, false, chunk_ptrs);
}

// ------------------------------------------------------------------------------------------------
// device chunk tier: a buffer of chunk-format slots in HBM, exported to peer replicas over CUDA IPC.
// The index (which key sits in which slot, LRU, pins) is a b200kv_pool in shm owned by the host side.
// ------------------------------------------------------------------------------------------------
extern "C" int b200kv_tier_create(b200kv_ctx* ctx, uint32_t n_slots, uint64_t* base_out) {
  if (!ctx || !n_slots || !base_out) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ctx->tier_base) return B200KV_EEXIST;
  void* p = nullptr;
  CU_TRY(cudaMalloc(&p, static_cast<size_t>(n_slots) * ctx->g.chunk_bytes));
  ctx->tier_base = p;
  ctx->tier_slots = n_slots;
  *base_out = reinterpret_cast<uint64_t>(p);
  return B200KV_OK;
}

extern "C" int b200kv_tier_export(b200kv_ctx* ctx, b200kv_ipc_desc* desc_out) {
  if (!ctx || !desc_out || !ctx->tier_base) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::memset(desc_out, 0, sizeof(*desc_out));
  cudaIpcMemHandle_t h;
  CU_TRY(cudaIpcGetMemHandle(&h, ctx->tier_base));
  std::memcpy(desc_out->handle, &h, 64);
  desc_out->offset = 0;
  desc_out->alloc_bytes = static_cast<uint64_t>(ctx->tier_slots) * ctx->g.chunk_bytes;
  return B200KV_OK;
}

extern "C" int b200kv_tier_import(b200kv_ctx* ctx, const b200kv_ipc_desc* desc, uint64_t* mapped_base_out) {
  if (!ctx || !desc || !mapped_base_out) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  cudaIpcMemHandle_t h;
  std::memcpy(&h, desc->handle, 64);
  void* base = nullptr;
  CU_TRY(cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess));
  ctx->tier_imports.push_back(base);
  *mapped_base_out = reinterpret_cast<uint64_t>(base) + desc->offset;
  return B200KV_OK;
}

// ------------------------------------------------------------------------------------------------
// store: paged HBM -> staging (kernel) -> pinned pool (DMA)
// ------------------------------------------------------------------------------------------------
// Chunk c of the op holds chunk_tokens[c] tokens whose slots are slot_mapping[c*C .. c*C + chunk_tokens[c]): a
// single request (every chunk full but the last) or the chunks of SEVERAL requests back to back, each
// request's tail padded to the chunk size (b200kv_store_batch_async: one table, one launch per staging
// batch and one ticket for a whole engine step).
static int store_impl(b200kv_ctx* ctx, const uint64_t* keys, const int32_t* chunk_tokens, int32_t n_chunks,
                      const int64_t* slot_mapping, void* compute_stream, uint64_t* ticket) {
  if (!ctx || !keys || !chunk_tokens || !slot_mapping || n_chunks <= 0 || !ticket) return B200KV_EINVAL;
  if (!ctx->pool || !ctx->kv_registered || ctx->stage.empty()) return B200KV_EINVAL;
  const Geometry& g = ctx->g;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  reap(ctx);
  cudaStream_t cs = static_cast<cudaStream_t>(compute_stream);
  *ticket = 0;

  // 0. validate every slot BEFORE touching the pool: a malformed mapping must not leave chunks
  //    reserved-but-never-committed
  int rc = check_chunk_slots(ctx, slot_mapping, chunk_tokens, n_chunks);
  if (rc) return rc;
  // 1. reserve pool slots; chunks already present (or not placeable) are skipped
  struct Todo { int32_t c; uint32_t slot; uint32_t n_tok; };
  std::vector<Todo> todo;
  OpGuard guard(ctx, ctx->s_gather, ctx->s_d2h, nullptr, nullptr);   // undoes the reservations on any early return
  for (int32_t c = 0; c < n_chunks; ++c) {
    const uint32_t n_tok = static_cast<uint32_t>(chunk_tokens[c]);
    uint32_t slot = 0;
    rc = b200kv_pool_reserve(ctx->pool, keys[c], static_cast<int32_t>(n_tok), pool_fmt(ctx), ctx->cfg.owner, &slot);
    if (rc == B200KV_OK) { todo.push_back({c, slot, n_tok}); guard.reserved.push_back(keys[c]); }
    else if (rc != B200KV_EEXIST && rc != B200KV_ENOSPC) return rc;
  }
  ++ctx->stats.n_store_ops;
  if (todo.empty()) return B200KV_OK;

  guard.op.reset(new Op());
  Op* op = guard.op.get();
  op->id = ctx->next_ticket++;
  op->pool = ctx->pool;
  CU_TRY(cudaEventCreateWithFlags(&op->done, cudaEventDisableTiming));
  rc = stream_wait(ctx, ctx->s_gather, cs);
  if (rc) return rc;

  timing_reset(ctx, kTimeGather);
  const size_t n_stage = ctx->n_store_slots;
  for (size_t b0 = 0; b0 < todo.size(); b0 += n_stage) {
    const size_t nb = std::min(n_stage, todo.size() - b0);
    std::vector<Span> spans(nb);
    for (size_t i = 0; i < nb; ++i) spans[i] = {static_cast<int64_t>(todo[b0 + i].c) * g.C, todo[b0 + i].n_tok};
    OpTable table;
    rc = op_table(ctx, slot_mapping, spans, &table);
    if (rc) return rc;
    std::vector<uint64_t> addrs(nb);
    std::vector<uint32_t> sidx(nb);
    for (size_t i = 0; i < nb; ++i) {
      sidx[i] = ctx->store_next;
      ctx->store_next = (ctx->store_next + 1) % static_cast<uint32_t>(n_stage);
      addrs[i] = reinterpret_cast<uint64_t>(ctx->d_staging) + static_cast<uint64_t>(sidx[i]) * g.chunk_bytes;
      if (ctx->stage[sidx[i]].used) CU_TRY(cudaStreamWaitEvent(ctx->s_gather, ctx->stage[sidx[i]].free_ev, 0));
    }
    TableView tv;
    rc = stage_table(ctx, table, addrs.data(), ctx->s_gather, &tv);
    if (rc) return rc;

    rc = timing_begin(ctx, kTimeGather, ctx->s_gather);
    if (rc) return rc;
    rc = launch_op(ctx, kStore, table, tv, 0, static_cast<uint32_t>(nb), ctx->s_gather);
    if (rc) return rc;
    rc = timing_end(ctx, kTimeGather, ctx->s_gather);
    if (rc) return rc;
    CU_TRY(cudaEventRecord(tv.slot->done_ev, ctx->s_gather));
    // the pages may be reused as soon as the gather is done: compute waits for the kernel only
    CU_TRY(cudaStreamWaitEvent(cs, tv.slot->done_ev, 0));
    CU_TRY(cudaStreamWaitEvent(ctx->s_d2h, tv.slot->done_ev, 0));
    for (size_t i = 0; i < nb; ++i) {
      const Todo& t = todo[b0 + i];
      rc = copy_chunk_planes(ctx, b200kv_pool_slot_ptr(ctx->pool, t.slot), reinterpret_cast<void*>(addrs[i]),
                             t.n_tok, cudaMemcpyDeviceToHost, ctx->s_d2h);
      if (rc) return rc;
      CU_TRY(cudaEventRecord(ctx->stage[sidx[i]].free_ev, ctx->s_d2h));
      ctx->stage[sidx[i]].used = true;
      op->commit_keys.push_back(keys[t.c]);
      ctx->stats.n_stored_tokens += t.n_tok;
    }
  }
  // chunks whose D2H was never queued (none on this path) would stay reserved: every todo chunk is in commit_keys
  CU_TRY(cudaLaunchHostFunc(ctx->s_d2h, op_host_cb, op));
  guard.cb_enqueued = true;
  CU_TRY(cudaEventRecord(op->done, ctx->s_d2h));
  *ticket = op->id;
  ctx->ops.emplace(op->id, std::move(guard.op));
  guard.armed = false;
  return B200KV_OK;
}

extern "C" int b200kv_store_async(b200kv_ctx* ctx, const uint64_t* keys, int32_t n_chunks,
                                  const int64_t* slot_mapping, int64_t n_tokens,
                                  void* compute_stream, uint64_t* ticket) {
  if (!ctx || n_tokens <= 0) return B200KV_EINVAL;
  const int64_t C = ctx->g.C;
  if (n_chunks != static_cast<int32_t>((n_tokens + C - 1) / C)) return B200KV_EINVAL;
  std::vector<int32_t> ct(static_cast<size_t>(n_chunks));
  for (int32_t c = 0; c < n_chunks; ++c) ct[c] = static_cast<int32_t>(std::min<int64_t>(C, n_tokens - c * C));
  return store_impl(ctx, keys, ct.data(), n_chunks, slot_mapping, compute_stream, ticket);
}

extern "C" int b200kv_store_batch_async(b200kv_ctx* ctx, const uint64_t* keys, const int32_t* chunk_tokens,
                                        int32_t n_chunks, const int64_t* slot_mapping, void* compute_stream,
                                        uint64_t* ticket) {
  return store_impl(ctx, keys, chunk_tokens, n_chunks, slot_mapping, compute_stream, ticket);
}

// ------------------------------------------------------------------------------------------------
// load: pinned pool -> staging (DMA) -> paged HBM (kernel), pipelined per chunk
// ------------------------------------------------------------------------------------------------
// Chunk layout as in store_impl.  Request r owns chunks [req_first[r], req_first[r+1]); each request is loaded
// up to its first missing chunk (prefix semantics of lmcache_engine.retrieve), independently of the others.
static int load_impl(b200kv_ctx* ctx, const uint64_t* keys, const int32_t* chunk_tokens, int32_t n_chunks,
                     const int32_t* req_first, int32_t n_reqs, const int64_t* slot_mapping, void* compute_stream,
                     uint64_t* ticket, int64_t* req_loaded, int32_t layers_per_group) {
  if (!ctx || !keys || !chunk_tokens || !req_first || !slot_mapping || n_chunks <= 0 || n_reqs <= 0 || !ticket ||
      layers_per_group < 0)
    return B200KV_EINVAL;
  if (!ctx->pool || !ctx->kv_registered || ctx->stage.empty()) return B200KV_EINVAL;
  const Geometry& g = ctx->g;
  if (req_first[0] != 0 || req_first[n_reqs] != n_chunks) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  reap(ctx);
  cudaStream_t cs = static_cast<cudaStream_t>(compute_stream);
  *ticket = 0;
  if (req_loaded) std::fill(req_loaded, req_loaded + n_reqs, 0);
  int rc = check_chunk_slots(ctx, slot_mapping, chunk_tokens, n_chunks);   // before pinning anything
  if (rc) return rc;
  for (int32_t r = 0; r < n_reqs; ++r)
    if (req_first[r] > req_first[r + 1]) return B200KV_EINVAL;

  struct Todo { int32_t c; uint32_t slot; uint32_t n_tok; };
  std::vector<Todo> todo;
  for (int32_t r = 0; r < n_reqs; ++r) {
    for (int32_t c = req_first[r]; c < req_first[r + 1]; ++c) {
      const uint32_t want = static_cast<uint32_t>(chunk_tokens[c]);
      uint32_t slot = 0, fmt = 0;
      int32_t have = 0;
      if (b200kv_pool_acquire(ctx->pool, keys[c], &slot, &have, &fmt) != B200KV_OK) break;
      if (static_cast<uint32_t>(have) != want || fmt != pool_fmt(ctx)) {
        b200kv_pool_release(ctx->pool, keys[c]);
        break;
      }
      todo.push_back({c, slot, want});
      if (req_loaded) req_loaded[r] += want;
    }
  }
  ++ctx->stats.n_load_ops;
  if (todo.empty()) return B200KV_OK;

  OpGuard guard(ctx, ctx->s_h2d, ctx->s_scatter, nullptr, nullptr);
  guard.op.reset(new Op());
  Op* op = guard.op.get();
  op->id = ctx->next_ticket++;
  op->pool = ctx->pool;
  for (const Todo& t : todo) op->release_keys.push_back(keys[t.c]);
  // From here on every early return drops the pins and the op's events through `guard` (not every failure
  // below is fatal: stage_table refuses an op whose run table does not fit).
  CU_TRY(cudaEventCreateWithFlags(&op->done, cudaEventDisableTiming));

  const bool detached = compute_stream == B200KV_STREAM_DETACHED;
  if (!detached) {
    rc = stream_wait(ctx, ctx->s_scatter, cs);
    if (rc) return rc;
  }

  timing_reset(ctx, kTimeScatter);
  const size_t n_stage = ctx->stage.size() - ctx->n_store_slots;
  int64_t loaded = 0;
  // Layer-wise: every chunk must own a staging slot for the whole op (the groups of all chunks are
  // interleaved); an op larger than the load half of the ring falls back to the chunk-wise path.
  const bool layerwise = layers_per_group > 0 && todo.size() <= n_stage;
  const size_t batch = layerwise ? todo.size() : n_stage;
  for (size_t b0 = 0; b0 < todo.size(); b0 += batch) {
    const uint32_t nb = static_cast<uint32_t>(std::min(batch, todo.size() - b0));
    std::vector<Span> spans(nb);
    for (uint32_t i = 0; i < nb; ++i) spans[i] = {static_cast<int64_t>(todo[b0 + i].c) * g.C, todo[b0 + i].n_tok};
    OpTable table;
    rc = op_table(ctx, slot_mapping, spans, &table);
    if (rc) return rc;
    std::vector<uint64_t> addrs(nb);
    std::vector<uint32_t> sidx(nb);
    for (uint32_t i = 0; i < nb; ++i) {
      sidx[i] = ctx->n_store_slots + ctx->load_next;
      ctx->load_next = (ctx->load_next + 1) % static_cast<uint32_t>(n_stage);
      addrs[i] = reinterpret_cast<uint64_t>(ctx->d_staging) + static_cast<uint64_t>(sidx[i]) * g.chunk_bytes;
      if (layerwise && ctx->stage[sidx[i]].used) CU_TRY(cudaStreamWaitEvent(ctx->s_h2d, ctx->stage[sidx[i]].free_ev, 0));
    }
    TableView tv;
    rc = stage_table(ctx, table, addrs.data(), ctx->s_scatter, &tv);
    if (rc) return rc;

    if (layerwise) {
      const uint32_t G = static_cast<uint32_t>(layers_per_group);
      const uint32_t n_groups = (g.L + G - 1) / G;
      op->layers_per_group = layers_per_group;
      op->group_ev.resize(n_groups, nullptr);
      for (uint32_t gi = 0; gi < n_groups; ++gi) {
        const uint32_t pb = g.planes_per_layer * gi * G;
        const uint32_t np = std::min<uint32_t>(g.planes_per_layer * G, g.planes - pb);
        for (uint32_t i = 0; i < nb; ++i) {
          const Todo& t = todo[b0 + i];
          rc = copy_chunk_planes(ctx, reinterpret_cast<void*>(addrs[i]), b200kv_pool_slot_ptr(ctx->pool, t.slot),
                                 t.n_tok, cudaMemcpyHostToDevice, ctx->s_h2d, pb, np, gi == 0);
          if (rc) return rc;
        }
        rc = stream_wait(ctx, ctx->s_scatter, ctx->s_h2d);   // this group of every chunk has landed
        if (rc) return rc;
        rc = timing_begin(ctx, kTimeScatter, ctx->s_scatter);
        if (rc) return rc;
        // RAW: one launch per chunk, as on the chunk-wise path
        const uint32_t step = ctx->cfg.format == B200KV_FMT_RAW ? 1 : nb;
        for (uint32_t c = 0; c < nb && rc == B200KV_OK; c += step)
          rc = launch_op(ctx, kLoad, table, tv, c, c + step, ctx->s_scatter, pb, np);
        if (rc) return rc;
        rc = timing_end(ctx, kTimeScatter, ctx->s_scatter);
        if (rc) return rc;
        CU_TRY(cudaEventCreateWithFlags(&op->group_ev[gi], cudaEventDisableTiming));
        CU_TRY(cudaEventRecord(op->group_ev[gi], ctx->s_scatter));
      }
      for (uint32_t i = 0; i < nb; ++i) {
        CU_TRY(cudaEventRecord(ctx->stage[sidx[i]].free_ev, ctx->s_scatter));
        ctx->stage[sidx[i]].used = true;
        loaded += todo[b0 + i].n_tok;
      }
    } else {
      for (uint32_t i = 0; i < nb; ++i) {
        const Todo& t = todo[b0 + i];
        StageSlot& ss = ctx->stage[sidx[i]];
        if (ss.used) CU_TRY(cudaStreamWaitEvent(ctx->s_h2d, ss.free_ev, 0));
        rc = copy_chunk_planes(ctx, reinterpret_cast<void*>(addrs[i]), b200kv_pool_slot_ptr(ctx->pool, t.slot),
                               t.n_tok, cudaMemcpyHostToDevice, ctx->s_h2d);
        if (rc) return rc;
        CU_TRY(cudaEventRecord(ss.free_ev, ctx->s_h2d));  // reused as "chunk landed" first ...
        CU_TRY(cudaStreamWaitEvent(ctx->s_scatter, ss.free_ev, 0));
        rc = timing_begin(ctx, kTimeScatter, ctx->s_scatter);
        if (rc) return rc;
        rc = launch_op(ctx, kLoad, table, tv, i, i + 1, ctx->s_scatter);
        if (rc) return rc;
        rc = timing_end(ctx, kTimeScatter, ctx->s_scatter);
        if (rc) return rc;
        CU_TRY(cudaEventRecord(ss.free_ev, ctx->s_scatter));  // ... then as "slot drained"
        ss.used = true;
        loaded += t.n_tok;
      }
    }
    CU_TRY(cudaEventRecord(tv.slot->done_ev, ctx->s_scatter));
  }
  CU_TRY(cudaLaunchHostFunc(ctx->s_scatter, op_host_cb, op));
  guard.cb_enqueued = true;
  CU_TRY(cudaEventRecord(op->done, ctx->s_scatter));
  // chunk-wise: the forward pass must see the loaded pages; layer-wise: it waits per layer instead
  if (!detached && !layerwise) CU_TRY(cudaStreamWaitEvent(cs, op->done, 0));
  ctx->stats.n_loaded_tokens += loaded;
  *ticket = op->id;
  ctx->ops.emplace(op->id, std::move(guard.op));
  guard.armed = false;
  return B200KV_OK;
}

static int load_single(b200kv_ctx* ctx, const uint64_t* keys, int32_t n_chunks, const int64_t* slot_mapping,
                       int64_t n_tokens, int32_t skip_chunks, void* compute_stream, uint64_t* ticket,
                       int64_t* n_loaded_tokens, int32_t layers_per_group) {
  if (!ctx || !keys || !slot_mapping || n_tokens <= 0 || !ticket || skip_chunks < 0) return B200KV_EINVAL;
  const int64_t C = ctx->g.C;
  if (n_chunks != static_cast<int32_t>((n_tokens + C - 1) / C)) return B200KV_EINVAL;
  if (ticket) *ticket = 0;
  if (n_loaded_tokens) *n_loaded_tokens = 0;
  std::vector<int32_t> ct(static_cast<size_t>(n_chunks));
  for (int32_t c = 0; c < n_chunks; ++c) ct[c] = static_cast<int32_t>(std::min<int64_t>(C, n_tokens - c * C));
  // slots of the masked prefix are validated too (the old single-request contract); load_impl checks the rest
  const int32_t skip = std::min(skip_chunks, n_chunks);
  const int rc_skip = check_chunk_slots(ctx, slot_mapping, ct.data(), skip);
  if (rc_skip) return rc_skip;
  if (skip == n_chunks) return (ctx->pool && ctx->kv_registered && !ctx->stage.empty()) ? B200KV_OK : B200KV_EINVAL;
  const int32_t first[2] = {0, n_chunks - skip};
  int64_t loaded = 0;
  const int rc = load_impl(ctx, keys + skip, ct.data() + skip, n_chunks - skip, first, 1, slot_mapping + skip * C,
                           compute_stream, ticket, &loaded, layers_per_group);
  if (rc == B200KV_OK && n_loaded_tokens) *n_loaded_tokens = loaded;
  return rc;
}

extern "C" int b200kv_load_async(b200kv_ctx* ctx, const uint64_t* keys, int32_t n_chunks,
                                 const int64_t* slot_mapping, int64_t n_tokens, int32_t skip_chunks,
                                 void* compute_stream, uint64_t* ticket, int64_t* n_loaded_tokens) {
  return load_single(ctx, keys, n_chunks, slot_mapping, n_tokens, skip_chunks, compute_stream, ticket,
                     n_loaded_tokens, 0);
}

extern "C" int b200kv_load_layerwise_async(b200kv_ctx* ctx, const uint64_t* keys, int32_t n_chunks,
                                           const int64_t* slot_mapping, int64_t n_tokens, int32_t skip_chunks,
                                           int32_t layers_per_group, void* compute_stream, uint64_t* ticket,
                                           int64_t* n_loaded_tokens) {
  if (layers_per_group <= 0) return B200KV_EINVAL;
  return load_single(ctx, keys, n_chunks, slot_mapping, n_tokens, skip_chunks, compute_stream, ticket,
                     n_loaded_tokens, layers_per_group);
}

extern "C" int b200kv_load_batch_async(b200kv_ctx* ctx, const uint64_t* keys, const int32_t* chunk_tokens,
                                       int32_t n_chunks, const int32_t* req_first_chunk, int32_t n_reqs,
                                       const int64_t* slot_mapping, int32_t layers_per_group, void* compute_stream,
                                       uint64_t* ticket, int64_t* req_loaded_tokens) {
  return load_impl(ctx, keys, chunk_tokens, n_chunks, req_first_chunk, n_reqs, slot_mapping, compute_stream, ticket,
                   req_loaded_tokens, layers_per_group);
}

extern "C" int b200kv_wait_layer(b200kv_ctx* ctx, uint64_t ticket, int32_t layer, void* compute_stream) {
  if (!ctx || layer < 0) return B200KV_EINVAL;
  if (ticket == 0) return B200KV_OK;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  auto it = ctx->ops.find(ticket);
  if (it == ctx->ops.end()) return B200KV_OK;  // finished and reaped: the pages are already there
  Op* op = it->second.get();
  cudaStream_t cs = static_cast<cudaStream_t>(compute_stream);
  if (op->group_ev.empty()) {  // the op fell back to the chunk-wise path: wait for all of it
    CU_TRY(cudaStreamWaitEvent(cs, op->done, 0));
    return B200KV_OK;
  }
  const size_t gi = std::min<size_t>(static_cast<size_t>(layer / op->layers_per_group), op->group_ev.size() - 1);
  CU_TRY(cudaStreamWaitEvent(cs, op->group_ev[gi], 0));
  return B200KV_OK;
}

// ------------------------------------------------------------------------------------------------
// tickets
// ------------------------------------------------------------------------------------------------
extern "C" int b200kv_poll(b200kv_ctx* ctx, uint64_t ticket, int* done) {
  if (!ctx || !done) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  if (ticket == 0) { *done = 1; return B200KV_OK; }
  auto it = ctx->ops.find(ticket);
  if (it == ctx->ops.end()) { *done = 1; return B200KV_OK; }  // already reaped
  Op* op = it->second.get();
  const cudaError_t q = cudaEventQuery(op->done);
  if (q == cudaSuccess && op->host_done.load(std::memory_order_acquire)) {
    destroy_op_events(op);
    ctx->ops.erase(it);
    *done = 1;
  } else if (q == cudaSuccess || q == cudaErrorNotReady) {
    *done = 0;
  } else {
    set_err("cudaEventQuery", q, __LINE__);
    return B200KV_ENODEV;
  }
  return B200KV_OK;
}

extern "C" int b200kv_wait(b200kv_ctx* ctx, uint64_t ticket) {
  if (!ctx) return B200KV_EINVAL;
  if (ticket == 0) return B200KV_OK;
  DeviceGuard dg(ctx->cfg.device);
  cudaEvent_t ev = nullptr;
  {
    std::lock_guard<std::mutex> lk(ctx->mu);
    auto it = ctx->ops.find(ticket);
    if (it == ctx->ops.end()) return B200KV_OK;
    ev = it->second->done;
  }
  CU_TRY(cudaEventSynchronize(ev));
  std::lock_guard<std::mutex> lk(ctx->mu);
  auto it = ctx->ops.find(ticket);
  if (it != ctx->ops.end()) {
    while (!it->second->host_done.load(std::memory_order_acquire)) { /* callback precedes event */ }
    destroy_op_events(it->second.get());
    ctx->ops.erase(it);
  }
  return B200KV_OK;
}

extern "C" int b200kv_wait_all(b200kv_ctx* ctx) {
  if (!ctx) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  for (cudaStream_t s : {ctx->s_gather, ctx->s_d2h, ctx->s_h2d, ctx->s_scatter})
    if (s) CU_TRY(cudaStreamSynchronize(s));
  std::lock_guard<std::mutex> lk(ctx->mu);
  reap(ctx);
  return B200KV_OK;
}

// ------------------------------------------------------------------------------------------------
// peers
// ------------------------------------------------------------------------------------------------
extern "C" int b200kv_export_ipc(b200kv_ctx* ctx, b200kv_ipc_desc* descs_out, int32_t n_descs) {
  if (!ctx || !descs_out) return B200KV_EINVAL;
  const Geometry& g = ctx->g;
  if (!ctx->kv_registered || n_descs != static_cast<int32_t>(g.n_bases)) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  typedef CUresult (*GetRange)(CUdeviceptr*, size_t*, CUdeviceptr);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qr;
  CU_TRY(cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &qr));
  if (!fn || qr != cudaDriverEntryPointSuccess) return B200KV_ENODEV;
  GetRange get_range = reinterpret_cast<GetRange>(fn);
  for (uint32_t i = 0; i < g.n_bases; ++i) {
    const uint64_t p = ctx->h_bases[base_slot(g, i / g.L, i % g.L)];
    CUdeviceptr base = 0;
    size_t size = 0;
    if (get_range(&base, &size, static_cast<CUdeviceptr>(p)) != CUDA_SUCCESS) return B200KV_ENODEV;
    b200kv_ipc_desc& d = descs_out[i];
    std::memset(&d, 0, sizeof(d));
    cudaIpcMemHandle_t h;
    CU_TRY(cudaIpcGetMemHandle(&h, reinterpret_cast<void*>(base)));
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t is 64 bytes");
    std::memcpy(d.handle, &h, 64);
    d.offset = p - static_cast<uint64_t>(base);
    d.alloc_bytes = size;
  }
  return B200KV_OK;
}

// A head slice a K/V engine can pull (b200kv_import_peer_sliced): inside [0, peer_heads) and [0, H), whole 16-byte
// rows, and a peer block stride that holds a block of peer_heads heads.
static int check_slice(const Geometry& g, const b200kv_head_slice& sl, uint64_t peer_block_stride) {
  if (g.mla || g.row_bytes % 16) return B200KV_EINVAL;
  if (sl.peer_heads <= 0 || sl.peer_heads > 65536 || sl.n_heads <= 0 || sl.src_head0 < 0 || sl.dst_head0 < 0 ||
      sl.src_head0 + sl.n_heads > sl.peer_heads || sl.dst_head0 + sl.n_heads > static_cast<int32_t>(g.H))
    return B200KV_EINVAL;
  if (peer_block_stride < static_cast<uint64_t>(g.bs) * static_cast<uint64_t>(sl.peer_heads) * g.row_bytes)
    return B200KV_EINVAL;
  return B200KV_OK;
}

// Installs a peer whole or not at all: ctx->peers[peer_id] is written only once its base table is on the device,
// with its head slice when `slice` is given.  It then owns `opened`; on failure nothing of the peer is left, and the
// caller still owns `opened`.
static int install_peer(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device, const std::vector<uint64_t>& bases,
                        uint64_t stride, uint64_t n_blocks, std::vector<void*>* opened,
                        const b200kv_head_slice* slice) {
  if (ctx->peers[peer_id].valid) return B200KV_EEXIST;
  Peer p;
  if (slice) {
    p.sliced = true;
    p.slice = *slice;
  }
  CU_TRY(cudaMalloc(&p.d_bases, sizeof(uint64_t) * bases.size()));
  const cudaError_t e = cudaMemcpy(p.d_bases, bases.data(), sizeof(uint64_t) * bases.size(), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    cudaFree(p.d_bases);
    set_err("cudaMemcpy(peer bases)", e, __LINE__);
    return B200KV_ENODEV;
  }
  p.device = peer_device;
  p.block_stride = stride;
  p.n_blocks = n_blocks;
  p.opened = std::move(*opened);
  p.valid = true;
  ctx->peers[peer_id] = std::move(p);
  return B200KV_OK;
}

static int import_peer(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device, const b200kv_ipc_desc* descs,
                       int32_t n_descs, uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks,
                       const b200kv_head_slice* slice) {
  if (!ctx || !descs || peer_id < 0 || peer_id >= kMaxPeers) return B200KV_EINVAL;
  const Geometry& g = ctx->g;
  if (n_descs != static_cast<int32_t>(g.n_bases) || peer_n_blocks == 0 || peer_n_blocks * g.bs > 0x7fffffffull)
    return B200KV_EINVAL;
  if (slice && check_slice(g, *slice, peer_block_stride_bytes)) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  // one cudaIpcOpenMemHandle per distinct allocation
  std::vector<std::pair<std::string, void*>> seen;
  std::vector<void*> opened;
  std::vector<uint64_t> bases(g.n_bases);
  int rc = B200KV_OK;
  for (uint32_t i = 0; i < g.n_bases; ++i) {
    const b200kv_ipc_desc& d = descs[i];
    const std::string key(reinterpret_cast<const char*>(d.handle), 64);
    void* base = nullptr;
    for (auto& s : seen)
      if (s.first == key) base = s.second;
    if (!base) {
      cudaIpcMemHandle_t h;
      std::memcpy(&h, d.handle, 64);
      const cudaError_t e = cudaIpcOpenMemHandle(&base, h, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        set_err("cudaIpcOpenMemHandle", e, __LINE__);
        rc = B200KV_ENODEV;
        break;
      }
      seen.emplace_back(key, base);
      opened.push_back(base);
    }
    bases[base_slot(g, i / g.L, i % g.L)] = reinterpret_cast<uint64_t>(base) + d.offset;
  }
  if (rc == B200KV_OK)
    rc = install_peer(ctx, peer_id, peer_device, bases, peer_block_stride_bytes, peer_n_blocks, &opened, slice);
  if (rc)   // the mappings this call opened; install_peer took none of them
    for (void* m : opened) cudaIpcCloseMemHandle(m);
  return rc;
}

extern "C" int b200kv_import_peer(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device,
                                  const b200kv_ipc_desc* descs, int32_t n_descs,
                                  uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks) {
  return import_peer(ctx, peer_id, peer_device, descs, n_descs, peer_block_stride_bytes, peer_n_blocks, nullptr);
}

extern "C" int b200kv_import_peer_sliced(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device,
                                         const b200kv_ipc_desc* descs, int32_t n_descs,
                                         uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks,
                                         const b200kv_head_slice* slice) {
  if (!slice) return B200KV_EINVAL;
  return import_peer(ctx, peer_id, peer_device, descs, n_descs, peer_block_stride_bytes, peer_n_blocks, slice);
}

static int import_peer_ptrs(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device, const void* const* k_ptrs,
                            const void* const* v_ptrs, uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks,
                            const b200kv_head_slice* slice) {
  if (!ctx || peer_id < 0 || peer_id >= kMaxPeers) return B200KV_EINVAL;
  if (peer_n_blocks == 0 || peer_n_blocks * ctx->g.bs > 0x7fffffffull) return B200KV_EINVAL;
  if (slice && check_slice(ctx->g, *slice, peer_block_stride_bytes)) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  std::vector<uint64_t> bases;
  const int rc = plane_bases(ctx->g, k_ptrs, v_ptrs, &bases);
  if (rc) return rc;
  if (peer_device != ctx->cfg.device) {
    int can = 0;
    CU_TRY(cudaDeviceCanAccessPeer(&can, ctx->cfg.device, peer_device));
    if (!can) return B200KV_ENOTSUP;
    const cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
    if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
      set_err("cudaDeviceEnablePeerAccess", e, __LINE__);
      return B200KV_ENODEV;
    }
    cudaGetLastError();
  }
  std::vector<void*> none;   // raw pointers: no mappings to close
  return install_peer(ctx, peer_id, peer_device, bases, peer_block_stride_bytes, peer_n_blocks, &none, slice);
}

extern "C" int b200kv_import_peer_ptrs(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device,
                                       const void* const* k_ptrs, const void* const* v_ptrs,
                                       uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks) {
  return import_peer_ptrs(ctx, peer_id, peer_device, k_ptrs, v_ptrs, peer_block_stride_bytes, peer_n_blocks, nullptr);
}

extern "C" int b200kv_import_peer_ptrs_sliced(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device,
                                              const void* const* k_ptrs, const void* const* v_ptrs,
                                              uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks,
                                              const b200kv_head_slice* slice) {
  if (!slice) return B200KV_EINVAL;
  return import_peer_ptrs(ctx, peer_id, peer_device, k_ptrs, v_ptrs, peer_block_stride_bytes, peer_n_blocks, slice);
}

extern "C" int b200kv_peer_pull_async(b200kv_ctx* ctx, int32_t peer_id, const int64_t* src_slots,
                                      const int64_t* dst_slots, int64_t n_tokens,
                                      void* compute_stream, uint64_t* ticket) {
  if (!ctx || !src_slots || !dst_slots || n_tokens <= 0 || !ticket) return B200KV_EINVAL;
  if (peer_id < 0 || peer_id >= kMaxPeers || !ctx->peers[peer_id].valid) return B200KV_ENOENT;
  if (!ctx->kv_registered) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  reap(ctx);
  const Peer& peer = ctx->peers[peer_id];
  cudaStream_t cs = static_cast<cudaStream_t>(compute_stream);
  *ticket = 0;

  OpTable table;
  std::vector<Run> partial;
  int rc = build_pull_runs(src_slots, dst_slots, n_tokens, static_cast<int64_t>(peer.n_blocks) * ctx->g.bs,
                           static_cast<int64_t>(ctx->cfg.n_blocks) * ctx->g.bs, static_cast<int32_t>(ctx->g.bs),
                           ctx->g.hnd, &table.runs, &partial);
  if (rc) return rc;
  table.full_off.push_back(static_cast<uint32_t>(table.runs.size()));
  table.part_off.push_back(static_cast<uint32_t>(partial.size()));
  table.runs.insert(table.runs.end(), partial.begin(), partial.end());
  const uint64_t no_chunk = 0;   // a pull copies pages to pages: its one chunk has no buffer
  TableView tv;
  rc = stage_table(ctx, table, &no_chunk, ctx->s_scatter, &tv);
  if (rc) return rc;

  OpGuard guard(ctx, ctx->s_scatter, nullptr, nullptr, nullptr);
  guard.op.reset(new Op());
  Op* op = guard.op.get();
  op->id = ctx->next_ticket++;
  CU_TRY(cudaEventCreateWithFlags(&op->done, cudaEventDisableTiming));
  const bool detached = compute_stream == B200KV_STREAM_DETACHED;
  if (!detached) {
    rc = stream_wait(ctx, ctx->s_scatter, cs);
    if (rc) return rc;
  }

  timing_reset(ctx, kTimePull);
  rc = timing_begin(ctx, kTimePull, ctx->s_scatter);
  if (rc) return rc;
  rc = launch_op(ctx, kPull, table, tv, 0, 1, ctx->s_scatter, 0, 0, &peer);
  if (rc) return rc;
  rc = timing_end(ctx, kTimePull, ctx->s_scatter);
  if (rc) return rc;
  CU_TRY(cudaEventRecord(tv.slot->done_ev, ctx->s_scatter));
  CU_TRY(cudaLaunchHostFunc(ctx->s_scatter, op_host_cb, op));
  CU_TRY(cudaEventRecord(op->done, ctx->s_scatter));
  if (!detached) CU_TRY(cudaStreamWaitEvent(cs, op->done, 0));
  ++ctx->stats.n_pull_ops;
  ctx->stats.n_pulled_tokens += n_tokens;
  const uint64_t token_bytes = peer.sliced ? static_cast<uint64_t>(peer.slice.n_heads) * ctx->g.row_bytes
                                           : ctx->g.token_bytes;
  ctx->stats.p2p_bytes += static_cast<uint64_t>(n_tokens) * token_bytes * ctx->g.planes;
  if (ctx->g.indexed) ctx->stats.p2p_bytes += static_cast<uint64_t>(n_tokens) * (ctx->g.idx_vb + ctx->g.idx_sb) * ctx->g.L;
  *ticket = op->id;
  ctx->ops.emplace(op->id, std::move(guard.op));
  guard.armed = false;
  return B200KV_OK;
}

// ------------------------------------------------------------------------------------------------
// stats
// ------------------------------------------------------------------------------------------------
extern "C" int b200kv_engine_get_stats(b200kv_ctx* ctx, b200kv_engine_stats* out) {
  if (!ctx || !out) return B200KV_EINVAL;
  std::lock_guard<std::mutex> lk(ctx->mu);
  *out = ctx->stats;
  return B200KV_OK;
}

extern "C" int b200kv_last_kernel_ms(b200kv_ctx* ctx, int which, float* ms_out) {
  if (!ctx || !ms_out || which < 0 || which >= kTimingSlots) return B200KV_EINVAL;
  DeviceGuard dg(ctx->cfg.device);
  std::lock_guard<std::mutex> lk(ctx->mu);
  float total = 0.f;
  auto& t = ctx->timing[which];
  for (size_t i = 0; i < t.used; ++i) {
    float ms = 0.f;
    CU_TRY(cudaEventSynchronize(t.ev[i].second));
    CU_TRY(cudaEventElapsedTime(&ms, t.ev[i].first, t.ev[i].second));
    total += ms;
  }
  *ms_out = total;
  return B200KV_OK;
}
