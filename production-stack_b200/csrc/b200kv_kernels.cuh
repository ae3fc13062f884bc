// b200kv_kernels.cuh — sm_90a (H100) kernels of the KV offload / transfer hot path.
//
// What they replace: LMCache's paged-memory GPU connector (`VLLMPagedMemGPUConnectorV2`,
// named at vllm/.../lmcache_integration/vllm_v1_adapter.py:19-23,533-541) — an element-wise
// gather/scatter between vLLM's paged KV cache and a contiguous (L,2,C,H,D) chunk — plus the
// UCX/NIXL peer copy the reference configures for disaggregated prefill
// (helm/templates/deployment-vllm-multi.yaml:296-324).
//
// All of them are HBM-bound byte movers (SURVEY.md §8d): no tensor cores.  The design rules
// that matter are coalescing, enough bytes in flight per SM to cover DRAM latency, and a grid
// that is a multiple of the SM count (132 on H100).
//
//   kv_bulk_copy_kernel    RAW store / load / peer pull.  One elected thread per CTA drives the
//                          TMA engine: cp.async.bulk global->smem (mbarrier complete_tx) into an
//                          S-stage ring, then cp.async.bulk smem->global (bulk_group).  No
//                          registers touch the payload.  Persistent grid.
//   kv_ldg_copy_kernel     same contract with 128-bit ld.global.nc / st.global (A/B variant).
//   kv_hnd_partial_kernel  RAW runs that cover part of an HND tile, moved one (run, plane, head) row
//                          range at a time.
//   kv_fp8_store3_kernel   FP8 store of block-structured ops (the default): persistent, warp-specialised;
//                          a TMA producer warp feeds two consumer groups, one (chunk, plane, head) unit
//                          at a time.
//   kv_fp8_store_kernel    FP8 store of every other op: cluster of 8 CTAs per (chunk, layer, K/V) slab;
//                          warp 0 bulk-loads the CTA's tokens into smem (one run per lane), per-head
//                          absmax in registers -> smem, every CTA pushes its maxima into all 8 CTAs'
//                          smem with DSMEM atomics (red.shared::cluster.max) between a split cluster
//                          barrier (arrive early, wait late) and one full one, quantise to e4m3 from
//                          smem, coalesced stores.  HBM is read exactly once.  NHD and HND tiles.
//   kv_fp8_load_kernel     bulk-load e4m3 piece -> dequantise -> 16-byte stores into the pages.
//   kv_q4_store_kernel /   group-wise 4-bit chunks: one 16-byte vector per thread, a group is a quad
//   kv_q4_load_kernel      of lanes.
//   kv_q4_store_fp8_kernel /  the same records from and to fp8 pages (e4m3 or e5m2): a group is a pair of lanes.
//   kv_q4_load_fp8_kernel
//   kv_mla_fp8_store_kernel /  FP8 latent records of MLA engines: one warp per (token, plane), a group of
//   kv_mla_fp8_load_kernel     128 elements is 16 lanes; no shared memory.
//   kv_indexer_copy_kernel the indexer planes of sparse-attention MLA engines (split [values][scales] tiles),
//                          verbatim, store / load / pull: TMA bulk pieces, a 4-byte warp copy for unaligned scales.
//   kv_head_slice_pull_kernel  peer pull from a replica of another tensor-parallel size: a contiguous range of the
//                          peer's heads into a contiguous range of ours, 16-byte vectors.
//
// Every kernel takes one KernelArgs, filled by kernel_args() in b200kv_engine.cu.  The seven FP8 / Q4 / MLA FP8
// kernels are also built per cache element type (bf16, fp16: template argument DT, see Src below).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "b200kv_runs.h"

namespace b200kv {

struct PagedSide {
  const uint64_t* bases;  // device array: K plane of layer l at [2l], V at [2l+1]; MLA: latent (or indexer) at [l]
  uint64_t block_stride;  // bytes between consecutive blocks of one plane
  uint32_t block_tokens;
  uint32_t token_bytes;   // H*D*elem (NHD: one token's heads are contiguous)
};

struct ChunkSide {
  const uint64_t* chunk_addrs;  // device array [n_chunks]: where chunk c of this op lives
  uint64_t slab_bytes;          // C * token_bytes: one (layer, K/V) slab
  uint32_t chunk_tokens;
  uint32_t token_bytes;         // bytes per token per slab in this format: RAW H*D*elem, FP8 H*D, Q4 one record
  uint64_t scales_off;          // FP8: byte offset of the (planes, H) fp32 scales inside a chunk
};

// The one parameter block of every kernel.  A field a kernel does not read is still filled.  It must stay within
// 128 bytes: nvcc keeps a larger by-value kernel parameter in memory and reads every field through its address,
// which costs registers (kv_q4_store_kernel: 39 -> 47).  The order of the 32-bit fields keeps the bulk copy
// kernel's parameter loads, and so its code, as they were.
struct KernelArgs {
  PagedSide paged;                // local pages (store src / load dst / pull dst)
  PagedSide peer;                 // pull src (peer mapping)
  ChunkSide chunk;
  const Run* runs;
  const uint32_t* chunk_run_off;  // FP8 stores: [n_chunks+1] run range of each chunk
  uint32_t n_heads;
  uint32_t n_planes;              // planes covered by this launch (2*L, or one layer group of it)
  uint32_t plane_begin;           // first plane of the launch (layer-wise loads walk the planes in groups)
  uint32_t pieces;                // bulk copy: pieces per run = ceil(block_tokens / piece_tokens)
  uint32_t piece_tokens;          // bulk copy: tokens per piece (piece bytes <= stage bytes)
  uint32_t total_units;           // units of work of the launch; each kernel says what its unit is
  uint32_t row_bytes;             // D * elem: one (token, head) row (D*2 for FP8, D*2 or D for Q4)
  uint32_t hnd;                   // pages hold [H][block_tokens][D] tiles
};
static_assert(sizeof(KernelArgs) <= 128, "KernelArgs must stay within 128 bytes (see above)");

enum CopyMode { kStore = 0, kLoad = 1, kPull = 2 };

// ---------------------------------------------------------------------------------------------
// PTX helpers
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global -> shared (this CTA), completion signalled on an mbarrier in bytes.  SASS: UBLKCP.
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
          "r"(smem_u32(smem_dst)),
      "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// shared -> global, tracked by the thread's bulk async-group.
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
               "r"(smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() {
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_read() {  // <= N groups still reading smem
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_all() {  // <= N groups not yet complete (writes done)
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_na_v4(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_na_v2(void* p, const uint2& v) {
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y)
               : "memory");
}
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;\n\tbarrier.cluster.wait.acquire.aligned;" ::
                   : "memory");
}
__device__ __forceinline__ void cluster_arrive_release() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
}
__device__ __forceinline__ void cluster_wait_acquire() {
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// atomic max into the same shared variable of CTA `rank` of this cluster (DSMEM)
__device__ __forceinline__ void red_dsmem_max_u32(void* local_smem_ptr, uint32_t rank, uint32_t v) {
  uint32_t remote;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(local_smem_ptr)), "r"(rank));
  asm volatile("red.relaxed.cluster.shared::cluster.max.u32 [%0], %1;" ::"r"(remote), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_dsmem_u32(const void* local_smem_ptr, uint32_t rank) {
  uint32_t remote, v;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;"
               : "=r"(remote)
               : "r"(smem_u32(local_smem_ptr)), "r"(rank));
  asm volatile("ld.shared::cluster.u32 %0, [%1];" : "=r"(v) : "r"(remote) : "memory");
  return v;
}

// ---------------------------------------------------------------------------------------------
// addressing
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t paged_addr(const PagedSide& s, uint32_t plane, uint32_t slot) {
  const uint32_t blk = slot / s.block_tokens;
  const uint32_t off = slot - blk * s.block_tokens;
  return __ldg(s.bases + plane) + static_cast<uint64_t>(blk) * s.block_stride +
         static_cast<uint64_t>(off) * s.token_bytes;
}
// HND tiles: row `off` of head h inside the slot's block
__device__ __forceinline__ uint64_t paged_addr_hnd(const PagedSide& s, uint32_t plane, uint32_t slot,
                                                   uint32_t h, uint32_t row_bytes) {
  const uint32_t blk = slot / s.block_tokens;
  const uint32_t off = slot - blk * s.block_tokens;
  return __ldg(s.bases + plane) + static_cast<uint64_t>(blk) * s.block_stride +
         static_cast<uint64_t>(h) * s.block_tokens * row_bytes + static_cast<uint64_t>(off) * row_bytes;
}

// an op-relative token index as (chunk c, token t inside chunk c)
struct ChunkPos {
  uint32_t c, t;
};
__device__ __forceinline__ ChunkPos chunk_pos(const ChunkSide& s, uint32_t tok) {
  const uint32_t c = tok / s.chunk_tokens;
  return {c, tok - c * s.chunk_tokens};
}

__device__ __forceinline__ uint64_t chunk_addr(const ChunkSide& s, uint32_t plane, uint32_t tok) {
  const ChunkPos cp = chunk_pos(s, tok);
  return __ldg(s.chunk_addrs + cp.c) + static_cast<uint64_t>(plane) * s.slab_bytes +
         static_cast<uint64_t>(cp.t) * s.token_bytes;
}
// HND: the chunk stores the tiles verbatim
__device__ __forceinline__ uint64_t chunk_addr_hnd(const ChunkSide& s, uint32_t plane, uint32_t tok,
                                                   uint32_t h, uint32_t block_tokens, uint32_t row_bytes) {
  const ChunkPos cp = chunk_pos(s, tok);
  const uint32_t tile = cp.t / block_tokens;
  const uint32_t off = cp.t - tile * block_tokens;
  return __ldg(s.chunk_addrs + cp.c) + static_cast<uint64_t>(plane) * s.slab_bytes +
         static_cast<uint64_t>(tile) * block_tokens * s.token_bytes +
         static_cast<uint64_t>(h) * block_tokens * row_bytes + static_cast<uint64_t>(off) * row_bytes;
}

// Source and destination of a RAW copy by direction, `off` tokens into the run: a store reads the pages at slot
// run.a and writes the chunk at token run.b, a load the other way round, a pull reads the peer's pages at slot
// run.a and writes the local pages at slot run.b.  paged(side, slot) and chunk(tok) give one side's address.
template <int MODE, class PagedAt, class ChunkAt>
__device__ __forceinline__ void copy_ends(const KernelArgs& p, const Run& run, int32_t off, PagedAt paged,
                                          ChunkAt chunk, uint64_t* src, uint64_t* dst) {
  if (MODE == kStore) {
    *src = paged(p.paged, static_cast<uint32_t>(run.a + off));
    *dst = chunk(static_cast<uint32_t>(run.b + off));
  } else if (MODE == kLoad) {
    *src = chunk(static_cast<uint32_t>(run.b + off));
    *dst = paged(p.paged, static_cast<uint32_t>(run.a + off));
  } else {
    *src = paged(p.peer, static_cast<uint32_t>(run.a + off));
    *dst = paged(p.paged, static_cast<uint32_t>(run.b + off));
  }
}

struct Unit {
  uint64_t src, dst;
  uint32_t bytes;
};

template <int MODE>
__device__ __forceinline__ Unit decode_unit(const KernelArgs& p, uint32_t u) {
  // plane fastest: consecutive units of one CTA stride across planes of the same run.
  const uint32_t plane = p.plane_begin + u % p.n_planes;
  const uint32_t t = u / p.n_planes;
  const uint32_t piece = t % p.pieces;
  const uint32_t r = t / p.pieces;
  const Run run = p.runs[r];
  const int32_t off = static_cast<int32_t>(piece * p.piece_tokens);
  int32_t n = run.n - off;
  n = n < 0 ? 0 : (n > static_cast<int32_t>(p.piece_tokens) ? static_cast<int32_t>(p.piece_tokens) : n);
  Unit out;
  out.bytes = static_cast<uint32_t>(n) * p.paged.token_bytes;
  copy_ends<MODE>(
      p, run, off,
      [&](const PagedSide& s, uint32_t slot) { return paged_addr(s, plane, slot); },
      [&](uint32_t tok) { return chunk_addr(p.chunk, plane, tok); }, &out.src, &out.dst);
  return out;
}

// ---------------------------------------------------------------------------------------------
// RAW path, TMA-engine variant.  One warp per CTA, lane 0 does everything:
//   iteration j:  (B) issue bulk load of unit j into stage j%S   (after the store that last used
//                     that stage finished READING smem)
//                 (A) wait for unit j-LAG's bytes, issue its bulk store, commit one group.
// Loads in flight per CTA: LAG; stores in flight: S-LAG.
// ---------------------------------------------------------------------------------------------
// A unit is one piece of one run in one plane: total_units = n_runs * n_planes * pieces.
template <int MODE, int S, int LAG>
__global__ void __launch_bounds__(32) kv_bulk_copy_kernel(const KernelArgs p, uint32_t stage_bytes) {
  static_assert(LAG >= 1 && LAG < S, "need 1 <= LAG < S");
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem);               // S mbarriers
  uint64_t* dsts = reinterpret_cast<uint64_t*>(smem + 64);          // S pending dst addresses
  uint32_t* lens = reinterpret_cast<uint32_t*>(smem + 64 + 8 * S);  // S pending lengths
  uint8_t* stage0 = smem + 256;

  if (threadIdx.x != 0) return;
#pragma unroll
  for (int s = 0; s < S; ++s) mbar_init(&full[s], 1);
  fence_mbar_init();

  const uint32_t first = blockIdx.x;
  const uint32_t step = gridDim.x;
  const uint32_t n = first < p.total_units ? (p.total_units - first + step - 1) / step : 0;

  for (uint32_t j = 0; j < n + LAG; ++j) {
    if (j < n) {
      const uint32_t s = j % S;
      if (j >= S) bulk_wait_read<S - 1 - LAG>();  // store of unit j-S has drained its stage
      const Unit u = decode_unit<MODE>(p, first + j * step);
      dsts[s] = u.dst;
      lens[s] = u.bytes;
      if (u.bytes) bulk_g2s(stage0 + static_cast<size_t>(s) * stage_bytes,
                            reinterpret_cast<const void*>(u.src), u.bytes, &full[s]);
      mbar_arrive_expect_tx(&full[s], u.bytes);
    }
    if (j >= LAG) {
      const uint32_t k = j - LAG;
      const uint32_t s = k % S;
      mbar_wait(&full[s], (k / S) & 1u);
      const uint32_t bytes = lens[s];
      if (bytes) bulk_s2g(reinterpret_cast<void*>(dsts[s]),
                          stage0 + static_cast<size_t>(s) * stage_bytes, bytes);
      bulk_commit();
    }
  }
  bulk_wait_all<0>();  // every store has landed before the grid is considered complete
}

// ---------------------------------------------------------------------------------------------
// RAW path, LSU variant: a CTA copies one unit at a time with 128-bit loads, 4 in flight/thread.
// ---------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(256) kv_ldg_copy_kernel(const KernelArgs p) {
  for (uint32_t ui = blockIdx.x; ui < p.total_units; ui += gridDim.x) {
    const Unit u = decode_unit<MODE>(p, ui);
    const uint4* __restrict__ src = reinterpret_cast<const uint4*>(u.src);
    uint4* __restrict__ dst = reinterpret_cast<uint4*>(u.dst);
    const uint32_t nvec = u.bytes >> 4;
    uint32_t i = threadIdx.x;
    for (; i + 3 * 256 < nvec; i += 4 * 256) {
      const uint4 a = ld_nc_v4(src + i), b = ld_nc_v4(src + i + 256);
      const uint4 c = ld_nc_v4(src + i + 512), d = ld_nc_v4(src + i + 768);
      st_na_v4(dst + i, a);
      st_na_v4(dst + i + 256, b);
      st_na_v4(dst + i + 512, c);
      st_na_v4(dst + i + 768, d);
    }
    for (; i < nvec; i += 256) st_na_v4(dst + i, ld_nc_v4(src + i));
  }
}

// ---------------------------------------------------------------------------------------------
// HND tiles ([H][block_tokens][D] inside a block).  A whole-block run is one contiguous tile and
// goes through the kernels above unchanged (the chunk stores tiles verbatim).  Runs that cover
// only part of a tile — the ragged tail of a request, or token-granular mappings — are moved
// per head by this kernel: one unit = (run, plane, head) = n * D * elem contiguous bytes, so
// total_units = n_runs * n_planes * n_heads.
// ---------------------------------------------------------------------------------------------
template <int MODE>
__global__ void __launch_bounds__(128) kv_hnd_partial_kernel(const KernelArgs p) {
  for (uint32_t ui = blockIdx.x; ui < p.total_units; ui += gridDim.x) {
    const uint32_t h = ui % p.n_heads;
    const uint32_t t = ui / p.n_heads;
    const uint32_t plane = p.plane_begin + t % p.n_planes;
    const Run run = p.runs[t / p.n_planes];
    uint64_t src, dst;
    copy_ends<MODE>(
        p, run, 0,
        [&](const PagedSide& s, uint32_t slot) { return paged_addr_hnd(s, plane, slot, h, p.row_bytes); },
        [&](uint32_t tok) { return chunk_addr_hnd(p.chunk, plane, tok, h, p.paged.block_tokens, p.row_bytes); },
        &src, &dst);
    const uint32_t nvec = (static_cast<uint32_t>(run.n) * p.row_bytes) >> 4;
    for (uint32_t i = threadIdx.x; i < nvec; i += 128)
      st_na_v4(reinterpret_cast<uint4*>(dst) + i, ld_nc_v4(reinterpret_cast<const uint4*>(src) + i));
  }
}

// ---------------------------------------------------------------------------------------------
// FP8 store.  grid = (kCluster * n_slabs), cluster (kCluster,1,1); slab = (chunk c, plane).
// CTA `rank` owns tokens [rank*W, rank*W+W) of the chunk, W = C / kCluster.
// ---------------------------------------------------------------------------------------------
constexpr int kCluster = 8;
constexpr int kFp8Threads = 256;
constexpr int kMaxHeads = 64;

// |x| max of packed 16-bit pairs: the sign bit cleared, integer order equals magnitude order for bf16 and fp16 alike
__device__ __forceinline__ uint32_t absmax_u16x2(uint32_t acc, uint32_t w) {
  return __vmaxu2(acc, w & 0x7fff7fffu);
}

// ---------------------------------------------------------------------------------------------
// Element type of the paged cache the lossy kernels read and write (B200KV_DTYPE_*).  It is a template argument,
// not a KernelArgs field (see the 128-byte note on KernelArgs).  Everything else about a format is the same for
// both types: the absmax is taken on the 16-bit magnitude bits, quantisation works on the exact fp32 value, and
// decoding rounds the fp32 product once to the cache's type (RN).  Q4 scales stay bf16 bits in either case.
// Specification of the fp16 builds: tests/fp16_oracle.py.
// ---------------------------------------------------------------------------------------------
enum CacheDtype { kBf16 = 0, kFp16 = 1 };

template <int DT>
struct Src;
template <>
struct Src<kBf16> {
  // the two elements of a packed pair as fp32: lo = element 0 (low half), hi = element 1
  static __device__ __forceinline__ float lo(uint32_t w) { return __uint_as_float(w << 16); }
  static __device__ __forceinline__ float hi(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
  // two fp32 -> a packed pair, round to nearest even
  static __device__ __forceinline__ uint32_t pack_rn(float a, float b) {
    const __nv_bfloat162 r = __floats2bfloat162_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&r);
  }
  // 16-bit magnitude bits (an absmax) -> fp32
  static __device__ __forceinline__ float from_bits(uint32_t m) { return __uint_as_float(m << 16); }
};
template <>
struct Src<kFp16> {
  // two scalar conversions: __half22float2 costs kv_q4_store_kernel 4 registers (39 -> 43) and so one CTA per SM
  static __device__ __forceinline__ float lo(uint32_t w) {
    return __half2float(__ushort_as_half(static_cast<unsigned short>(w & 0xffffu)));
  }
  static __device__ __forceinline__ float hi(uint32_t w) {
    return __half2float(__ushort_as_half(static_cast<unsigned short>(w >> 16)));
  }
  static __device__ __forceinline__ uint32_t pack_rn(float a, float b) {
    const __half2 r = __floats2half2_rn(a, b);
    return *reinterpret_cast<const uint32_t*>(&r);
  }
  static __device__ __forceinline__ float from_bits(uint32_t m) {
    return __half2float(__ushort_as_half(static_cast<unsigned short>(m)));
  }
};

// e4m3 of 8 cache elements scaled by inv (fp32 multiply, RN, satfinite) -> 8 bytes.
template <int DT>
__device__ __forceinline__ uint2 quant8(const uint4& v, float inv) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t o[2];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float a0 = Src<DT>::lo(w[2 * i]) * inv;
    const float a1 = Src<DT>::hi(w[2 * i]) * inv;
    const float b0 = Src<DT>::lo(w[2 * i + 1]) * inv;
    const float b1 = Src<DT>::hi(w[2 * i + 1]) * inv;
    const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(a0, a1), __NV_SATFINITE, __NV_E4M3);
    const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(b0, b1), __NV_SATFINITE, __NV_E4M3);
    o[i] = lo | (hi << 16);
  }
  return make_uint2(o[0], o[1]);
}

template <int DT>
__global__ void __cluster_dims__(kCluster, 1, 1) __launch_bounds__(kFp8Threads)
    kv_fp8_store_kernel(const KernelArgs p) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ uint32_t s_absmax[kMaxHeads];  // this CTA's |x| max per head (16-bit magnitude bits)
  __shared__ uint32_t s_all[kMaxHeads];     // cluster-wide max: every CTA pushes its value into every CTA's copy
  __shared__ float s_inv[kMaxHeads];

  const uint32_t rank = cluster_ctarank();
  const uint32_t slab = blockIdx.x / kCluster;
  const uint32_t c = slab / p.n_planes;
  const uint32_t plane = slab - c * p.n_planes;
  const uint32_t W = p.chunk.chunk_tokens / kCluster;
  const uint32_t tb = p.paged.token_bytes;
  const uint32_t win_lo = c * p.chunk.chunk_tokens + rank * W;  // op-relative token index
  uint32_t n_valid = 0;
  // tokens of this chunk = end of its last run (runs are sorted by b): a batch of several requests may hold
  // partial chunks anywhere, not only at its end
  uint32_t chunk_hi = c * p.chunk.chunk_tokens;
  {
    const uint32_t rr0 = p.chunk_run_off[c], rr1 = p.chunk_run_off[c + 1];
    if (rr1 > rr0) chunk_hi = static_cast<uint32_t>(p.runs[rr1 - 1].b + p.runs[rr1 - 1].n);
  }
  if (win_lo < chunk_hi) n_valid = min(W, chunk_hi - win_lo);
  if (win_lo + n_valid > chunk_hi) n_valid = chunk_hi > win_lo ? chunk_hi - win_lo : 0;

  if (threadIdx.x < kMaxHeads) {
    s_absmax[threadIdx.x] = 0;
    s_all[threadIdx.x] = 0;
  }
  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();  // barrier initialised before any lane can signal it
  if (threadIdx.x < 32) {
    // warp 0 walks the chunk's run list in parallel (one run per lane): the table reads are one
    // L2 round trip instead of a serial chain, and every lane issues its own bulk copy.
    uint32_t mine = 0;
    const uint32_t r0 = p.chunk_run_off[c], r1 = p.chunk_run_off[c + 1];
    const uint32_t bs = p.paged.block_tokens;
    for (uint32_t r = r0 + threadIdx.x; r < r1; r += 32) {
      const Run run = p.runs[r];
      const int32_t lo = max(run.b, static_cast<int32_t>(win_lo));
      const int32_t hi = min(run.b + run.n, static_cast<int32_t>(win_lo + n_valid));
      if (hi <= lo) continue;
      const uint32_t slot = static_cast<uint32_t>(run.a + (lo - run.b));
      const uint32_t rel = static_cast<uint32_t>(lo - static_cast<int32_t>(win_lo));
      const uint32_t n = static_cast<uint32_t>(hi - lo);
      if (!p.hnd || (n == bs && (slot % bs) == 0 && (rel % bs) == 0)) {
        // NHD run, or a whole HND tile: one contiguous piece
        bulk_g2s(smem + static_cast<size_t>(rel) * tb, reinterpret_cast<const void*>(paged_addr(p.paged, plane, slot)),
                 n * tb, &bar);
        mine += n * tb;
      } else {
        // partial HND tile: one piece per head (runs never cross a tile on either side)
        const uint32_t row = p.row_bytes;  // D*2
        uint8_t* tile = smem + static_cast<size_t>(rel / bs) * bs * tb + static_cast<size_t>(rel % bs) * row;
        for (uint32_t h = 0; h < p.n_heads; ++h) {
          bulk_g2s(tile + static_cast<size_t>(h) * bs * row,
                   reinterpret_cast<const void*>(paged_addr_hnd(p.paged, plane, slot, h, row)), n * row, &bar);
          mine += n * row;
        }
      }
    }
    const uint32_t total = __reduce_add_sync(0xffffffffu, mine);
    // complete_tx may land before this expect_tx: the phase cannot complete until the arrive
    if (threadIdx.x == 0) mbar_arrive_expect_tx(&bar, total);
  }
  // Cluster barrier #1, split: arrive now (publishes the zeroed s_all), wait only just before the
  // DSMEM pushes — its latency hides behind the bulk loads that are already in flight.
  cluster_arrive_release();
  mbar_wait(&bar, 0);

  const uint32_t vpt = tb >> 4;  // 16-byte vectors per token
  // HND window = W/bs whole tiles [H][bs][D]: vector idx = ((tile*H + h)*bs + row)*rv + c.
  const uint32_t rv = p.row_bytes >> 4;                 // 16-byte vectors per (token, head) row
  const uint32_t tile_rows = p.paged.block_tokens * rv;  // vectors per (tile, head)
  const uint32_t n_tiles = W / p.paged.block_tokens;
  if (p.hnd) {
    // One warp per head (heads w, w+8, ...): the valid rows of a (tile, head) block are a prefix of it
    // ([bs][D] rows are contiguous), so the warp streams the block with 16-byte loads, folds the lanes
    // with one REDUX and owns s_absmax[h] — no index arithmetic per vector, no atomics.
    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t h = threadIdx.x >> 5; h < p.n_heads; h += kFp8Threads >> 5) {
      uint32_t acc = 0;
      for (uint32_t tile = 0; tile < n_tiles; ++tile) {
        const uint32_t t0 = tile * p.paged.block_tokens;
        const uint32_t nv = (n_valid > t0 ? min(p.paged.block_tokens, n_valid - t0) : 0u) * rv;
        const uint8_t* blk = smem + static_cast<size_t>(tile * p.n_heads + h) * tile_rows * 16;
#pragma unroll 8
        for (uint32_t v = lane; v < nv; v += 32) {
          const uint4 x = *reinterpret_cast<const uint4*>(blk + static_cast<size_t>(v) * 16);
          acc = absmax_u16x2(absmax_u16x2(absmax_u16x2(absmax_u16x2(acc, x.x), x.y), x.z), x.w);
        }
      }
      const uint32_t m = __reduce_max_sync(0xffffffffu, max(acc & 0xffffu, acc >> 16));
      if (lane == 0) s_absmax[h] = m;
    }
  } else {
  // ---- per-head absmax over this CTA's tokens: a thread's 16-byte column has a fixed head ----
    // When a token has fewer than 256 vectors the spare threads split the tokens between them.
    const uint32_t groups = vpt < kFp8Threads ? kFp8Threads / vpt : 1;
    const uint32_t grp = threadIdx.x / vpt;
    if (grp < groups) {
      const uint32_t col_step = groups == 1 ? kFp8Threads : vpt;
      for (uint32_t col = threadIdx.x - grp * vpt; col < vpt; col += col_step) {
        uint32_t acc = 0;
        const uint8_t* q = smem + static_cast<size_t>(col) * 16;
        for (uint32_t t = grp; t < n_valid; t += groups) {
          const uint4 v = *reinterpret_cast<const uint4*>(q + static_cast<size_t>(t) * tb);
          acc = absmax_u16x2(absmax_u16x2(absmax_u16x2(absmax_u16x2(acc, v.x), v.y), v.z), v.w);
        }
        const uint32_t m = max(acc & 0xffffu, acc >> 16);
        atomicMax(&s_absmax[(col * 16) / p.row_bytes], m);
      }
    }
  }
  __syncthreads();
  cluster_wait_acquire();  // #1: every CTA of the cluster has zeroed its s_all
  if (threadIdx.x < p.n_heads) {
    const uint32_t mine = s_absmax[threadIdx.x];
#pragma unroll
    for (uint32_t r = 0; r < kCluster; ++r) red_dsmem_max_u32(&s_all[threadIdx.x], r, mine);
  }
  // Cluster barrier #2: all pushes have landed everywhere.  Nothing remote is touched after it, so
  // no trailing barrier is needed to keep shared memory alive.
  cluster_arrive_release();
  cluster_wait_acquire();

  if (threadIdx.x < p.n_heads) {
    const uint32_t m = s_all[threadIdx.x];
    const float amax = Src<DT>::from_bits(m);
    const float inv = (m == 0) ? 1.0f : __fdiv_rn(448.0f, amax);
    s_inv[threadIdx.x] = inv;
    if (rank == 0) {
      float* scales = reinterpret_cast<float*>(p.chunk.chunk_addrs[c] + p.chunk.scales_off);
      scales[plane * p.n_heads + threadIdx.x] = (m == 0) ? 1.0f : __fdiv_rn(amax, 448.0f);
    }
  }
  __syncthreads();

  if (p.hnd) {
    // the packed slab mirrors the tiles at half size: same vector index, 8 bytes each
    uint8_t* outh = reinterpret_cast<uint8_t*>(p.chunk.chunk_addrs[c] + static_cast<uint64_t>(plane) * p.chunk.slab_bytes +
                                               static_cast<uint64_t>(rank * W) * (tb >> 1));
    const uint32_t lane = threadIdx.x & 31u;
    for (uint32_t h = threadIdx.x >> 5; h < p.n_heads; h += kFp8Threads >> 5) {
      const float inv = s_inv[h];
      for (uint32_t tile = 0; tile < n_tiles; ++tile) {
        const uint32_t t0 = tile * p.paged.block_tokens;
        const uint32_t nv = (n_valid > t0 ? min(p.paged.block_tokens, n_valid - t0) : 0u) * rv;
        const size_t base = static_cast<size_t>(tile * p.n_heads + h) * tile_rows;
#pragma unroll 8
        for (uint32_t v = lane; v < nv; v += 32) {
          const uint4 x = *reinterpret_cast<const uint4*>(smem + (base + v) * 16);
          st_na_v2(outh + (base + v) * 8, quant8<DT>(x, inv));
        }
      }
    }
    return;
  }

  // ---- quantise from smem, 8-byte coalesced stores ----
  uint8_t* out = reinterpret_cast<uint8_t*>(p.chunk.chunk_addrs[c] + static_cast<uint64_t>(plane) * p.chunk.slab_bytes +
                                            static_cast<uint64_t>(rank * W) * (tb >> 1));
  const uint32_t nvec = n_valid * vpt;
  if ((kFp8Threads % vpt) == 0) {
    // i % vpt == threadIdx.x % vpt for every i of this thread: one head, one scale, no division
    const float inv = s_inv[((threadIdx.x % vpt) * 16) / p.row_bytes];
    for (uint32_t i = threadIdx.x; i < nvec; i += kFp8Threads) {
      const uint4 v = *reinterpret_cast<const uint4*>(smem + static_cast<size_t>(i) * 16);
      st_na_v2(out + static_cast<size_t>(i) * 8, quant8<DT>(v, inv));
    }
  } else {
    for (uint32_t i = threadIdx.x; i < nvec; i += kFp8Threads) {
      const uint32_t col = i % vpt;
      const uint4 v = *reinterpret_cast<const uint4*>(smem + static_cast<size_t>(i) * 16);
      st_na_v2(out + static_cast<size_t>(i) * 8, quant8<DT>(v, s_inv[(col * 16) / p.row_bytes]));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// FP8 store, persistent warp-specialised pipeline (the default for block-structured ops).
//
// Unit of work = (chunk, plane, head): the C x D bf16 elements one scale covers (64 KiB for C=256,
// D=128), i.e. exactly what has to be seen before anything can be quantised.  Nothing is exchanged
// between CTAs: no cluster, no DSMEM, no atomics.  One CTA per SM:
//   warp 0           producer: for every unit one TMA copy per paged block ([bs][D] of head h, 4 KiB) into the
//                    unit buffer of the consumer group that will take it, completion on its `full` mbarrier.
//                    HND tiles: the piece is contiguous -> cp.async.bulk (UBLKCP).  NHD tiles: the piece is
//                    bs rows of D elements strided by the token size -> cp.async.bulk.tensor.4d through a
//                    per-plane tensor map {D, H, bs, NB}, box {D, 1, bs, 1} (UTMALDG).  Either way the unit
//                    lands as [C tokens][D] in shared memory.
//   2 x 8 warps      two consumer groups ping-pong over the units: wait `full`, copy the unit into registers
//                    (16 x 16 B per thread, conflict-free), release the stage at once (`empty`), absmax
//                    (packed u16 max, one REDUX per warp, one named barrier per group), quantise from
//                    registers, 8-byte stores that fill whole 128-byte lines.
// A group releases its buffer as soon as the unit is in registers, so while it reduces and quantises unit i its
// unit i+2 is already streaming in, and so is the other group's: the memory pipe never drains between the load -> absmax -> quantise phases of a unit (the cluster kernel above
// runs at 33 % warps active with exactly that bubble).  HBM is read once and written once.
// Eligibility (checked on the host, else the cluster kernel runs): the geometry fits the unit buffers, and every
// chunk is a sequence of whole, block-aligned runs, the last one possibly short (whole_block_chunks in
// b200kv_runs.h) — what any vLLM block table produces.  Run j of chunk c is then paged block j of the chunk.
// total_units = n_chunks * n_planes * H.
// ---------------------------------------------------------------------------------------------
constexpr int kS3Groups = 2;
constexpr int kS3Stages = kS3Groups;   // stage g is filled for, and drained by, consumer group g only: consecutive uses of a
                                       // stage are strictly ordered, so a parity wait can never alias an older phase (with a
                                       // shared ring a group could ask for use k of a stage whose use k-1 — the OTHER group's
                                       // unit — had not landed yet, pass on the parity of use k-2 and corrupt the barrier)
constexpr int kS3GroupThreads = 256;
constexpr int kS3Threads = 32 + kS3Groups * kS3GroupThreads;
constexpr int kS3MaxVec = 16;          // 16-byte vectors per consumer thread per unit
constexpr uint32_t kS3MaxUnitBytes = kS3MaxVec * kS3GroupThreads * 16;   // 64 KiB

__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// 4-D tiled TMA load global -> shared (this CTA), completion on an mbarrier.  SASS: UTMALDG.
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const void* tmap, int32_t c0, int32_t c1, int32_t c2,
                                            int32_t c3, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];" ::
          "r"(smem_u32(smem_dst)),
      "l"(tmap), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t n_threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(n_threads) : "memory");
}

template <int DT>
__global__ void __launch_bounds__(kS3Threads, 1) kv_fp8_store3_kernel(const KernelArgs p,
                     const void* tmaps) {   // one CUtensorMap per plane (NHD pages); nullptr for HND pages
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t full_bar[kS3Stages];
  __shared__ __align__(8) uint64_t empty_bar[kS3Stages];
  __shared__ uint32_t s_max[kS3Groups][2][kS3GroupThreads / 32];

  const uint32_t bs = p.paged.block_tokens;
  const uint32_t piece_bytes = bs * p.row_bytes;                   // one block's rows of one head
  const uint32_t unit_bytes = p.chunk.chunk_tokens * p.row_bytes;  // stage size (<= 64 KiB, host-checked)
  const uint32_t H = p.n_heads;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kS3Stages; ++s) {
      mbar_init(&full_bar[s], 1);
      mbar_init(&empty_bar[s], kS3GroupThreads / 32);   // one arrive per warp of the consuming group
    }
    fence_mbar_init();
  }
  __syncthreads();

  const uint32_t n_mine = p.total_units > blockIdx.x ? (p.total_units - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  if (threadIdx.x < 32) {
    // ------------------------------- producer -------------------------------
    const uint32_t lane = threadIdx.x;
    for (uint32_t i = 0; i < n_mine; ++i) {
      const uint32_t u = blockIdx.x + i * gridDim.x;
      const uint32_t h = u % H;
      const uint32_t plane = (u / H) % p.n_planes;
      const uint32_t c = u / (H * p.n_planes);
      const uint32_t s = i % kS3Groups, k = i / kS3Groups;    // stage == consumer group; k-th use of that stage
      const uint32_t r0 = __ldg(p.chunk_run_off + c), r1 = __ldg(p.chunk_run_off + c + 1);
      const uint32_t n_blocks = r1 - r0;
      if (k > 0) mbar_wait(&empty_bar[s], (k - 1) & 1);
      if (lane == 0) mbar_arrive_expect_tx(&full_bar[s], n_blocks * piece_bytes);
      __syncwarp();
      uint8_t* stage = smem + static_cast<size_t>(s) * unit_bytes;
      for (uint32_t j = lane; j < n_blocks; j += 32) {
        const uint32_t block = static_cast<uint32_t>(p.runs[r0 + j].a) / bs;
        uint8_t* dst = stage + static_cast<size_t>(j) * piece_bytes;
        if (tmaps) {   // NHD pages
          const uint8_t* tm = static_cast<const uint8_t*>(tmaps) + static_cast<size_t>(plane) * 128;
          tma_load_4d(dst, tm, 0, static_cast<int32_t>(h), 0, static_cast<int32_t>(block), &full_bar[s]);
        } else {
          const uint64_t src = __ldg(p.paged.bases + plane) + static_cast<uint64_t>(block) * p.paged.block_stride +
                               static_cast<uint64_t>(h) * piece_bytes;   // HND tile [H][bs][D]
          bulk_g2s(dst, reinterpret_cast<const void*>(src), piece_bytes, &full_bar[s]);
        }
      }
    }
    return;
  }

  // ------------------------------- consumers -------------------------------
  const uint32_t g = (threadIdx.x - 32) / kS3GroupThreads;
  const uint32_t t = (threadIdx.x - 32) % kS3GroupThreads;
  const uint32_t warp = t >> 5, lane = t & 31u;
  const uint32_t rv = p.row_bytes >> 4;          // 16-byte vectors per (token, head) row; power of two (host-checked)
  const uint32_t col8 = (t % rv) * 8;             // byte offset of this thread's 8 output bytes inside a row
  const uint32_t tok0 = t / rv;                   // token of vector kk = tok0 + kk * tok_step
  const uint32_t tok_step = kS3GroupThreads / rv;
  const uint32_t out_row = p.row_bytes >> 1;     // D bytes of e4m3 per (token, head)
  uint32_t it = 0;
  for (uint32_t i = g; i < n_mine; i += kS3Groups, ++it) {
    const uint32_t u = blockIdx.x + i * gridDim.x;
    const uint32_t h = u % H;
    const uint32_t plane = (u / H) % p.n_planes;
    const uint32_t c = u / (H * p.n_planes);
    const uint32_t s = g, k = it;
    // run j of the chunk is its paged block j, all full but possibly the last (host-checked)
    const uint32_t cr0 = __ldg(p.chunk_run_off + c), cr1 = __ldg(p.chunk_run_off + c + 1);
    const uint32_t n_valid = (cr1 - cr0 - 1) * bs + static_cast<uint32_t>(p.runs[cr1 - 1].n);
    const uint8_t* stage = smem + static_cast<size_t>(s) * unit_bytes;

    mbar_wait(&full_bar[s], k & 1);
    uint4 x[kS3MaxVec];
    uint32_t acc = 0;
#pragma unroll
    for (int kk = 0; kk < kS3MaxVec; ++kk) {
      const uint32_t tok = tok0 + kk * tok_step;
      if (tok < n_valid) {
        x[kk] = *reinterpret_cast<const uint4*>(stage + (static_cast<size_t>(kk) * kS3GroupThreads + t) * 16);
        acc = absmax_u16x2(absmax_u16x2(absmax_u16x2(absmax_u16x2(acc, x[kk].x), x[kk].y), x[kk].z), x[kk].w);
      } else {
        x[kk] = make_uint4(0, 0, 0, 0);
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);    // the unit lives in registers now: the stage can be refilled

    const uint32_t wmax = __reduce_max_sync(0xffffffffu, max(acc & 0xffffu, acc >> 16));
    const uint32_t par = it & 1;
    if (lane == 0) s_max[g][par][warp] = wmax;
    named_bar_sync(1 + g, kS3GroupThreads);
    uint32_t m = 0;
#pragma unroll
    for (int w = 0; w < kS3GroupThreads / 32; ++w) m = max(m, s_max[g][par][w]);
    const float amax = Src<DT>::from_bits(m);
    const float inv = (m == 0) ? 1.0f : __fdiv_rn(448.0f, amax);
    const uint64_t chunk_base = __ldg(p.chunk.chunk_addrs + c);
    if (t == 0) {
      float* scales = reinterpret_cast<float*>(chunk_base + p.chunk.scales_off);
      scales[plane * H + h] = (m == 0) ? 1.0f : __fdiv_rn(amax, 448.0f);
    }
    uint8_t* slab = reinterpret_cast<uint8_t*>(chunk_base + static_cast<uint64_t>(plane) * p.chunk.slab_bytes);
    // output offset of vector kk is linear in kk: NHD [token][H][D]; HND [tile][H][bs][D] when a step of
    // tok_step tokens is a whole number of tiles (the host checks tok_step % bs == 0 before choosing this kernel)
    uint32_t off0, off_step;
    if (p.hnd) {
      const uint32_t tile0 = tok0 / bs, row0 = tok0 - tile0 * bs;
      off0 = ((tile0 * H + h) * bs + row0) * out_row + col8;
      off_step = (tok_step / bs) * H * bs * out_row;
    } else {
      off0 = (tok0 * H + h) * out_row + col8;
      off_step = tok_step * H * out_row;
    }
    uint8_t* dst = slab + off0;
#pragma unroll
    for (int kk = 0; kk < kS3MaxVec; ++kk) {
      if (tok0 + kk * tok_step < n_valid) st_na_v2(dst + static_cast<size_t>(kk) * off_step, quant8<DT>(x[kk], inv));
    }
  }
}

// ---------------------------------------------------------------------------------------------
// FP8 load: one CTA per (run, plane) unit (total_units = n_runs * n_planes); e4m3 * scale -> the cache's type
// (one RN rounding of the fp32 product) into the pages.
// ---------------------------------------------------------------------------------------------
template <int DT>
__device__ __forceinline__ uint4 dequant8(const uint2& q, float scale) {
  const uint32_t w[2] = {q.x, q.y};
  uint32_t o[4];
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const __half2_raw h0 = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w[i] & 0xffffu), __NV_E4M3);
    const __half2_raw h1 = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(w[i] >> 16), __NV_E4M3);
    const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&h0));
    const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&h1));
    o[2 * i] = Src<DT>::pack_rn(f0.x * scale, f0.y * scale);
    o[2 * i + 1] = Src<DT>::pack_rn(f1.x * scale, f1.y * scale);
  }
  return make_uint4(o[0], o[1], o[2], o[3]);
}

template <int DT>
__global__ void __launch_bounds__(kFp8Threads) kv_fp8_load_kernel(const KernelArgs p) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar;
  __shared__ float s_scale[kMaxHeads];
  const uint32_t tb = p.paged.token_bytes;  // 16-bit cache bytes per token
  const uint32_t qtb = tb >> 1;

  if (threadIdx.x == 0) {
    mbar_init(&bar, 1);
    fence_mbar_init();
  }
  __syncthreads();

  uint32_t phase = 0;
  for (uint32_t ui = blockIdx.x; ui < p.total_units; ui += gridDim.x, phase ^= 1u) {
    const uint32_t plane = p.plane_begin + ui % p.n_planes;
    const Run run = p.runs[ui / p.n_planes];
    const ChunkPos cp = chunk_pos(p.chunk, static_cast<uint32_t>(run.b));
    const uint32_t t = cp.t;
    const uint64_t cbase = __ldg(p.chunk.chunk_addrs + cp.c);
    const uint32_t bs = p.paged.block_tokens;
    // NHD: the run's n tokens are contiguous in the packed slab.  HND: fetch the whole packed tile
    // ([H][bs][D] bytes) the run lives in and pick its rows.
    const uint32_t q_off = p.hnd ? (t / bs) * bs * qtb : t * qtb;
    const uint32_t qbytes = p.hnd ? bs * qtb : static_cast<uint32_t>(run.n) * qtb;
    if (threadIdx.x == 0) {
      bulk_g2s(smem, reinterpret_cast<const void*>(cbase + static_cast<uint64_t>(plane) * p.chunk.slab_bytes + q_off),
               qbytes, &bar);
      mbar_arrive_expect_tx(&bar, qbytes);
    }
    if (threadIdx.x < p.n_heads)
      s_scale[threadIdx.x] =
          reinterpret_cast<const float*>(cbase + p.chunk.scales_off)[plane * p.n_heads + threadIdx.x];
    __syncthreads();
    mbar_wait(&bar, phase);
    const uint32_t vpt = tb >> 4;
    if (p.hnd) {
      const uint32_t rv = p.row_bytes >> 4;   // 16-byte output vectors per (token, head) row
      const uint32_t o_src = t % bs;          // first row inside the packed tile
      const uint32_t n = static_cast<uint32_t>(run.n);
      const uint32_t total = p.n_heads * n * rv;
      for (uint32_t e = threadIdx.x; e < total; e += kFp8Threads) {
        const uint32_t cc = e % rv;
        const uint32_t r = (e / rv) % n;
        const uint32_t h = e / (rv * n);
        const uint2 q = *reinterpret_cast<const uint2*>(smem + (static_cast<size_t>(h) * bs + o_src + r) * (p.row_bytes >> 1) +
                                                        static_cast<size_t>(cc) * 8);
        uint8_t* d = reinterpret_cast<uint8_t*>(paged_addr_hnd(p.paged, plane, static_cast<uint32_t>(run.a), h, p.row_bytes));
        st_na_v4(d + static_cast<size_t>(r) * p.row_bytes + static_cast<size_t>(cc) * 16, dequant8<DT>(q, s_scale[h]));
      }
      __syncthreads();
      continue;
    }
    uint8_t* dst = reinterpret_cast<uint8_t*>(paged_addr(p.paged, plane, static_cast<uint32_t>(run.a)));
    const uint32_t nvec = static_cast<uint32_t>(run.n) * vpt;
    if ((kFp8Threads % vpt) == 0) {
      const float sc = s_scale[((threadIdx.x % vpt) * 16) / p.row_bytes];
      for (uint32_t i = threadIdx.x; i < nvec; i += kFp8Threads) {
        const uint2 q = *reinterpret_cast<const uint2*>(smem + static_cast<size_t>(i) * 8);
        st_na_v4(dst + static_cast<size_t>(i) * 16, dequant8<DT>(q, sc));
      }
    } else {
      for (uint32_t i = threadIdx.x; i < nvec; i += kFp8Threads) {
        const uint32_t col = i % vpt;
        const uint2 q = *reinterpret_cast<const uint2*>(smem + static_cast<size_t>(i) * 8);
        st_na_v4(dst + static_cast<size_t>(i) * 16, dequant8<DT>(q, s_scale[(col * 16) / p.row_bytes]));
      }
    }
    __syncthreads();  // smem + s_scale reusable
  }
}

// ---------------------------------------------------------------------------------------------
// Q4: group-wise 4-bit format (B200KV_FMT_Q4; oracle: q4_pack_chunk / q4_unpack_chunk).  A stored
// token of one plane is a record [H*D/2 code bytes][H*D/32 bf16 scales]; records are token-major in the
// slab whatever the order inside the paged tiles.  One 16-byte vector (8 elements) per thread, a group
// of 32 elements = 4 adjacent lanes: absmax by two shuffles, no shared memory, no cluster.  One unit per
// (run, plane): total_units = n_runs * n_planes.  chunk.token_bytes is the record size, H*D/2 + H*D/32*2.
// Bit-exact against the oracle on an H100 (tests/test_gpu_q4.py); still instruction-bound, the address
// arithmetic is done per vector (DESIGN §3, §5).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint64_t q4_src_addr(const KernelArgs& p, uint32_t plane, uint32_t slot, uint32_t v) {
  // v = 16-byte vector index inside the token: head h = v / rv, vector c of that head
  if (!p.hnd) return paged_addr(p.paged, plane, slot) + static_cast<uint64_t>(v) * 16;
  const uint32_t rv = p.row_bytes >> 4;
  const uint32_t h = v / rv, c = v - h * rv;
  return paged_addr_hnd(p.paged, plane, slot, h, p.row_bytes) + static_cast<uint64_t>(c) * 16;
}

constexpr int kQ4Unroll = 4;   // 16-byte vectors a thread keeps in flight (the kernels are pure streaming)

__device__ __forceinline__ void q4_split(uint32_t idx, uint32_t vpt, uint32_t vpt_shift, uint32_t* t, uint32_t* v) {
  if (vpt_shift != 0xffffffffu) { *t = idx >> vpt_shift; *v = idx & (vpt - 1); }
  else { *t = idx / vpt; *v = idx - *t * vpt; }
}

// q = rint(x * inv) (exact product, ties to even), inv = fl32(1 / s), s = bf16(absmax_group / 7)
// (oracle/kv_oracle.py q4_pack_chunk): one IEEE division per group, then one FMA per element.  The scale is bf16
// for fp16 caches too.
template <int DT>
__global__ void __launch_bounds__(256) kv_q4_store_kernel(const KernelArgs p) {
  const uint32_t vpt = (p.n_heads * p.row_bytes) >> 4;      // vectors per token (multiple of 4)
  const uint32_t vpt_shift = (vpt & (vpt - 1)) == 0 ? 31u - __clz(vpt) : 0xffffffffu;
  const uint32_t codes_bytes = vpt * 4;
  for (uint32_t ui = blockIdx.x; ui < p.total_units; ui += gridDim.x) {
    const uint32_t plane = p.plane_begin + ui % p.n_planes;
    const Run run = p.runs[ui / p.n_planes];
    const ChunkPos cp = chunk_pos(p.chunk, static_cast<uint32_t>(run.b));
    const uint32_t t0 = cp.t;
    uint8_t* slab =
        reinterpret_cast<uint8_t*>(__ldg(p.chunk.chunk_addrs + cp.c) + static_cast<uint64_t>(plane) * p.chunk.slab_bytes);
    const uint32_t nvec = static_cast<uint32_t>(run.n) * vpt;
    for (uint32_t base = 0; base < nvec; base += 256 * kQ4Unroll) {   // uniform trip count: every lane shuffles
      uint4 x[kQ4Unroll];
      uint32_t tt[kQ4Unroll], vv[kQ4Unroll];
      bool ok[kQ4Unroll];
#pragma unroll
      for (int j = 0; j < kQ4Unroll; ++j) {                 // all loads first: kQ4Unroll x 16 B in flight per thread
        const uint32_t idx = base + j * 256 + threadIdx.x;   // 256 and vpt are multiples of 4: quads stay whole
        ok[j] = idx < nvec;
        tt[j] = vv[j] = 0;
        if (ok[j]) q4_split(idx, vpt, vpt_shift, &tt[j], &vv[j]);
        x[j] = ok[j] ? ld_nc_v4(reinterpret_cast<const void*>(q4_src_addr(p, plane, static_cast<uint32_t>(run.a) + tt[j], vv[j])))
                     : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int j = 0; j < kQ4Unroll; ++j) {
        uint32_t acc = absmax_u16x2(absmax_u16x2(absmax_u16x2(absmax_u16x2(0u, x[j].x), x[j].y), x[j].z), x[j].w);
        uint32_t m = max(acc & 0xffffu, acc >> 16);
        m = max(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = max(m, __shfl_xor_sync(0xffffffffu, m, 2));
        const float amax = Src<DT>::from_bits(m);
        const __nv_bfloat16 sb = m ? __float2bfloat16_rn(__fdiv_rn(amax, 7.0f)) : __float2bfloat16_rn(1.0f);
        const float inv = __fdiv_rn(1.0f, __bfloat162float(sb));
        // rint(x * inv) for |x * inv| <= 7.03 without a convert: fma(x, inv, 1.5 * 2^23) rounds the EXACT product to
        // the nearest integer (ties to even) into the low mantissa bits, whose low nibble is the two's-complement
        // code.  No clamp is needed: |x| <= absmax and scale >= absmax / 7 * (1 - 2^-9).
        const uint32_t w[4] = {x[j].x, x[j].y, x[j].z, x[j].w};
        uint32_t packed = 0;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float lo = Src<DT>::lo(w[i]), hi = Src<DT>::hi(w[i]);
          const uint32_t ql = __float_as_uint(__fmaf_rn(lo, inv, 12582912.0f)) & 0xFu;
          const uint32_t qh = __float_as_uint(__fmaf_rn(hi, inv, 12582912.0f)) & 0xFu;
          packed |= (ql | (qh << 4)) << (8 * i);
        }
        if (!ok[j]) continue;
        uint8_t* rec = slab + static_cast<uint64_t>(t0 + tt[j]) * p.chunk.token_bytes;
        *reinterpret_cast<uint32_t*>(rec + static_cast<size_t>(vv[j]) * 4) = packed;
        if ((vv[j] & 3u) == 0) *reinterpret_cast<__nv_bfloat16*>(rec + codes_bytes + static_cast<size_t>(vv[j] >> 2) * 2) = sb;
      }
    }
  }
}

template <int DT>
__global__ void __launch_bounds__(256) kv_q4_load_kernel(const KernelArgs p) {
  const uint32_t vpt = (p.n_heads * p.row_bytes) >> 4;
  const uint32_t vpt_shift = (vpt & (vpt - 1)) == 0 ? 31u - __clz(vpt) : 0xffffffffu;
  const uint32_t codes_bytes = vpt * 4;
  for (uint32_t ui = blockIdx.x; ui < p.total_units; ui += gridDim.x) {
    const uint32_t plane = p.plane_begin + ui % p.n_planes;
    const Run run = p.runs[ui / p.n_planes];
    const ChunkPos cp = chunk_pos(p.chunk, static_cast<uint32_t>(run.b));
    const uint32_t t0 = cp.t;
    const uint8_t* slab = reinterpret_cast<const uint8_t*>(__ldg(p.chunk.chunk_addrs + cp.c) +
                                                           static_cast<uint64_t>(plane) * p.chunk.slab_bytes);
    const uint32_t nvec = static_cast<uint32_t>(run.n) * vpt;
    for (uint32_t base = threadIdx.x; base < nvec; base += 256 * kQ4Unroll) {
      uint32_t packed[kQ4Unroll], tt[kQ4Unroll], vv[kQ4Unroll];
      uint16_t sbits[kQ4Unroll];
#pragma unroll
      for (int j = 0; j < kQ4Unroll; ++j) {                 // all loads first
        const uint32_t idx = base + j * 256;
        packed[j] = 0;
        sbits[j] = 0;
        tt[j] = vv[j] = 0;
        if (idx < nvec) {
          q4_split(idx, vpt, vpt_shift, &tt[j], &vv[j]);
          const uint8_t* rec = slab + static_cast<uint64_t>(t0 + tt[j]) * p.chunk.token_bytes;
          packed[j] = __ldg(reinterpret_cast<const uint32_t*>(rec + static_cast<size_t>(vv[j]) * 4));
          sbits[j] = __ldg(reinterpret_cast<const uint16_t*>(rec + codes_bytes + static_cast<size_t>(vv[j] >> 2) * 2));
        }
      }
#pragma unroll
      for (int j = 0; j < kQ4Unroll; ++j) {
        if (base + j * 256 >= nvec) continue;
        const float s = __uint_as_float(static_cast<uint32_t>(sbits[j]) << 16);
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int b = static_cast<int>((packed[j] >> (8 * i)) & 0xffu);
          const int ql = ((b & 0xF) ^ 8) - 8, qh = ((b >> 4) ^ 8) - 8;   // sign-extend the nibbles
          o[i] = Src<DT>::pack_rn(static_cast<float>(ql) * s, static_cast<float>(qh) * s);
        }
        st_na_v4(reinterpret_cast<void*>(q4_src_addr(p, plane, static_cast<uint32_t>(run.a) + tt[j], vv[j])),
                 make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Q4 of fp8 pages (1-byte engines, B200KV_DTYPE_E4M3 / B200KV_DTYPE_E5M2; spec: tests/fp8_cache_oracle.py).  The
// record is the one above, bf16 scales included.  A 16-byte vector holds 16 codes, so a group of 32 elements is a
// pair of lanes (one shuffle); each vector writes 8 code bytes and the even lane of the pair writes the scale.
// Codes decode exactly to fp32 through f16 (cvt.rn.f16x2.e4m3x2 / e5m2x2).  The group absmax is taken on the 7
// magnitude bits: their integer order is magnitude order, finite codes below inf (e5m2) below NaN.  The store then
// quantises like kv_q4_store_kernel; the load computes q * s exactly in fp32 and encodes it once with
// cvt.rn.satfinite to the cache's type.  vLLM's k_scale / v_scale multiply the code's value on both sides of the
// cache, so they cancel and neither kernel needs them.  Units, runs and addressing (q4_src_addr, NHD and HND) are
// those of the 16-bit kernels: row_bytes is D here.
// ---------------------------------------------------------------------------------------------
template <__nv_fp8_interpretation_t FT>
__device__ __forceinline__ float2 fp8x2_to_f32(uint32_t two_codes) {
  const __half2_raw h = __nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(two_codes & 0xffffu), FT);
  return __half22float2(*reinterpret_cast<const __half2*>(&h));
}

template <__nv_fp8_interpretation_t FT>
__global__ void __launch_bounds__(256) kv_q4_store_fp8_kernel(const KernelArgs p) {
  const uint32_t vpt = (p.n_heads * p.row_bytes) >> 4;      // vectors per token (even: D % 32 == 0)
  const uint32_t vpt_shift = (vpt & (vpt - 1)) == 0 ? 31u - __clz(vpt) : 0xffffffffu;
  const uint32_t codes_bytes = vpt * 8;
  const bool st8 = (p.chunk.token_bytes & 7u) == 0;         // records 8-byte aligned (else 4: H*D % 64 == 0)
  for (uint32_t ui = blockIdx.x; ui < p.total_units; ui += gridDim.x) {
    const uint32_t plane = p.plane_begin + ui % p.n_planes;
    const Run run = p.runs[ui / p.n_planes];
    const ChunkPos cp = chunk_pos(p.chunk, static_cast<uint32_t>(run.b));
    const uint32_t t0 = cp.t;
    uint8_t* slab =
        reinterpret_cast<uint8_t*>(__ldg(p.chunk.chunk_addrs + cp.c) + static_cast<uint64_t>(plane) * p.chunk.slab_bytes);
    const uint32_t nvec = static_cast<uint32_t>(run.n) * vpt;
    for (uint32_t base = 0; base < nvec; base += 256 * kQ4Unroll) {   // uniform trip count: every lane shuffles
      uint4 x[kQ4Unroll];
      uint32_t tt[kQ4Unroll], vv[kQ4Unroll];
      bool ok[kQ4Unroll];
#pragma unroll
      for (int j = 0; j < kQ4Unroll; ++j) {                 // all loads first: kQ4Unroll x 16 B in flight per thread
        const uint32_t idx = base + j * 256 + threadIdx.x;   // 256 and vpt are even: pairs stay whole
        ok[j] = idx < nvec;
        tt[j] = vv[j] = 0;
        if (ok[j]) q4_split(idx, vpt, vpt_shift, &tt[j], &vv[j]);
        x[j] = ok[j] ? ld_nc_v4(reinterpret_cast<const void*>(q4_src_addr(p, plane, static_cast<uint32_t>(run.a) + tt[j], vv[j])))
                     : make_uint4(0, 0, 0, 0);
      }
#pragma unroll
      for (int j = 0; j < kQ4Unroll; ++j) {
        const uint32_t w[4] = {x[j].x, x[j].y, x[j].z, x[j].w};
        uint32_t acc = __vmaxu4(__vmaxu4(w[0] & 0x7f7f7f7fu, w[1] & 0x7f7f7f7fu), __vmaxu4(w[2] & 0x7f7f7f7fu, w[3] & 0x7f7f7f7fu));
        acc = max(max(acc & 0xffu, (acc >> 8) & 0xffu), max((acc >> 16) & 0xffu, acc >> 24));
        const uint32_t m = max(acc, __shfl_xor_sync(0xffffffffu, acc, 1));
        const float amax = fp8x2_to_f32<FT>(m).x;
        const __nv_bfloat16 sb = m ? __float2bfloat16_rn(__fdiv_rn(amax, 7.0f)) : __float2bfloat16_rn(1.0f);
        const float inv = __fdiv_rn(1.0f, __bfloat162float(sb));
        // rint(x * inv) by fma(x, inv, 1.5 * 2^23), as in kv_q4_store_kernel
        uint32_t packed[2] = {0u, 0u};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const float2 a = fp8x2_to_f32<FT>(w[i]), b = fp8x2_to_f32<FT>(w[i] >> 16);
          const uint32_t q0 = __float_as_uint(__fmaf_rn(a.x, inv, 12582912.0f)) & 0xFu;
          const uint32_t q1 = __float_as_uint(__fmaf_rn(a.y, inv, 12582912.0f)) & 0xFu;
          const uint32_t q2 = __float_as_uint(__fmaf_rn(b.x, inv, 12582912.0f)) & 0xFu;
          const uint32_t q3 = __float_as_uint(__fmaf_rn(b.y, inv, 12582912.0f)) & 0xFu;
          packed[i >> 1] |= (q0 | (q1 << 4) | (q2 << 8) | (q3 << 12)) << (16 * (i & 1));
        }
        if (!ok[j]) continue;
        uint8_t* rec = slab + static_cast<uint64_t>(t0 + tt[j]) * p.chunk.token_bytes;
        uint8_t* codes = rec + static_cast<size_t>(vv[j]) * 8;
        if (st8) {
          *reinterpret_cast<uint2*>(codes) = make_uint2(packed[0], packed[1]);
        } else {
          reinterpret_cast<uint32_t*>(codes)[0] = packed[0];
          reinterpret_cast<uint32_t*>(codes)[1] = packed[1];
        }
        if ((vv[j] & 1u) == 0) *reinterpret_cast<__nv_bfloat16*>(rec + codes_bytes + static_cast<size_t>(vv[j] >> 1) * 2) = sb;
      }
    }
  }
}

template <__nv_fp8_interpretation_t FT>
__global__ void __launch_bounds__(256) kv_q4_load_fp8_kernel(const KernelArgs p) {
  const uint32_t vpt = (p.n_heads * p.row_bytes) >> 4;
  const uint32_t vpt_shift = (vpt & (vpt - 1)) == 0 ? 31u - __clz(vpt) : 0xffffffffu;
  const uint32_t codes_bytes = vpt * 8;
  const bool ld8 = (p.chunk.token_bytes & 7u) == 0;
  for (uint32_t ui = blockIdx.x; ui < p.total_units; ui += gridDim.x) {
    const uint32_t plane = p.plane_begin + ui % p.n_planes;
    const Run run = p.runs[ui / p.n_planes];
    const ChunkPos cp = chunk_pos(p.chunk, static_cast<uint32_t>(run.b));
    const uint32_t t0 = cp.t;
    const uint8_t* slab = reinterpret_cast<const uint8_t*>(__ldg(p.chunk.chunk_addrs + cp.c) +
                                                           static_cast<uint64_t>(plane) * p.chunk.slab_bytes);
    const uint32_t nvec = static_cast<uint32_t>(run.n) * vpt;
    for (uint32_t base = threadIdx.x; base < nvec; base += 256 * kQ4Unroll) {
      uint2 packed[kQ4Unroll];
      uint32_t tt[kQ4Unroll], vv[kQ4Unroll];
      uint16_t sbits[kQ4Unroll];
#pragma unroll
      for (int j = 0; j < kQ4Unroll; ++j) {                 // all loads first
        const uint32_t idx = base + j * 256;
        packed[j] = make_uint2(0, 0);
        sbits[j] = 0;
        tt[j] = vv[j] = 0;
        if (idx < nvec) {
          q4_split(idx, vpt, vpt_shift, &tt[j], &vv[j]);
          const uint8_t* rec = slab + static_cast<uint64_t>(t0 + tt[j]) * p.chunk.token_bytes;
          const uint8_t* codes = rec + static_cast<size_t>(vv[j]) * 8;
          if (ld8) {
            packed[j] = __ldg(reinterpret_cast<const uint2*>(codes));
          } else {
            packed[j].x = __ldg(reinterpret_cast<const uint32_t*>(codes));
            packed[j].y = __ldg(reinterpret_cast<const uint32_t*>(codes) + 1);
          }
          sbits[j] = __ldg(reinterpret_cast<const uint16_t*>(rec + codes_bytes + static_cast<size_t>(vv[j] >> 1) * 2));
        }
      }
#pragma unroll
      for (int j = 0; j < kQ4Unroll; ++j) {
        if (base + j * 256 >= nvec) continue;
        const float s = __uint_as_float(static_cast<uint32_t>(sbits[j]) << 16);
        const uint32_t pw[2] = {packed[j].x, packed[j].y};
        uint32_t o[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int b = static_cast<int>((pw[i >> 1] >> (16 * (i & 1))) & 0xffffu);
          const int q0 = ((b & 0xF) ^ 8) - 8, q1 = (((b >> 4) & 0xF) ^ 8) - 8;   // sign-extend the nibbles
          const int q2 = (((b >> 8) & 0xF) ^ 8) - 8, q3 = ((b >> 12) ^ 8) - 8;
          const uint32_t lo = __nv_cvt_float2_to_fp8x2(make_float2(static_cast<float>(q0) * s, static_cast<float>(q1) * s),
                                                       __NV_SATFINITE, FT);
          const uint32_t hi = __nv_cvt_float2_to_fp8x2(make_float2(static_cast<float>(q2) * s, static_cast<float>(q3) * s),
                                                       __NV_SATFINITE, FT);
          o[i] = lo | (hi << 16);
        }
        st_na_v4(reinterpret_cast<void*>(q4_src_addr(p, plane, static_cast<uint32_t>(run.a) + tt[j], vv[j])),
                 make_uint4(o[0], o[1], o[2], o[3]));
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// FP8 latent records of an MLA engine (B200KV_LAYOUT_MLA + B200KV_FMT_FP8; spec: tests/mla_oracle.py, and
// tests/fp16_oracle.py for fp16 caches).
// A page row is 576 16-bit elements = 72 16-byte vectors: latent vectors 0..63 (group g = vectors
// [16g, 16g+16)), RoPE vectors 64..71.  A record is [512 e4m3 codes][4 fp32 scales][64 RoPE elements in the
// cache's own type].
// One warp per (token, plane): lane l holds latent vectors l and l+32, so lanes 0-15 see groups 0 and 2 and
// lanes 16-31 groups 1 and 3, and each half reduces both of its groups at once with four shuffles of two
// packed bf16 magnitudes.  Lane l writes 8 code bytes per vector (256 contiguous bytes per warp and vector),
// lane 0 writes the four scales as one 16-byte store, lanes 0-7 move the RoPE vectors.  No shared memory.
// A unit is one (run, plane): total_units = n_runs * n_planes; the warp walks the run kMlaTokens tokens at a
// time with all of their loads issued first.
// ---------------------------------------------------------------------------------------------
constexpr uint32_t kMlaDim = 576;            // kv_lora_rank 512 + qk_rope_head_dim 64
constexpr uint32_t kMlaRecordBytes = 656;    // 41 * 16
constexpr uint32_t kMlaScalesOff = 512;
constexpr uint32_t kMlaRopeOff = 528;        // 33 * 16
constexpr int kMlaThreads = 256;
constexpr int kMlaTokens = 4;

// scale = fl32(absmax / 448), inv = fl32(448 / absmax), both 1 when absmax is 0 (m = 16-bit magnitude bits of absmax)
template <int DT>
__device__ __forceinline__ float mla_scale(uint32_t m) { return m ? __fdiv_rn(Src<DT>::from_bits(m), 448.0f) : 1.0f; }
template <int DT>
__device__ __forceinline__ float mla_inv(uint32_t m) { return m ? __fdiv_rn(448.0f, Src<DT>::from_bits(m)) : 1.0f; }

__device__ __forceinline__ uint32_t absmax_vec(const uint4& v) {
  const uint32_t acc = absmax_u16x2(absmax_u16x2(absmax_u16x2(absmax_u16x2(0u, v.x), v.y), v.z), v.w);
  return max(acc & 0xffffu, acc >> 16);
}

template <int DT>
__global__ void __launch_bounds__(kMlaThreads) kv_mla_fp8_store_kernel(const KernelArgs p) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t n_warps = gridDim.x * (kMlaThreads / 32);
  for (uint32_t ui = blockIdx.x * (kMlaThreads / 32) + threadIdx.x / 32; ui < p.total_units; ui += n_warps) {
    const uint32_t plane = p.plane_begin + ui % p.n_planes;
    const Run run = p.runs[ui / p.n_planes];
    for (int32_t j = 0; j < run.n; j += kMlaTokens) {
      uint4 a[kMlaTokens], b[kMlaTokens], r[kMlaTokens];
#pragma unroll
      for (int k = 0; k < kMlaTokens; ++k) {   // every load of the step first
        r[k] = a[k] = b[k] = make_uint4(0, 0, 0, 0);
        if (j + k >= run.n) continue;
        const uint8_t* row = reinterpret_cast<const uint8_t*>(paged_addr(p.paged, plane, static_cast<uint32_t>(run.a + j + k)));
        a[k] = ld_nc_v4(row + 16 * lane);
        b[k] = ld_nc_v4(row + 512 + 16 * lane);
        if (lane < 8) r[k] = ld_nc_v4(row + 1024 + 16 * lane);
      }
#pragma unroll
      for (int k = 0; k < kMlaTokens; ++k) {
        if (j + k >= run.n) break;   // uniform over the warp
        uint32_t m = absmax_vec(a[k]) | (absmax_vec(b[k]) << 16);   // lo: group lane/16, hi: group 2 + lane/16
        m = __vmaxu2(m, __shfl_xor_sync(0xffffffffu, m, 1));
        m = __vmaxu2(m, __shfl_xor_sync(0xffffffffu, m, 2));
        m = __vmaxu2(m, __shfl_xor_sync(0xffffffffu, m, 4));
        m = __vmaxu2(m, __shfl_xor_sync(0xffffffffu, m, 8));
        const uint32_t other = __shfl_xor_sync(0xffffffffu, m, 16);
        uint8_t* rec = reinterpret_cast<uint8_t*>(chunk_addr(p.chunk, plane, static_cast<uint32_t>(run.b + j + k)));
        st_na_v2(rec + 8 * lane, quant8<DT>(a[k], mla_inv<DT>(m & 0xffffu)));
        st_na_v2(rec + 256 + 8 * lane, quant8<DT>(b[k], mla_inv<DT>(m >> 16)));
        if (lane == 0) {
          const float4 s = make_float4(mla_scale<DT>(m & 0xffffu), mla_scale<DT>(other & 0xffffu), mla_scale<DT>(m >> 16),
                                       mla_scale<DT>(other >> 16));
          st_na_v4(rec + kMlaScalesOff, *reinterpret_cast<const uint4*>(&s));
        }
        if (lane < 8) st_na_v4(rec + kMlaRopeOff + 16 * lane, r[k]);
      }
    }
  }
}

template <int DT>
__global__ void __launch_bounds__(kMlaThreads) kv_mla_fp8_load_kernel(const KernelArgs p) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t half = lane >> 4;
  const uint32_t n_warps = gridDim.x * (kMlaThreads / 32);
  for (uint32_t ui = blockIdx.x * (kMlaThreads / 32) + threadIdx.x / 32; ui < p.total_units; ui += n_warps) {
    const uint32_t plane = p.plane_begin + ui % p.n_planes;
    const Run run = p.runs[ui / p.n_planes];
    for (int32_t j = 0; j < run.n; j += kMlaTokens) {
      uint2 qa[kMlaTokens], qb[kMlaTokens];
      float sa[kMlaTokens], sb[kMlaTokens];
      uint4 r[kMlaTokens];
#pragma unroll
      for (int k = 0; k < kMlaTokens; ++k) {   // every load of the step first
        qa[k] = qb[k] = make_uint2(0, 0);
        sa[k] = sb[k] = 0.0f;
        r[k] = make_uint4(0, 0, 0, 0);
        if (j + k >= run.n) continue;
        const uint8_t* rec = reinterpret_cast<const uint8_t*>(chunk_addr(p.chunk, plane, static_cast<uint32_t>(run.b + j + k)));
        qa[k] = __ldg(reinterpret_cast<const uint2*>(rec + 8 * lane));
        qb[k] = __ldg(reinterpret_cast<const uint2*>(rec + 256 + 8 * lane));
        sa[k] = __ldg(reinterpret_cast<const float*>(rec + kMlaScalesOff) + half);
        sb[k] = __ldg(reinterpret_cast<const float*>(rec + kMlaScalesOff) + 2 + half);
        if (lane < 8) r[k] = ld_nc_v4(rec + kMlaRopeOff + 16 * lane);
      }
#pragma unroll
      for (int k = 0; k < kMlaTokens; ++k) {
        if (j + k >= run.n) break;
        uint8_t* row = reinterpret_cast<uint8_t*>(paged_addr(p.paged, plane, static_cast<uint32_t>(run.a + j + k)));
        st_na_v4(row + 16 * lane, dequant8<DT>(qa[k], sa[k]));
        st_na_v4(row + 512 + 16 * lane, dequant8<DT>(qb[k], sb[k]));
        if (lane < 8) st_na_v4(row + 1024 + 16 * lane, r[k]);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// Indexer planes of a sparse-attention MLA engine (b200kv_set_indexer; spec: tests/mla_sparse_oracle.py):
// DeepSeek-V3.2's indexer key cache, one split tile per block ([bs][vb] values, then [bs][sb] scales), copied
// verbatim between the pages and a chunk's indexer slabs ([C][vb], then [C][sb] per layer), or from a peer's pages.
// Store, load and pull; launched by launch_op right after the latent kernel of the same runs, on the same stream.
// KernelArgs describe the indexer planes here:
//   paged / peer  bases = the L indexer planes, block_stride = their block stride, token_bytes = vb
//   chunk         slab_bytes = one layer's indexer slab C*(vb+sb), scales_off = where the indexer slabs start
//   row_bytes     sb
// A unit is one (run, layer): total_units = n_runs * n_planes.  Each warp takes one unit at a time through its own
// shared-memory stage of bs*(vb+sb) bytes: lane 0 moves the value piece, and the scale piece when it is 16-byte
// granular (bulk_piece: every whole block when bs % 4 == 0), with the TMA engine (global -> smem -> global, the
// stores of one unit overlapping the loads of the next); any other scale piece is copied by the warp, 4 bytes per
// lane.  A run never crosses a block, so a stage holds any unit.
// ---------------------------------------------------------------------------------------------
constexpr int kIdxWarps = 4;
constexpr uint32_t kIdxBarBytes = 128;   // the warps' mbarriers, ahead of the stages

__device__ __forceinline__ uint32_t idx_stage_bytes(uint32_t bs, uint32_t vb, uint32_t sb) {
  return (bs * (vb + sb) + 15u) & ~15u;
}

template <int MODE>
__global__ void __launch_bounds__(kIdxWarps * 32) kv_indexer_copy_kernel(const KernelArgs p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31u;
  const uint32_t bs = p.paged.block_tokens, vb = p.paged.token_bytes, sb = p.row_bytes;
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem) + warp;
  uint8_t* stage = smem + kIdxBarBytes + static_cast<size_t>(warp) * idx_stage_bytes(bs, vb, sb);
  uint8_t* stage_s = stage + static_cast<size_t>(bs) * vb;
  if (lane == 0) {
    mbar_init(bar, 1);
    fence_mbar_init();
  }
  __syncwarp();
  const SplitTile tile{bs, p.chunk.chunk_tokens, vb, sb, MODE == kPull ? p.peer.block_stride : p.paged.block_stride,
                       p.paged.block_stride};
  uint32_t phase = 0;
  for (uint32_t u = blockIdx.x * kIdxWarps + warp; u < p.total_units; u += gridDim.x * kIdxWarps, phase ^= 1u) {
    const uint32_t plane = p.plane_begin + u % p.n_planes;
    const Run run = p.runs[u / p.n_planes];
    SplitPiece v, s;
    split_run_pieces(tile, MODE, run, &v, &s);
    // the offsets' bases: pages at slot run.a, and the chunk slab (store / load) or local pages (pull) at run.b
    const uint64_t page_a = __ldg((MODE == kPull ? p.peer.bases : p.paged.bases) + plane);
    const uint64_t side_b = MODE == kPull ? __ldg(p.paged.bases + plane)
                                          : __ldg(p.chunk.chunk_addrs + chunk_pos(p.chunk, static_cast<uint32_t>(run.b)).c) +
                                                p.chunk.scales_off + static_cast<uint64_t>(plane) * p.chunk.slab_bytes;
    const uint64_t src_base = MODE == kLoad ? side_b : page_a, dst_base = MODE == kLoad ? page_a : side_b;
    v.src += src_base; v.dst += dst_base;
    s.src += src_base; s.dst += dst_base;
    const bool s_bulk = bulk_piece(s);
    if (lane == 0) {
      bulk_wait_read<0>();   // the previous unit's stores have read the stage
      mbar_arrive_expect_tx(bar, v.bytes + (s_bulk ? s.bytes : 0u));
      bulk_g2s(stage, reinterpret_cast<const void*>(v.src), v.bytes, bar);
      if (s_bulk) bulk_g2s(stage_s, reinterpret_cast<const void*>(s.src), s.bytes, bar);
    }
    if (!s_bulk) {
      const uint32_t* src = reinterpret_cast<const uint32_t*>(s.src);
      uint32_t* dst = reinterpret_cast<uint32_t*>(s.dst);
      for (uint32_t i = lane; i < s.bytes / 4; i += 32) dst[i] = __ldg(src + i);
    }
    if (lane == 0) {
      mbar_wait(bar, phase);
      bulk_s2g(reinterpret_cast<void*>(v.dst), stage, v.bytes);
      if (s_bulk) bulk_s2g(reinterpret_cast<void*>(s.dst), stage_s, s.bytes);
      bulk_commit();
    }
  }
  if (lane == 0) bulk_wait_all<0>();   // every store has landed before the grid is considered complete
}

// ---------------------------------------------------------------------------------------------
// Head-slice peer pull: a producer replica of another tensor-parallel size holds heads [src_head0, src_head0 + n)
// of its H_p local heads that this engine keeps at [dst_head0, dst_head0 + n) of its H (b200kv_import_peer_sliced).
// K/V planes only.  Runs come from build_pull_runs (run.a = peer slot, run.b = local slot, never across a block).
// A pull reads no chunk, so KernelArgs carry the slice in the chunk side's fields:
//   peer.token_bytes   H_p * D * elem    (the peer's NHD token row)
//   paged.token_bytes  H * D * elem      (ours)
//   chunk.chunk_tokens n: heads moved
//   chunk.slab_bytes   src_head0: first head of the slice among the peer's
//   chunk.scales_off   dst_head0: where it lands among ours
//   row_bytes          D * elem (a multiple of 16)
// A unit is one (run, plane), total_units = n_runs * n_planes, and moves `cnt` pieces of `len` bytes:
//   NHD  cnt = run.n rows of n * D * elem, strided by each side's token row
//   HND  a whole-block run is one piece of n * bs * D * elem (the slice's tiles are adjacent on both sides);
//        a partial run is n pieces of run.n * D * elem, one per head, strided by bs * D * elem
// The CTA copies the unit's 16-byte vectors (flattened over pieces) with ld.global.nc from the peer mapping, read
// over NVLink as in kv_bulk_copy_kernel<kPull>, four in flight per thread.  No shared memory, no barrier.
// ---------------------------------------------------------------------------------------------
constexpr int kSliceThreads = 256;

__global__ void __launch_bounds__(kSliceThreads) kv_head_slice_pull_kernel(const KernelArgs p) {
  const uint32_t bs = p.paged.block_tokens, row = p.row_bytes, nh = p.chunk.chunk_tokens;
  for (uint32_t u = blockIdx.x; u < p.total_units; u += gridDim.x) {
    const uint32_t plane = p.plane_begin + u % p.n_planes;
    const Run run = p.runs[u / p.n_planes];
    const uint32_t sb = static_cast<uint32_t>(run.a) / bs, so = static_cast<uint32_t>(run.a) - sb * bs;
    const uint32_t db = static_cast<uint32_t>(run.b) / bs, dof = static_cast<uint32_t>(run.b) - db * bs;
    const uint8_t* src = reinterpret_cast<const uint8_t*>(__ldg(p.peer.bases + plane) +
                                                          static_cast<uint64_t>(sb) * p.peer.block_stride);
    uint8_t* dst = reinterpret_cast<uint8_t*>(__ldg(p.paged.bases + plane) +
                                              static_cast<uint64_t>(db) * p.paged.block_stride);
    uint32_t cnt, len, ss, ds;
    if (!p.hnd) {
      src += static_cast<uint64_t>(so) * p.peer.token_bytes + p.chunk.slab_bytes * row;
      dst += static_cast<uint64_t>(dof) * p.paged.token_bytes + p.chunk.scales_off * row;
      cnt = static_cast<uint32_t>(run.n);
      len = nh * row;
      ss = p.peer.token_bytes;
      ds = p.paged.token_bytes;
    } else {
      const uint32_t tile = bs * row;
      src += p.chunk.slab_bytes * tile + static_cast<uint64_t>(so) * row;
      dst += p.chunk.scales_off * tile + static_cast<uint64_t>(dof) * row;
      const bool whole = static_cast<uint32_t>(run.n) == bs;
      cnt = whole ? 1u : nh;
      len = whole ? nh * tile : static_cast<uint32_t>(run.n) * row;
      ss = ds = tile;
    }
    const uint32_t vpp = len >> 4, nvec = cnt * vpp;
    auto at = [&](uint32_t i, uint32_t stride) {
      const uint32_t k = i / vpp;
      return static_cast<uint64_t>(k) * stride + static_cast<uint64_t>(i - k * vpp) * 16u;
    };
    uint32_t i = threadIdx.x;
    for (; i + 3 * kSliceThreads < nvec; i += 4 * kSliceThreads) {
      uint4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = ld_nc_v4(src + at(i + j * kSliceThreads, ss));
#pragma unroll
      for (int j = 0; j < 4; ++j) st_na_v4(dst + at(i + j * kSliceThreads, ds), v[j]);
    }
    for (; i < nvec; i += kSliceThreads) st_na_v4(dst + at(i, ds), ld_nc_v4(src + at(i, ss)));
  }
}

}  // namespace b200kv
