/*
 * b200kv.h — C ABI of libb200kv.so, the H100-native (sm_90a) KV-cache offload /
 * cross-replica KV-transfer engine that fills the vLLM KV-connector slot which
 * vllm-project/production-stack fills with LMCache.
 *
 * Boundary being replaced (SURVEY.md §8b).  production-stack selects the connector by
 * string only (helm/templates/deployment-vllm-multi.yaml:194-207,
 * operator/internal/controller/vllmruntime_controller.go:536-543); the arithmetic lives in
 * the third-party `lmcache` wheel (pyproject.toml:49-52, lmcache==0.3.11), whose engine is
 * driven by vLLM's vendored adapter:
 *     lmcache_engine.store(tokens, mask, kvcaches, slot_mapping, offset, ...)
 *         vllm/.../lmcache_integration/vllm_v1_adapter.py:1115-1123
 *     lmcache_engine.retrieve(tokens, mask, kvcaches, slot_mapping, ...)
 *         vllm/.../lmcache_integration/vllm_v1_adapter.py:882-889
 *     lookup_client.lookup(token_ids, lookup_id, ...)
 *         vllm/.../lmcache_integration/vllm_v1_adapter.py:1187-1191
 * Every entry point below names the call it stands in for.  The host side above this ABI
 * is Python (production-stack_b200/b200kv), bound through ctypes; INTEGRATION.md shows the
 * stub.
 *
 * Conventions: extern "C"; plain pointers and sizes; no torch types; every function
 * returns 0 on success or a negative errno-style code (see b200kv_strerror); no C++
 * exception crosses the boundary; caller owns every pointer it passes in.  Functions in
 * the "pool" and "hash" groups never touch CUDA and are usable from the vLLM scheduler
 * process; functions in the "engine" group require a CUDA device and FAIL (-ENODEV) when
 * none is present — there is no CPU fallback anywhere in this library.
 */
#ifndef B200KV_H_
#define B200KV_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200KV_ABI_VERSION 1

/* ---- error codes (negative errno values; listed for documentation) -------------------- */
#define B200KV_OK 0
#define B200KV_EINVAL (-22)   /* malformed argument (unaligned, out of range, bad layout)   */
#define B200KV_ENOMEM (-12)   /* allocation failed                                          */
#define B200KV_ENODEV (-19)   /* no CUDA device / CUDA call failed                          */
#define B200KV_ENOENT (-2)    /* key / peer / ticket not found                              */
#define B200KV_EEXIST (-17)   /* key already present                                        */
#define B200KV_ENOSPC (-28)   /* pool full and nothing evictable                            */
#define B200KV_ENOTSUP (-95)  /* layout / feature not supported by this build               */
#define B200KV_EBUSY (-16)    /* resource still in use                                      */
#define B200KV_EIO (-5)       /* remote tier: connection lost / short read or write         */

/* ---- formats of a stored chunk -------------------------------------------------------- */
/* RAW  : (L, 2, C, H, D) elements of the cache dtype, token-major — the LMCache `kv_shape`
 *        (vllm_v1_adapter.py:471-477).  Bit-exact round trip.
 * FP8  : (L, 2, C, H, D) bytes of e4m3fn followed by (L, 2, H) fp32 scales; one scale per
 *        (chunk, layer, K/V, head) = absmax/448 (SURVEY.md §8c tolerance).  Source dtype
 *        bf16, or fp16 after b200kv_set_cache_dtype; decoding rounds once to the source dtype.
 *        Stands in for LMCACHE_REMOTE_SERDE=cachegen's lossy codec
 *        (helm/templates/deployment-vllm-multi.yaml:341-344).                              */
#define B200KV_FMT_RAW 0
#define B200KV_FMT_FP8 1
/* Q4 (experimental): group-wise 4-bit — per (token, head) groups of 32 elements, bf16 scale = absmax/7,
 * two's-complement nibbles; a stored token of one plane is [H*D/2 codes][H*D/32 scales] (4.5 bits per
 * element).  Specified by oracle/kv_oracle.py q4_pack_chunk (tests/fp16_oracle.py for fp16 caches,
 * tests/fp8_cache_oracle.py for fp8 caches).  Source dtype bf16, fp16, e4m3 or e5m2 (the scales stay bf16 for
 * all), D % 32 == 0; on fp8 caches also H*D % 64 == 0.                                            */
#define B200KV_FMT_Q4 2

/* ---- element type of the paged cache (b200kv_set_cache_dtype) ---------------------------- */
/* The lossy formats decode the cache's elements, so they must know which type they are.  RAW moves
 * bytes and needs no type, but the type is part of every chunk's format tag in either case, so bf16 and
 * fp16 chunks, and e4m3 and e5m2 chunks, never mix in a pool, a device tier or a cache server.
 * On a 1-byte (fp8) engine the default type 0 means e4m3 (vLLM's fp8 / fp8_e4m3 caches, e4m3fn): fp8 engines
 * created before the fp8 types existed were e4m3 in practice and keep their tags.  Q4 is the one lossy format
 * of an fp8 cache (tests/fp8_cache_oracle.py); FP8 is refused there, the pages already are fp8.          */
#define B200KV_DTYPE_BF16 0   /* default */
#define B200KV_DTYPE_FP16 1
#define B200KV_DTYPE_E4M3 0   /* the default of a 1-byte engine: the same value as BF16, so the same tags */
#define B200KV_DTYPE_E5M2 2

/* ---- order inside one (block, K|V) tile of the paged cache ------------------------------ */
/* NHD: [block_tokens][H][D] (FlashAttention default, vllm/v1/attention/backends/flash_attn.py:
 *      152-170).  HND: [H][block_tokens][D] — what vLLM's FlashInfer backend REQUIRES
 *      (vllm/v1/attention/selector.py:124-133 overrides the connector's wish).  Whole-block runs move as one contiguous tile in both; a
 *      chunk stores tiles verbatim, so chunks of the two layouts never mix (the layout is part
 *      of the pool's per-chunk format tag).                                                  */
#define B200KV_LAYOUT_NHD 0
#define B200KV_LAYOUT_HND 1
/* MLA: multi-head latent attention (DeepSeek-V2/V3, Kimi-K2).  ONE plane per layer, not a K and a V
 *      plane: vLLM's MLA backends allocate (num_blocks, block_size, head_size) per layer
 *      (MLACommonBackend.get_kv_cache_shape), so the tile is [block_tokens][D] and n_kv_heads must be 1.
 *      A RAW chunk is (L, 1, C, 1, D) — LMCache's MLA kv_shape (vllm_v1_adapter.py:463-477).
 *      FP8 on an MLA engine is a per-token latent record instead of the per-head format above: 656 bytes
 *      per (token, layer), the byte layout of vLLM's fp8_ds_mla cache entry
 *      (v1/attention/backends/mla/flashmla_sparse.py:68-79):
 *        [0, 512)    e4m3 codes of latent elements 0..511
 *        [512, 528)  4 fp32 scales, scale g = absmax(elements [128g, 128g+128)) / 448 (1 if absmax is 0)
 *        [528, 656)  RoPE elements 512..575, the cache's 16-bit bits copied verbatim
 *      A chunk is L slabs of C records (no separate scales area), rounded up to 256 bytes.  Needs a bf16
 *      or fp16 cache and D == 576; Q4 is not offered on MLA (-ENOTSUP).  In an fp16 cache the RoPE part
 *      is fp16 bits, where vLLM's fp8_ds_mla has bf16; such chunks carry the fp16 format tag.      */
#define B200KV_LAYOUT_MLA 2
/* Indexer planes (MLA with DeepSeek Sparse Attention: DeepSeek-V3.2).  After b200kv_set_indexer an MLA engine also
 *      moves one indexer plane per layer, verbatim, on every path.  vLLM's indexer_k_quant_and_cache writes a block
 *      of such a plane as a split tile: [block_tokens][value_bytes] e4m3 values, then [block_tokens][scale_bytes]
 *      (one fp32 scale per token); V3.2 has 128 + 4.  A chunk is the MLA chunk above (RAW slabs or FP8 records,
 *      not rounded) followed by L indexer slabs, each [C][value_bytes] then [C][scale_bytes], and the whole is
 *      rounded up to 256 bytes.  Such chunks carry bit 24 in their format tag (format | layout << 8 |
 *      dtype << 16 | 1 << 24).                                                                   */

/* ---- kernel variants (both are CUDA; selectable for A/B measurement) ------------------- */
#define B200KV_VARIANT_BULK 0 /* cp.async.bulk (TMA engine) through a shared-memory ring    */
#define B200KV_VARIANT_LDG 1  /* 128-bit ld.global.nc / st.global vector copy               */

typedef struct b200kv_pool b200kv_pool; /* pinned-host chunk pool + index (CPU side)        */
typedef struct b200kv_ctx b200kv_ctx;   /* per-GPU engine                                   */

/* ======================================================================================= */
/* misc                                                                                     */
/* ======================================================================================= */
int b200kv_abi_version(void);
const char* b200kv_strerror(int err);
/* Thread-local text of the most recent CUDA failure behind a -ENODEV (diagnostics only).   */
const char* b200kv_last_error(void);

/* ======================================================================================= */
/* hash group (CPU only)                                                                    */
/* ======================================================================================= */

/* XXH64 of a byte string (own implementation of the published algorithm; the reference
 * uses xxhash.xxh64 for its prefix trie, src/vllm_router/prefix/hashtrie.py:56-57, and the
 * helm chart pins PYTHONHASHSEED=123 only because LMCache keys were Python-hash derived,
 * helm/templates/deployment-vllm-multi.yaml:214-215 — these keys need no such coupling). */
uint64_t b200kv_xxh64(const void* data, size_t len, uint64_t seed);

/* Prefix-chained chunk keys of a token sequence: key[i] = XXH64(tokens[i*C:(i+1)*C] as
 * little-endian int32, seed = key[i-1]) with key[-1] = `seed`.  Replaces LMCache's
 * token-chunk hashing behind lookup/store/retrieve (SURVEY.md §8a row A5).  When
 * `include_partial` is nonzero a trailing chunk of fewer than C tokens gets a key too
 * (save_unfull_chunk / discard_partial_chunks=false, vllm_v1_adapter.py:329-333,662-667).
 * `keys_out` must hold ceil(n_tokens / C) entries; *n_keys_out receives the count.        */
int b200kv_chunk_keys(const int32_t* tokens, int64_t n_tokens, int32_t chunk_tokens,
                      uint64_t seed, int include_partial, uint64_t* keys_out,
                      int32_t* n_keys_out);

/* ======================================================================================= */
/* pool group (CPU only; safe in the scheduler process and across processes)               */
/* ======================================================================================= */

#define B200KV_POOL_CREATE 1u /* create (and size) the segment; fail with -EEXIST if present */
#define B200KV_POOL_ATTACH 2u /* attach to an existing named segment                         */
#define B200KV_POOL_CREATE_OR_ATTACH 3u

typedef struct b200kv_pool_config {
  const char* shm_name;  /* POSIX shm name ("/b200kv-…"); NULL = private anonymous mapping   */
  uint64_t pool_bytes;   /* payload bytes (LMCACHE_MAX_LOCAL_CPU_SIZE GB,                    */
                         /*   helm/templates/deployment-vllm-multi.yaml:326-333); CREATE only */
  uint64_t slot_bytes;   /* bytes of one chunk slot; CREATE only                             */
  uint32_t flags;        /* B200KV_POOL_*                                                    */
  uint32_t reserved;
} b200kv_pool_config;

typedef struct b200kv_pool_stats {
  uint64_t n_slots, n_used, slot_bytes;
  uint64_t n_lookups, n_lookup_chunks, n_hit_chunks;     /* lmcache:num_requested/hit_tokens  */
  uint64_t n_hit_tokens, n_requested_tokens;             /*   (helm/dashboards/lmcache-…json) */
  uint64_t n_stored_chunks, n_evicted_chunks, n_dropped_chunks;
  uint64_t n_reclaimed_chunks; /* slots / pins taken back from writers / readers that died        */
  uint64_t n_recoveries;       /* index rebuilt after a process died holding the pool lock       */
} b200kv_pool_stats;

int b200kv_pool_open(const b200kv_pool_config* cfg, b200kv_pool** out);
int b200kv_pool_close(b200kv_pool* pool);
int b200kv_pool_unlink(const char* shm_name);
/* Remove the named segments /dev/shm/<prefix>* that no live process has open (every opener holds a shared
 * flock on the segment for its lifetime) and that are at least min_age_s old: what a SIGKILLed or OOM-killed
 * engine left behind.  The reference's pool dies with its process (torch pinned memory); a shm pool does not. */
int b200kv_pool_sweep(const char* prefix, int32_t min_age_s, int32_t* n_removed);
/* Base address / byte length of the payload area (for cudaHostRegister by the engine).    */
int b200kv_pool_region(b200kv_pool* pool, void** base, uint64_t* bytes);
void* b200kv_pool_slot_ptr(b200kv_pool* pool, uint32_t slot);

/* lookup_client.lookup (vllm_v1_adapter.py:1187-1191): length of the longest stored prefix,
 * in whole chunks.  keys[i] from b200kv_chunk_keys; chunk_tokens[i] = tokens in chunk i
 * (all C except possibly the last).  Hit chunks are leased (not evictable) for `lease_ms`
 * so the worker can still find them when start_load_kv runs.  Side-effect free otherwise. */
int b200kv_pool_lookup(b200kv_pool* pool, const uint64_t* keys, const int32_t* chunk_tokens,
                       int32_t n_keys, uint32_t lease_ms, int32_t* n_hit_chunks,
                       int64_t* n_hit_tokens);
/* Per-key membership (not prefix): present[i] = 1 iff keys[i] is READY (and holds chunk_tokens[i]
 * tokens when chunk_tokens is given).  Present chunks are leased for lease_ms.  Used to combine
 * several tiers (host pool, device tiers of this and of peer replicas) into one prefix.        */
int b200kv_pool_contains(b200kv_pool* pool, const uint64_t* keys, const int32_t* chunk_tokens,
                         int32_t n_keys, uint32_t lease_ms, uint8_t* present);
/* First instance (owner tag given at reserve time) holding each of the first n_hit chunks;
 * answers the router's LookupMsg (src/vllm_router/routers/routing_logic.py:378-387).       */
int b200kv_pool_lookup_owner(b200kv_pool* pool, const uint64_t* keys, int32_t n_keys,
                             int32_t* n_hit_chunks, uint32_t* owner_out);

/* Writer protocol: reserve → fill slot → commit (or abort).  reserve evicts LRU unleased
 * READY chunks when full; -EEXIST if the key is present (READY or being written).          */
int b200kv_pool_reserve(b200kv_pool* pool, uint64_t key, int32_t n_tokens, uint32_t fmt,
                        uint32_t owner, uint32_t* slot_out);
int b200kv_pool_commit(b200kv_pool* pool, uint64_t key);
int b200kv_pool_abort(b200kv_pool* pool, uint64_t key);
/* Reader protocol: acquire (pins) → read slot → release.                                   */
int b200kv_pool_acquire(b200kv_pool* pool, uint64_t key, uint32_t* slot_out,
                        int32_t* n_tokens_out, uint32_t* fmt_out);
int b200kv_pool_release(b200kv_pool* pool, uint64_t key);
int b200kv_pool_get_stats(b200kv_pool* pool, b200kv_pool_stats* out);
/* Failure detection.  A process that dies between reserve and commit, or between acquire and
 * release, leaves a WRITING slot / a pin behind: both are taken back once older than
 * B200KV_POOL_STALE_MS (default 120 s; age, not pid — replicas may live in different pid
 * namespaces).  A process that dies while holding the pool lock triggers a rebuild of the free
 * list, LRU list and hash table from the slot array on the next call of any process.
 * b200kv_pool_check verifies those structures against the slot array (0, or -EIO).          */
int b200kv_pool_check(b200kv_pool* pool);
int b200kv_pool_clear(b200kv_pool* pool); /* KVConnectorBase_V1.reset_cache               */
/* Index rebuild (the disk tier's index after a restart): entry i puts keys[i] READY into slot slots[i], with its
 * token count, format tag and owner, appended to the LRU tail in the order given (oldest first).  An entry whose
 * slot is out of range or not free, whose key is already present, or whose n_tokens <= 0 is skipped.  Returns the
 * number of entries placed (>= 0) or a negative error.                                      */
int b200kv_pool_place(b200kv_pool* pool, const uint32_t* slots, const uint64_t* keys, const int32_t* n_tokens,
                      const uint32_t* fmts, const uint32_t* owners, int32_t n);
/* Remove one READY chunk (a reader found it corrupt).  -EBUSY while it is pinned, -ENOENT if absent. */
int b200kv_pool_drop(b200kv_pool* pool, uint64_t key);

/* ======================================================================================= */
/* engine group (CUDA, sm_90a)                                                              */
/* ======================================================================================= */

typedef struct b200kv_engine_config {
  int32_t device;            /* CUDA ordinal                                                 */
  int32_t n_layers;          /* L  (model_config.get_num_layers, vllm_v1_adapter.py:471)     */
  int32_t n_kv_heads;        /* H                                                            */
  int32_t head_dim;          /* D                                                            */
  int32_t elem_bytes;        /* bytes per cache element (2 = bf16/fp16, 1 = fp8 cache)        */
  int32_t block_tokens;      /* vLLM block_size (16)                                         */
  int32_t chunk_tokens;      /* LMCACHE_CHUNK_SIZE (256); multiple of block_tokens           */
  int32_t format;            /* B200KV_FMT_*                                                 */
  uint64_t block_stride_bytes; /* bytes between consecutive blocks of one layer's K (or V)   */
  uint64_t n_blocks;         /* blocks per layer (bounds check for slot ids)                 */
  uint64_t staging_bytes;    /* device staging ring (rounded down to whole chunks, >= 1)     */
  uint32_t owner;            /* instance tag recorded with stored chunks                     */
  int32_t variant;           /* B200KV_VARIANT_*                                             */
  int32_t stages;            /* smem ring depth for BULK (0 = default)                       */
  int32_t ctas_per_sm;       /* persistent CTAs per SM (0 = default)                         */
  int32_t kv_layout;         /* B200KV_LAYOUT_*: order inside one (block, K|V) tile            */
  int32_t numa_policy;       /* B200KV_NUMA_*: where the pool's host pages are placed when this
                              * engine is the first to pin them (0 = the GPU's own node)         */
} b200kv_engine_config;

/* Host-page placement of the pinned pool (the reference leaves it to first touch: LMCache's
 * LocalCPUBackend allocates with torch pin_memory, deployment-vllm-multi.yaml:326-333 only sizes it). */
#define B200KV_NUMA_LOCAL 0      /* prefer the NUMA node the GPU hangs off (per-engine pools)      */
#define B200KV_NUMA_INTERLEAVE 1 /* interleave over all nodes (one pool shared by a box's replicas) */
#define B200KV_NUMA_OFF 2        /* leave it to the kernel's first-touch policy                     */

typedef struct b200kv_engine_stats {
  uint64_t n_store_ops, n_load_ops, n_pull_ops;
  uint64_t n_stored_tokens, n_loaded_tokens, n_pulled_tokens;
  uint64_t n_kernel_launches;     /* launches of this library's own kernels                   */
  uint64_t h2d_bytes, d2h_bytes;  /* payload + tables moved by cudaMemcpyAsync                */
  uint64_t p2p_bytes;             /* payload read from peers                                  */
} b200kv_engine_stats;

/* Engine construction (stands in for _init_lmcache_engine, vllm_v1_adapter.py:433-558).
 * `pool` may be NULL for an engine used only through gather/scatter/peer_pull.             */
int b200kv_engine_create(const b200kv_engine_config* cfg, b200kv_pool* pool, b200kv_ctx** out);
/* Element type of the cache, B200KV_DTYPE_* (bf16, or e4m3 on a 1-byte engine, until set).  Legal between
 * b200kv_engine_create and b200kv_register_kv: -EBUSY after registration.  FP16 needs elem_bytes == 2 and E5M2
 * elem_bytes == 1, else -EINVAL.  A function
 * rather than a config field, so the v1 config layout and every existing binding stay valid.     */
int b200kv_set_cache_dtype(b200kv_ctx* ctx, int32_t dtype);
/* Gives an MLA engine an indexer plane per layer (B200KV_LAYOUT_MLA, indexer planes above); block_stride_bytes is
 * the bytes between consecutive blocks of one indexer plane (>= block_tokens * (value_bytes + scale_bytes), a
 * multiple of 16).  value_bytes % 16 == 0, scale_bytes % 4 == 0.  Legal between b200kv_engine_create and
 * b200kv_register_kv (and before b200kv_tier_create): -EBUSY after; -EINVAL on an engine that is not MLA.  The
 * staging ring is re-cut to the larger chunk; a pool whose slots are smaller than it gives -EINVAL.  From then on
 * the indexer planes are the engine's second kind of plane ("Planes and descriptors" at b200kv_register_kv), and a
 * peer's indexer planes are taken to have this engine's indexer block stride.                 */
int b200kv_set_indexer(b200kv_ctx* ctx, int32_t value_bytes, int32_t scale_bytes, uint64_t block_stride_bytes);
/* What the engine did about host-page placement when it pinned the pool (numa_policy above), as text
 * for logs and bench output, e.g. "mbind preferred node 1".                                  */
int b200kv_engine_numa_placement(b200kv_ctx* ctx, char* buf, uint64_t n);
int b200kv_engine_destroy(b200kv_ctx* ctx);
/* chunk_bytes for this engine's format — slot_bytes a pool must be created with.           */
int64_t b200kv_engine_chunk_bytes(const b200kv_engine_config* cfg);
/* chunk_bytes of the same engine after b200kv_set_indexer(ctx, value_bytes, scale_bytes, ...):
 * round_up(latent + L * C * (value_bytes + scale_bytes), 256), latent = L * C * D * elem_bytes (RAW) or
 * L * C * 656 (FP8 records).  -EINVAL for a geometry that is not MLA.                         */
int64_t b200kv_engine_chunk_bytes_indexed(const b200kv_engine_config* cfg, int32_t value_bytes, int32_t scale_bytes);

/* Planes and descriptors.  An engine has one or two kinds of plane per layer, passed as k_ptrs[l] and v_ptrs[l]
 * (device address of block 0 of layer l's plane, non-null and 16-byte aligned):
 *   B200KV_LAYOUT_NHD / _HND      k_ptrs: K planes    v_ptrs: V planes
 *   B200KV_LAYOUT_MLA             k_ptrs: latent      v_ptrs: NULL
 *   MLA after b200kv_set_indexer  k_ptrs: latent      v_ptrs: indexer planes
 * Anything else gives -EINVAL.  IPC descriptors follow the same order, kind-major: descriptor i is plane
 * (i / L, i % L), so there are 2*L of them with two kinds (k_ptrs' planes first) and L with one.
 *
 * register_kv_caches (KVConnectorBase_V1, vllm/.../v1/base.py:251): the engine's planes as above, NHD within a
 * block ([block_tokens][H][D]).
 * FlashAttention (2,NB,bs,H,D): v = k + NB*tile; FlashInfer (NB,2,bs,H,D): v = k + tile,
 * block_stride = 2*tile; cross-layer (NB,L,2,bs,H,D): block_stride = 2*L*tile.
 * A refused call leaves the registration as it was.                                          */
int b200kv_register_kv(b200kv_ctx* ctx, const void* const* k_ptrs, const void* const* v_ptrs);

/* lmcache_engine.store (vllm_v1_adapter.py:1115-1123).  Tokens [0,n_tokens) start on a
 * chunk boundary (the adapter's chunk-aligned `offset`); slot_mapping[i] = block*bs + i%bs
 * (vllm_v1_adapter.py:368-375) is a HOST array.  keys: one per chunk.  Chunks already in
 * the pool are skipped.  Gathers on an internal stream ordered after `compute_stream`, makes
 * `compute_stream` wait for the gather only, then streams to the pinned pool.  *ticket
 * completes when the data is in host memory and committed to the index.                    */
int b200kv_store_async(b200kv_ctx* ctx, const uint64_t* keys, int32_t n_chunks,
                       const int64_t* slot_mapping, int64_t n_tokens, void* compute_stream,
                       uint64_t* ticket);

/* lmcache_engine.retrieve (vllm_v1_adapter.py:882-889).  Same addressing; chunks
 * [0, skip_chunks) are the adapter's masked prefix (vLLM already has them) and are not
 * touched.  Loads the longest prefix of chunks present in the pool, scatters into the
 * paged cache, and makes `compute_stream` wait for the scatter.  *n_loaded_tokens counts
 * tokens of chunks >= skip_chunks that were scheduled (the adapter's ret_token_mask.sum). */
/* Pass as `compute_stream` to b200kv_load_async / b200kv_peer_pull_async for an ASYNCHRONOUS load
 * (KVConnectorBase_V1.get_num_new_matched_tokens -> (n, is_async=True), base.py:453-486): no
 * stream is made to wait; the caller polls the ticket and only then lets the request run.   */
#define B200KV_STREAM_DETACHED ((void*)(intptr_t)-1)

int b200kv_load_async(b200kv_ctx* ctx, const uint64_t* keys, int32_t n_chunks,
                      const int64_t* slot_mapping, int64_t n_tokens, int32_t skip_chunks,
                      void* compute_stream, uint64_t* ticket, int64_t* n_loaded_tokens);

/* Layer-wise retrieve (LMCache `use_layerwise`: lmcache_engine.retrieve_layer, adapter :870-880;
 * KVConnectorBase_V1.wait_for_layer_load, base.py:310-322).  Same arguments as b200kv_load_async,
 * but the H2D copies and scatters are issued per group of `layers_per_group` layers across all
 * chunks, group 0 first; `compute_stream` is NOT made to wait for the whole load.  Instead the
 * caller calls b200kv_wait_layer(ticket, layer, stream) before the attention of `layer` runs: the
 * PCIe transfer of later layers overlaps the forward pass of earlier ones.  Falls back to one
 * whole-op wait if the op does not fit the load half of the staging ring.                  */
int b200kv_load_layerwise_async(b200kv_ctx* ctx, const uint64_t* keys, int32_t n_chunks,
                                const int64_t* slot_mapping, int64_t n_tokens, int32_t skip_chunks,
                                int32_t layers_per_group, void* compute_stream, uint64_t* ticket,
                                int64_t* n_loaded_tokens);
int b200kv_wait_layer(b200kv_ctx* ctx, uint64_t ticket, int32_t layer, void* compute_stream);

/* One engine step in ONE op.  The adapter calls lmcache_engine.store / .retrieve once per scheduled request
 * (wait_for_save loop vllm_v1_adapter.py:1047-1128, start_load_kv loop :819-905) and moves the slot mapping
 * to the GPU per call (:1072 "TODO pre-allocated buffer"); here the chunks of every request of the step are
 * handed over together: one run table, one upload, one kernel launch per staging batch, one ticket.
 * Chunk c holds chunk_tokens[c] (1..C) tokens whose slots are slot_mapping[c*C .. c*C + chunk_tokens[c]) —
 * the caller lays the requests out back to back, each request's last chunk padded to C entries (padding is
 * never read).  Store: chunks already present are skipped, as in b200kv_store_async.  Load: request r owns
 * chunks [req_first_chunk[r], req_first_chunk[r+1]) and is loaded up to ITS first missing chunk;
 * req_loaded_tokens[r] receives the tokens scheduled for it.  layers_per_group > 0 = layer-wise (see above). */
int b200kv_store_batch_async(b200kv_ctx* ctx, const uint64_t* keys, const int32_t* chunk_tokens,
                             int32_t n_chunks, const int64_t* slot_mapping, void* compute_stream,
                             uint64_t* ticket);
int b200kv_load_batch_async(b200kv_ctx* ctx, const uint64_t* keys, const int32_t* chunk_tokens,
                            int32_t n_chunks, const int32_t* req_first_chunk, int32_t n_reqs,
                            const int64_t* slot_mapping, int32_t layers_per_group, void* compute_stream,
                            uint64_t* ticket, int64_t* req_loaded_tokens);

int b200kv_poll(b200kv_ctx* ctx, uint64_t ticket, int* done);
int b200kv_wait(b200kv_ctx* ctx, uint64_t ticket);
int b200kv_wait_all(b200kv_ctx* ctx);

/* Device-resident halves of store/retrieve (what the GPU connector's to_gpu/from_gpu do):
 * gather paged KV into / scatter from a caller-provided DEVICE buffer of
 * ceil(n_tokens/C) chunks laid out back to back.  Runs on `stream`.                        */
int b200kv_gather(b200kv_ctx* ctx, const int64_t* slot_mapping, int64_t n_tokens,
                  void* dev_chunks, void* stream);
int b200kv_scatter(b200kv_ctx* ctx, const int64_t* slot_mapping, int64_t n_tokens,
                   const void* dev_chunks, void* stream);

/* ---- cross-replica pull over NVLink (replaces the NIXL/UCX push the reference configures,
 * helm/templates/deployment-vllm-multi.yaml:296-324, examples/disaggregated_prefill/start_prefill.sh) */
typedef struct b200kv_ipc_desc {
  uint8_t handle[64];   /* cudaIpcMemHandle_t of the allocation containing the plane         */
  uint64_t offset;      /* byte offset of block 0 inside that allocation                     */
  uint64_t alloc_bytes; /* size of the allocation (informational)                            */
} b200kv_ipc_desc;

/* Export the descriptors of the registered cache, one per plane in the order given at
 * b200kv_register_kv; n_descs must be their count.  import_peer takes as many.             */
int b200kv_export_ipc(b200kv_ctx* ctx, b200kv_ipc_desc* descs_out, int32_t n_descs);
/* Map a peer replica's cache (same model geometry).  `peer_id` is caller-chosen (0..63).  An
 * import that is refused or fails installs nothing and keeps no mapping open (both imports). */
int b200kv_import_peer(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device,
                       const b200kv_ipc_desc* descs, int32_t n_descs,
                       uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks);
/* Same-process variant (tests, single-process multi-GPU): raw peer device pointers, k_ptrs and
 * v_ptrs as at b200kv_register_kv.                                                          */
int b200kv_import_peer_ptrs(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device,
                            const void* const* k_ptrs, const void* const* v_ptrs,
                            uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks);
/* A peer replica of another tensor-parallel size (disaggregated prefill at one TP size, decode at another).  Its
 * K/V planes hold peer_heads KV heads per token; heads [src_head0, src_head0 + n_heads) of them are this engine's
 * heads [dst_head0, dst_head0 + n_heads).  Both sides keep the engine's block_tokens, head_dim, elem_bytes and tile
 * order (NHD or HND).  Which slice a rank pulls from which peer rank: production-stack_b200/b200kv/pd.py, head_slices. */
typedef struct b200kv_head_slice {
  int32_t peer_heads;   /* H_p: KV heads per token in the peer's planes                              */
  int32_t src_head0;    /* first head of the slice among the peer's                                  */
  int32_t dst_head0;    /* first head of the slice among this engine's                               */
  int32_t n_heads;      /* heads in the slice                                                        */
} b200kv_head_slice;
/* b200kv_import_peer / b200kv_import_peer_ptrs of a peer with a head slice: the peer is installed with its slice or
 * not at all, and b200kv_peer_pull_async from it moves the slice's heads only (stats.p2p_bytes counts those).
 * -EINVAL for a NULL slice, a slice outside [0, peer_heads) or outside [0, n_kv_heads), head_dim * elem_bytes not a
 * multiple of 16, a peer block stride below block_tokens * peer_heads * head_dim * elem_bytes, or an MLA engine
 * (a latent is the same on every rank: import the peer whole).                                  */
int b200kv_import_peer_sliced(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device,
                              const b200kv_ipc_desc* descs, int32_t n_descs,
                              uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks,
                              const b200kv_head_slice* slice);
int b200kv_import_peer_ptrs_sliced(b200kv_ctx* ctx, int32_t peer_id, int32_t peer_device,
                                   const void* const* k_ptrs, const void* const* v_ptrs,
                                   uint64_t peer_block_stride_bytes, uint64_t peer_n_blocks,
                                   const b200kv_head_slice* slice);
/* Consumer-side pull: token i is read from peer slot src_slots[i] and written to local slot
 * dst_slots[i]; in-kernel P2P loads, no staging, no NCCL.  `compute_stream` waits for it.  */
int b200kv_peer_pull_async(b200kv_ctx* ctx, int32_t peer_id, const int64_t* src_slots,
                           const int64_t* dst_slots, int64_t n_tokens, void* compute_stream,
                           uint64_t* ticket);

/* ---- device chunk tier (BASELINE.json configs[3]: peer-GPU KV pull over NVLink, no host hop) ----- */
/* gather / scatter with one device pointer PER CHUNK instead of one contiguous buffer: the chunk may
 * sit in this engine's device tier or in a peer replica's (a pointer into a b200kv_tier_import
 * mapping: the scatter kernels then read it with P2P loads over NVSwitch).                        */
int b200kv_gather_chunks(b200kv_ctx* ctx, const int64_t* slot_mapping, int64_t n_tokens,
                         const uint64_t* chunk_ptrs, void* stream);
int b200kv_scatter_chunks(b200kv_ctx* ctx, const int64_t* slot_mapping, int64_t n_tokens,
                          const uint64_t* chunk_ptrs, void* stream);
/* A buffer of n_slots chunk-format slots in HBM (slot i at base + i * chunk_bytes).  Which key sits
 * where, LRU and pins are kept by the caller in a b200kv_pool index in shm, shared with the peers.   */
int b200kv_tier_create(b200kv_ctx* ctx, uint32_t n_slots, uint64_t* base_out);
int b200kv_tier_export(b200kv_ctx* ctx, b200kv_ipc_desc* desc_out);
int b200kv_tier_import(b200kv_ctx* ctx, const b200kv_ipc_desc* desc, uint64_t* mapped_base_out);

int b200kv_engine_get_stats(b200kv_ctx* ctx, b200kv_engine_stats* out);
/* Milliseconds of the most recent gather / scatter / pull kernel batch, measured with CUDA
 * events on the launching stream (valid after the op's ticket completed or the stream was
 * synchronised).  which: 0 = gather, 1 = scatter, 2 = peer pull.                           */
int b200kv_last_kernel_ms(b200kv_ctx* ctx, int which, float* ms_out);

/* ======================================================================================= */
/* remote group (CPU only): the cache-server tier                                           */
/* ======================================================================================= */
/* Stand-in for LMCache's cache server and its client: the chart runs
 * `/opt/venv/bin/lmcache_server 0.0.0.0 <port>` (helm/templates/deployment-cache-server.yaml:
 * 62-65) and gives every engine LMCACHE_REMOTE_URL=lm://<service>:<port> with
 * LMCACHE_REMOTE_SERDE naive|cachegen (helm/templates/deployment-vllm-multi.yaml:338-345,
 * helm/tests/lmcache_test.yaml:166-181).  The server keeps chunks in a b200kv pool of
 * `pool_bytes`, created by the first PUT with the clients' slot size; the client moves a
 * chunk between the socket and a slot of the LOCAL pinned pool directly, so a fetched chunk
 * is loadable by b200kv_load_async at once.  Own wire format (48-byte header + payload);
 * LMCache's is not available here — parity unpinned.  A `b200kv_remote` is one connection;
 * calls on it are serialised internally.                                                   */
typedef struct b200kv_server b200kv_server;
typedef struct b200kv_remote b200kv_remote;
/* host NULL/"0.0.0.0" = any; port 0 = pick one (read it back with b200kv_server_port).     */
int b200kv_server_start(const char* host, int port, uint64_t pool_bytes, b200kv_server** out);
int b200kv_server_port(b200kv_server* srv);
/* out5 = {chunks put, chunks served, get misses, payload bytes in, payload bytes out}.     */
int b200kv_server_get_stats(b200kv_server* srv, uint64_t* out5);
int b200kv_server_stop(b200kv_server* srv);

int b200kv_remote_connect(const char* host, int port, int timeout_ms, b200kv_remote** out);
int b200kv_remote_close(b200kv_remote* r);
int b200kv_remote_ping(b200kv_remote* r);
/* *n_prefix = how many leading keys the server holds (longest stored prefix, like lookup). */
int b200kv_remote_exists(b200kv_remote* r, const uint64_t* keys, int32_t n_keys, int32_t* n_prefix);
/* Local pool -> server.  -ENOENT: not READY locally; -EEXIST: server has it (nothing sent). */
int b200kv_remote_put(b200kv_remote* r, b200kv_pool* local, uint64_t key, uint32_t owner);
/* Server -> local pool (reserve / receive into the slot / commit).  OK if already local.   */
int b200kv_remote_get(b200kv_remote* r, b200kv_pool* local, uint64_t key, uint32_t owner);
int b200kv_remote_stats(b200kv_remote* r, b200kv_pool_stats* out);
int b200kv_remote_traffic(b200kv_remote* r, uint64_t* bytes_up, uint64_t* bytes_down);

/* ======================================================================================= */
/* disk group (CPU only): the local-disk tier                                               */
/* ======================================================================================= */
/* LMCACHE_LOCAL_DISK / LMCACHE_MAX_LOCAL_DISK_SIZE (helm/templates/deployment-vllm-multi.yaml:334-337): chunks
 * below the pinned pool, on local NVMe.  One preallocated file per (directory, chunk size),
 * <dir>/b200kv-disk-<chunk_bytes hex>.slots: a 4 KiB file header, then slots of a 4 KiB slot header (magic,
 * version, key, format tag, token count, owner, payload length, XXH64 of the payload, write time, the file's
 * UUID, XXH64 of the header) followed by the chunk rounded up to 4 KiB.  The index is a b200kv_pool in shm,
 * named after the file, with pool slot i <-> file slot i; every process that opens the file shares it, and one
 * that is new or describes another incarnation of the file is rebuilt from the slot headers.  O_DIRECT I/O
 * (buffered with POSIX_FADV_DONTNEED where the filesystem refuses it).  A `b200kv_disk` may be used from several
 * threads at once.                                                                          */
typedef struct b200kv_disk b200kv_disk;
typedef struct b200kv_disk_stats {
  uint64_t n_slots, n_used;    /* disk slots, slots in use (shared by every opener)                    */
  uint64_t slot_bytes;         /* bytes of one disk slot: 4 KiB header + chunk rounded up to 4 KiB     */
  uint64_t n_put, n_get;       /* chunks written / read back into a pool by this handle               */
  uint64_t n_get_miss;         /* gets of a key the index does not hold                               */
  uint64_t n_corrupt;          /* slots rejected by a header or payload check (never loaded)          */
  uint64_t n_evicted, n_dropped; /* index: LRU evictions; puts refused because every slot was pinned */
  uint64_t bytes_written, bytes_read;
  uint64_t hash_ns, copy_ns, io_ns; /* time in XXH64, in bounce-buffer copies, in pread/pwrite         */
  uint64_t n_restored;         /* chunks the index rebuild at open found in the file                  */
  int32_t direct_io;           /* 1: O_DIRECT, 0: buffered                                            */
  int32_t last_errno;          /* errno of the most recent failed read or write                       */
} b200kv_disk_stats;

/* Opens (creating and preallocating it if needed) the file for chunks of chunk_bytes in the existing directory
 * `dir`, sized to floor((disk_bytes - 4 KiB) / slot_bytes) slots; an existing file keeps its size.  -ENOENT /
 * -ENOTDIR: no such directory; -EACCES / -EROFS: not writable; -ENOSPC: the preallocation does not fit.      */
int b200kv_disk_open(const char* dir, uint64_t disk_bytes, uint64_t chunk_bytes, b200kv_disk** out);
int b200kv_disk_close(b200kv_disk* disk);
/* Local pool -> disk.  -ENOENT: not READY locally; -EEXIST: on disk already; -ENOSPC: every disk slot is
 * pinned or being written; -EIO: the write failed (stats.last_errno says why).              */
int b200kv_disk_put(b200kv_disk* disk, b200kv_pool* local, uint64_t key, uint32_t owner);
/* Disk -> local pool: pin the disk slot, reserve a pool slot, read, verify, commit.  OK also when the chunk is
 * already local.  -ENOENT: not on disk, or it failed its check (then it is dropped from the index);
 * -ENOSPC: no local slot could be freed; -EIO: the read failed.                              */
int b200kv_disk_get(b200kv_disk* disk, b200kv_pool* local, uint64_t key);
/* *n_prefix = how many leading keys the disk holds.                                          */
int b200kv_disk_lookup(b200kv_disk* disk, const uint64_t* keys, int32_t n_keys, int32_t* n_prefix);
int b200kv_disk_get_stats(b200kv_disk* disk, b200kv_disk_stats* out);
/* Empties the index and retires every slot header on disk (KVConnectorBase_V1.reset_cache); -EBUSY if a chunk
 * was pinned or being written and stayed.                                                     */
int b200kv_disk_clear(b200kv_disk* disk);

#ifdef __cplusplus
}
#endif
#endif /* B200KV_H_ */
