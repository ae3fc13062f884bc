// b200kv_pool.cpp — pinned-host chunk pool + cross-process index (CPU only).
//
// Stands in for LMCache's LocalCPUBackend (sized by LMCACHE_MAX_LOCAL_CPU_SIZE,
// helm/templates/deployment-vllm-multi.yaml:326-333) and for the scheduler<->worker lookup
// channel (lookup_client / lookup_server, vllm_v1_adapter.py:609-636): the whole index lives
// in one POSIX shared-memory segment, so the scheduler-role connector (no CUDA context), the
// worker-role connector and — for the "shared pinned-host KV pool" of BASELINE.json config 3 —
// the other replicas on the box all see the same chunks.  The engine cudaHostRegister()s the
// payload area; this file never calls CUDA.
//
// Layout:  [PoolHeader | Slot[n_slots] | bucket[table_cap] | pad to 2 MiB | payload]
#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <new>

#include <dirent.h>
#include <fcntl.h>
#include <sys/file.h>
#include <pthread.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include "b200kv.h"

namespace {

constexpr uint64_t kMagic = 0x6232303030304b56ull;  // "b20000KV"
constexpr uint32_t kVersion = 2;
constexpr uint32_t kNone = 0xffffffffu;
constexpr uint32_t kTomb = 0xfffffffeu;
constexpr uint32_t kEmpty = 0;  // bucket value = slot index + 1

enum SlotState : uint32_t { kFree = 0, kWriting = 1, kReady = 2 };

struct Slot {
  uint64_t key;
  uint64_t lease_until_ns;
  uint32_t state;
  uint32_t fmt;
  int32_t n_tokens;
  uint32_t owner;
  uint32_t pins;
  uint32_t lru_prev, lru_next;  // READY slots, oldest at head
  uint32_t free_next;
  uint32_t pad;
  uint64_t touched_ns;  // reserve time (WRITING) / last acquire (pins): a writer or reader that died
                        // is recognised by age, not by pid (replicas may sit in different pid namespaces)
};

struct PoolHeader {
  uint64_t magic;
  uint32_t version;
  volatile uint32_t ready;
  uint64_t total_bytes, payload_off, payload_bytes, slot_bytes;
  uint32_t n_slots, table_cap;
  uint64_t slots_off, table_off;
  pthread_mutex_t mu;
  uint32_t lru_head, lru_tail, free_head, n_used, n_tombs, pad;
  b200kv_pool_stats stats;
};

uint64_t now_ns() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return static_cast<uint64_t>(ts.tv_sec) * 1000000000ull + static_cast<uint64_t>(ts.tv_nsec);
}

uint64_t round_up(uint64_t x, uint64_t a) { return (x + a - 1) / a * a; }

uint32_t next_pow2(uint32_t x) {
  uint32_t p = 16;
  while (p < x) p <<= 1;
  return p;
}

inline uint64_t mix(uint64_t k) {  // keys are already hashes; cheap finaliser for bucket choice
  k ^= k >> 32;
  k *= 0x9e3779b97f4a7c15ull;
  return k ^ (k >> 29);
}

}  // namespace

struct b200kv_pool {
  PoolHeader* h = nullptr;
  Slot* slots = nullptr;
  uint32_t* table = nullptr;
  uint8_t* payload = nullptr;
  uint64_t map_bytes = 0;
  bool creator = false;
  char name[256] = {0};
  // Named segments: every process that has the pool open holds a shared flock on the segment's file for as
  // long as it lives (the kernel drops it when the process dies, however it dies).  b200kv_pool_sweep()
  // removes segments nobody holds: what a SIGKILLed / OOM-killed engine left behind in /dev/shm.
  int lock_fd = -1;
  ~b200kv_pool() { if (lock_fd >= 0) close(lock_fd); }

  uint64_t stale_ns = 120ull * 1000000000ull;  // B200KV_POOL_STALE_MS
  uint64_t die_key = 0;  // fault injection (tests): _exit inside the critical section of reserve(die_key)

  struct Guard {
    PoolHeader* h;
    explicit Guard(b200kv_pool* p) : h(p->h) {
      int rc = pthread_mutex_lock(&h->mu);
      if (rc == EOWNERDEAD) {
        // A process died inside a critical section: lists and table may be half-updated.  Slot
        // states and keys are written last-writer-wins and are the ground truth; rebuild the rest.
        p->recover();
        pthread_mutex_consistent(&h->mu);
      }
    }
    ~Guard() { pthread_mutex_unlock(&h->mu); }
  };

  // ---- index primitives (mutex held) ----------------------------------------------------
  uint32_t find(uint64_t key) const {
    const uint32_t mask = h->table_cap - 1;
    uint32_t b = static_cast<uint32_t>(mix(key)) & mask;
    for (uint32_t probe = 0; probe < h->table_cap; ++probe, b = (b + 1) & mask) {
      const uint32_t v = table[b];
      if (v == kEmpty) return kNone;
      if (v == kTomb) continue;
      if (slots[v - 1].key == key) return v - 1;
    }
    return kNone;
  }
  void table_insert(uint32_t slot) {
    const uint32_t mask = h->table_cap - 1;
    uint32_t b = static_cast<uint32_t>(mix(slots[slot].key)) & mask;
    while (table[b] != kEmpty && table[b] != kTomb) b = (b + 1) & mask;
    if (table[b] == kTomb) --h->n_tombs;
    table[b] = slot + 1;
  }
  void table_erase(uint32_t slot) {
    const uint32_t mask = h->table_cap - 1;
    uint32_t b = static_cast<uint32_t>(mix(slots[slot].key)) & mask;
    for (uint32_t probe = 0; probe < h->table_cap; ++probe, b = (b + 1) & mask) {
      if (table[b] == slot + 1) {
        table[b] = kTomb;
        ++h->n_tombs;
        break;
      }
      if (table[b] == kEmpty) break;
    }
  }
  void rebuild() {
    std::memset(table, 0, sizeof(uint32_t) * h->table_cap);
    h->n_tombs = 0;
    for (uint32_t s = 0; s < h->n_slots; ++s)
      if (slots[s].state != kFree) table_insert(s);
  }
  void lru_unlink(uint32_t s) {
    Slot& e = slots[s];
    if (e.lru_prev != kNone) slots[e.lru_prev].lru_next = e.lru_next;
    else if (h->lru_head == s) h->lru_head = e.lru_next;
    if (e.lru_next != kNone) slots[e.lru_next].lru_prev = e.lru_prev;
    else if (h->lru_tail == s) h->lru_tail = e.lru_prev;
    e.lru_prev = e.lru_next = kNone;
  }
  void lru_push_tail(uint32_t s) {
    Slot& e = slots[s];
    e.lru_prev = h->lru_tail;
    e.lru_next = kNone;
    if (h->lru_tail != kNone) slots[h->lru_tail].lru_next = s;
    h->lru_tail = s;
    if (h->lru_head == kNone) h->lru_head = s;
  }
  void free_slot(uint32_t s) {
    Slot& e = slots[s];
    table_erase(s);
    e.state = kFree;
    if (h->n_tombs > h->table_cap / 4) rebuild();  // after state flips: rebuild skips free slots
    e.pins = 0;
    e.lease_until_ns = 0;
    e.free_next = h->free_head;
    h->free_head = s;
    --h->n_used;
  }
  bool stale(const Slot& e, uint64_t t) const { return t > e.touched_ns && t - e.touched_ns > stale_ns; }
  uint32_t pop_free() {
    const uint32_t s = h->free_head;
    h->free_head = slots[s].free_next;
    return s;
  }
  uint32_t take_slot() {  // free list first, then LRU eviction, then slots abandoned by dead processes
    if (h->free_head != kNone) return pop_free();
    const uint64_t t = now_ns();
    for (uint32_t s = h->lru_head; s != kNone; s = slots[s].lru_next) {
      Slot& e = slots[s];
      if (e.pins && stale(e, t)) {  // a reader died between acquire and release
        e.pins = 0;
        ++h->stats.n_reclaimed_chunks;
      }
      if (e.pins == 0 && e.lease_until_ns <= t) {
        lru_unlink(s);
        free_slot(s);
        ++h->stats.n_evicted_chunks;
        return pop_free();
      }
    }
    for (uint32_t s = 0; s < h->n_slots; ++s) {  // a writer died between reserve and commit
      if (slots[s].state == kWriting && stale(slots[s], t)) {
        free_slot(s);
        ++h->stats.n_reclaimed_chunks;
        return pop_free();
      }
    }
    return kNone;
  }
  // Rebuild every derived structure from the slot array (after EOWNERDEAD).
  void recover() {
    h->free_head = kNone;
    h->lru_head = h->lru_tail = kNone;
    h->n_used = 0;
    for (uint32_t s = h->n_slots; s-- > 0;) {
      Slot& e = slots[s];
      if (e.state != kWriting && e.state != kReady) e.state = kFree;
      e.lru_prev = e.lru_next = kNone;
      if (e.state == kFree) {
        e.pins = 0;
        e.lease_until_ns = 0;
        e.free_next = h->free_head;
        h->free_head = s;
      } else {
        ++h->n_used;
      }
    }
    // duplicates of one key cannot both be kept (a reserve died after writing the second): keep READY
    rebuild_dedup();
    for (uint32_t s = 0; s < h->n_slots; ++s)
      if (slots[s].state == kReady) lru_push_tail(s);
    ++h->stats.n_recoveries;
  }
  void rebuild_dedup() {
    std::memset(table, 0, sizeof(uint32_t) * h->table_cap);
    h->n_tombs = 0;
    for (int pass = 0; pass < 2; ++pass) {  // READY first, so a WRITING twin loses
      for (uint32_t s = 0; s < h->n_slots; ++s) {
        Slot& e = slots[s];
        if (e.state != (pass == 0 ? kReady : kWriting)) continue;
        if (find(e.key) != kNone) {
          e.state = kFree;
          e.pins = 0;
          e.lease_until_ns = 0;
          e.free_next = h->free_head;
          h->free_head = s;
          --h->n_used;
          continue;
        }
        table_insert(s);
      }
    }
  }
};

namespace {

void init_header(b200kv_pool* p, uint64_t total, uint64_t slots_off, uint64_t table_off,
                 uint64_t payload_off, uint64_t payload_bytes, uint64_t slot_bytes,
                 uint32_t n_slots, uint32_t cap) {
  PoolHeader* h = p->h;
  std::memset(h, 0, sizeof(PoolHeader));
  h->magic = kMagic;
  h->version = kVersion;
  h->total_bytes = total;
  h->payload_off = payload_off;
  h->payload_bytes = payload_bytes;
  h->slot_bytes = slot_bytes;
  h->n_slots = n_slots;
  h->table_cap = cap;
  h->slots_off = slots_off;
  h->table_off = table_off;
  pthread_mutexattr_t at;
  pthread_mutexattr_init(&at);
  pthread_mutexattr_setpshared(&at, PTHREAD_PROCESS_SHARED);
  pthread_mutexattr_setrobust(&at, PTHREAD_MUTEX_ROBUST);
  pthread_mutex_init(&h->mu, &at);
  pthread_mutexattr_destroy(&at);
  h->lru_head = h->lru_tail = kNone;
  h->free_head = kNone;
  p->slots = reinterpret_cast<Slot*>(reinterpret_cast<uint8_t*>(h) + slots_off);
  p->table = reinterpret_cast<uint32_t*>(reinterpret_cast<uint8_t*>(h) + table_off);
  for (uint32_t s = n_slots; s-- > 0;) {
    Slot& e = p->slots[s];
    std::memset(&e, 0, sizeof(Slot));
    e.lru_prev = e.lru_next = kNone;
    e.free_next = h->free_head;
    h->free_head = s;
  }
  std::memset(p->table, 0, sizeof(uint32_t) * cap);
  h->stats.n_slots = n_slots;
  h->stats.slot_bytes = slot_bytes;
  __atomic_store_n(&h->ready, 1u, __ATOMIC_RELEASE);
}

void bind_views(b200kv_pool* p) {
  uint8_t* base = reinterpret_cast<uint8_t*>(p->h);
  p->slots = reinterpret_cast<Slot*>(base + p->h->slots_off);
  p->table = reinterpret_cast<uint32_t*>(base + p->h->table_off);
  p->payload = base + p->h->payload_off;
}

}  // namespace

extern "C" int b200kv_pool_open(const b200kv_pool_config* cfg, b200kv_pool** out) {
  if (!cfg || !out) return B200KV_EINVAL;
  *out = nullptr;
  const bool want_create = cfg->flags & B200KV_POOL_CREATE;
  const bool want_attach = cfg->flags & B200KV_POOL_ATTACH;
  if (!want_create && !want_attach) return B200KV_EINVAL;
  if (!cfg->shm_name && !want_create) return B200KV_EINVAL;

  b200kv_pool* p = new (std::nothrow) b200kv_pool();
  if (!p) return B200KV_ENOMEM;
  if (const char* e = getenv("B200KV_POOL_STALE_MS")) {
    const long long ms = atoll(e);
    if (ms > 0) p->stale_ns = static_cast<uint64_t>(ms) * 1000000ull;
  }
  if (const char* e = getenv("B200KV_POOL_TEST_DIE_KEY")) p->die_key = strtoull(e, nullptr, 10);

  int fd = -1;
  bool creating = false;
  if (cfg->shm_name) {
    if (cfg->shm_name[0] != '/' || std::strlen(cfg->shm_name) >= sizeof(p->name)) {
      delete p;
      return B200KV_EINVAL;
    }
    std::snprintf(p->name, sizeof(p->name), "%s", cfg->shm_name);
    if (want_create) {
      fd = shm_open(cfg->shm_name, O_RDWR | O_CREAT | O_EXCL, 0600);
      if (fd >= 0) creating = true;
      else if (errno != EEXIST || !want_attach) {
        const int e = errno;
        delete p;
        return -e;
      }
    }
    if (fd < 0) {
      fd = shm_open(cfg->shm_name, O_RDWR, 0600);
      if (fd < 0) {
        const int e = errno;
        delete p;
        return -e;
      }
    }
    flock(fd, LOCK_SH);
    p->lock_fd = fd;      // stays open (and locked) until b200kv_pool_close / process exit
  } else {
    creating = true;
  }

  if (creating) {
    if (cfg->slot_bytes == 0 || cfg->slot_bytes % 16 || cfg->pool_bytes < cfg->slot_bytes) {
      if (fd >= 0) shm_unlink(cfg->shm_name);
      delete p;
      return B200KV_EINVAL;
    }
    const uint64_t n_slots64 = cfg->pool_bytes / cfg->slot_bytes;
    if (n_slots64 > 0x7fffffffu) {
      if (fd >= 0) shm_unlink(cfg->shm_name);
      delete p;
      return B200KV_EINVAL;
    }
    const uint32_t n_slots = static_cast<uint32_t>(n_slots64);
    const uint32_t cap = next_pow2(n_slots * 4u);
    const uint64_t slots_off = round_up(sizeof(PoolHeader), 64);
    const uint64_t table_off = round_up(slots_off + sizeof(Slot) * n_slots, 64);
    const uint64_t payload_off = round_up(table_off + sizeof(uint32_t) * cap, 2ull << 20);
    const uint64_t payload_bytes = static_cast<uint64_t>(n_slots) * cfg->slot_bytes;
    const uint64_t total = payload_off + payload_bytes;
    void* m;
    if (fd >= 0) {
      if (ftruncate(fd, static_cast<off_t>(total)) != 0) {
        const int e = errno;
        shm_unlink(cfg->shm_name);
        delete p;
        return -e;
      }
      m = mmap(nullptr, total, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    } else {
      m = mmap(nullptr, total, PROT_READ | PROT_WRITE, MAP_SHARED | MAP_ANONYMOUS, -1, 0);
    }
    if (m == MAP_FAILED) {
      const int e = errno;
      if (cfg->shm_name) shm_unlink(cfg->shm_name);
      delete p;
      return -e;
    }
    p->h = static_cast<PoolHeader*>(m);
    p->map_bytes = total;
    p->creator = true;
    init_header(p, total, slots_off, table_off, payload_off, payload_bytes, cfg->slot_bytes,
                n_slots, cap);
    bind_views(p);
  } else {
    // Attach: wait (bounded) for the creator to size and initialise the segment.
    struct stat st;
    uint64_t size = 0;
    for (int i = 0; i < 5000; ++i) {
      if (fstat(fd, &st) == 0 && static_cast<uint64_t>(st.st_size) >= sizeof(PoolHeader)) {
        size = static_cast<uint64_t>(st.st_size);
        break;
      }
      usleep(1000);
    }
    if (!size) {
      delete p;
      return B200KV_ENOENT;
    }
    void* m = mmap(nullptr, size, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
    if (m == MAP_FAILED) {
      const int e = errno;
      delete p;
      return -e;
    }
    p->h = static_cast<PoolHeader*>(m);
    p->map_bytes = size;
    bool ok = false;
    for (int i = 0; i < 5000; ++i) {
      if (__atomic_load_n(&p->h->ready, __ATOMIC_ACQUIRE) == 1u) {
        ok = true;
        break;
      }
      usleep(1000);
    }
    if (!ok || p->h->magic != kMagic || p->h->version != kVersion ||
        p->h->total_bytes != size) {
      munmap(m, size);
      delete p;
      return B200KV_EINVAL;
    }
    if (cfg->slot_bytes && cfg->slot_bytes != p->h->slot_bytes) {
      munmap(m, size);
      delete p;
      return B200KV_EINVAL;  // geometry mismatch between replicas sharing one pool
    }
    bind_views(p);
  }
  *out = p;
  return B200KV_OK;
}

extern "C" int b200kv_pool_close(b200kv_pool* pool) {
  if (!pool) return B200KV_EINVAL;
  if (pool->h) munmap(pool->h, pool->map_bytes);
  delete pool;
  return B200KV_OK;
}

extern "C" int b200kv_pool_sweep(const char* prefix, int32_t min_age_s, int32_t* n_removed) {
  if (!prefix || !*prefix) return B200KV_EINVAL;
  if (n_removed) *n_removed = 0;
  const char* pfx = prefix[0] == '/' ? prefix + 1 : prefix;
  DIR* d = opendir("/dev/shm");
  if (!d) return -errno;
  const size_t n = std::strlen(pfx);
  const time_t now = time(nullptr);
  while (dirent* e = readdir(d)) {
    if (std::strncmp(e->d_name, pfx, n) != 0) continue;
    char name[300];
    std::snprintf(name, sizeof(name), "/%s", e->d_name);
    const int fd = shm_open(name, O_RDWR, 0600);
    if (fd < 0) continue;
    struct stat st;
    // young segments may belong to a creator that has not taken its lock yet
    if (fstat(fd, &st) == 0 && S_ISREG(st.st_mode) && now - st.st_mtime >= min_age_s &&
        flock(fd, LOCK_EX | LOCK_NB) == 0) {
      if (shm_unlink(name) == 0 && n_removed) ++*n_removed;
    }
    close(fd);
  }
  closedir(d);
  return B200KV_OK;
}

extern "C" int b200kv_pool_unlink(const char* shm_name) {
  if (!shm_name) return B200KV_EINVAL;
  if (shm_unlink(shm_name) != 0) return -errno;
  return B200KV_OK;
}

extern "C" int b200kv_pool_region(b200kv_pool* pool, void** base, uint64_t* bytes) {
  if (!pool || !base || !bytes) return B200KV_EINVAL;
  *base = pool->payload;
  *bytes = pool->h->payload_bytes;
  return B200KV_OK;
}

extern "C" void* b200kv_pool_slot_ptr(b200kv_pool* pool, uint32_t slot) {
  if (!pool || slot >= pool->h->n_slots) return nullptr;
  return pool->payload + static_cast<uint64_t>(slot) * pool->h->slot_bytes;
}

extern "C" int b200kv_pool_lookup(b200kv_pool* pool, const uint64_t* keys,
                                  const int32_t* chunk_tokens, int32_t n_keys,
                                  uint32_t lease_ms, int32_t* n_hit_chunks,
                                  int64_t* n_hit_tokens) {
  if (!pool || n_keys < 0 || (n_keys > 0 && (!keys || !chunk_tokens))) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  const uint64_t lease = now_ns() + static_cast<uint64_t>(lease_ms) * 1000000ull;
  int32_t hits = 0;
  int64_t toks = 0, req = 0;
  for (int32_t i = 0; i < n_keys; ++i) req += chunk_tokens[i];
  for (int32_t i = 0; i < n_keys; ++i) {
    const uint32_t s = pool->find(keys[i]);
    if (s == kNone) break;
    Slot& e = pool->slots[s];
    if (e.state != kReady || e.n_tokens != chunk_tokens[i]) break;
    if (lease_ms && e.lease_until_ns < lease) e.lease_until_ns = lease;
    pool->lru_unlink(s);
    pool->lru_push_tail(s);
    ++hits;
    toks += e.n_tokens;
  }
  pool->h->stats.n_lookups += 1;
  pool->h->stats.n_lookup_chunks += static_cast<uint64_t>(n_keys);
  pool->h->stats.n_hit_chunks += static_cast<uint64_t>(hits);
  pool->h->stats.n_hit_tokens += static_cast<uint64_t>(toks);
  pool->h->stats.n_requested_tokens += static_cast<uint64_t>(req);
  if (n_hit_chunks) *n_hit_chunks = hits;
  if (n_hit_tokens) *n_hit_tokens = toks;
  return B200KV_OK;
}

extern "C" int b200kv_pool_lookup_owner(b200kv_pool* pool, const uint64_t* keys, int32_t n_keys,
                                        int32_t* n_hit_chunks, uint32_t* owner_out) {
  if (!pool || n_keys < 0 || (n_keys > 0 && !keys)) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  int32_t hits = 0;
  for (int32_t i = 0; i < n_keys; ++i) {
    const uint32_t s = pool->find(keys[i]);
    if (s == kNone || pool->slots[s].state != kReady) break;
    if (owner_out) owner_out[i] = pool->slots[s].owner;
    ++hits;
  }
  if (n_hit_chunks) *n_hit_chunks = hits;
  return B200KV_OK;
}

extern "C" int b200kv_pool_contains(b200kv_pool* pool, const uint64_t* keys, const int32_t* chunk_tokens,
                                    int32_t n_keys, uint32_t lease_ms, uint8_t* present) {
  if (!pool || n_keys < 0 || (n_keys > 0 && (!keys || !present))) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  const uint64_t lease = now_ns() + static_cast<uint64_t>(lease_ms) * 1000000ull;
  for (int32_t i = 0; i < n_keys; ++i) {
    const uint32_t s = pool->find(keys[i]);
    present[i] = 0;
    if (s == kNone) continue;
    Slot& e = pool->slots[s];
    if (e.state != kReady || (chunk_tokens && e.n_tokens != chunk_tokens[i])) continue;
    if (lease_ms && e.lease_until_ns < lease) e.lease_until_ns = lease;
    present[i] = 1;
  }
  return B200KV_OK;
}

extern "C" int b200kv_pool_reserve(b200kv_pool* pool, uint64_t key, int32_t n_tokens,
                                   uint32_t fmt, uint32_t owner, uint32_t* slot_out) {
  if (!pool || !slot_out || n_tokens <= 0) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  const uint32_t twin = pool->find(key);
  if (twin != kNone) {
    Slot& t = pool->slots[twin];
    if (t.state != kWriting || !pool->stale(t, now_ns())) return B200KV_EEXIST;
    pool->free_slot(twin);  // its writer died long ago: take the key over
    ++pool->h->stats.n_reclaimed_chunks;
  }
  const uint32_t s = pool->take_slot();
  if (s == kNone) {
    ++pool->h->stats.n_dropped_chunks;
    return B200KV_ENOSPC;
  }
  Slot& e = pool->slots[s];
  e.key = key;
  e.state = kWriting;
  e.fmt = fmt;
  e.n_tokens = n_tokens;
  e.owner = owner;
  e.pins = 0;
  e.lease_until_ns = 0;
  e.touched_ns = now_ns();
  e.lru_prev = e.lru_next = kNone;
  pool->table_insert(s);
  if (pool->die_key && key == pool->die_key) _exit(9);  // lock held, n_used not yet updated
  ++pool->h->n_used;
  *slot_out = s;
  return B200KV_OK;
}

extern "C" int b200kv_pool_commit(b200kv_pool* pool, uint64_t key) {
  if (!pool) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  const uint32_t s = pool->find(key);
  if (s == kNone || pool->slots[s].state != kWriting) return B200KV_ENOENT;
  pool->slots[s].state = kReady;
  pool->lru_push_tail(s);
  ++pool->h->stats.n_stored_chunks;
  return B200KV_OK;
}

extern "C" int b200kv_pool_abort(b200kv_pool* pool, uint64_t key) {
  if (!pool) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  const uint32_t s = pool->find(key);
  if (s == kNone || pool->slots[s].state != kWriting) return B200KV_ENOENT;
  pool->free_slot(s);
  return B200KV_OK;
}

extern "C" int b200kv_pool_acquire(b200kv_pool* pool, uint64_t key, uint32_t* slot_out,
                                   int32_t* n_tokens_out, uint32_t* fmt_out) {
  if (!pool || !slot_out) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  const uint32_t s = pool->find(key);
  if (s == kNone || pool->slots[s].state != kReady) return B200KV_ENOENT;
  Slot& e = pool->slots[s];
  ++e.pins;
  e.touched_ns = now_ns();
  pool->lru_unlink(s);
  pool->lru_push_tail(s);
  *slot_out = s;
  if (n_tokens_out) *n_tokens_out = e.n_tokens;
  if (fmt_out) *fmt_out = e.fmt;
  return B200KV_OK;
}

extern "C" int b200kv_pool_release(b200kv_pool* pool, uint64_t key) {
  if (!pool) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  const uint32_t s = pool->find(key);
  if (s == kNone || pool->slots[s].state != kReady || pool->slots[s].pins == 0)
    return B200KV_ENOENT;
  --pool->slots[s].pins;
  return B200KV_OK;
}

extern "C" int b200kv_pool_place(b200kv_pool* pool, const uint32_t* slots, const uint64_t* keys,
                                 const int32_t* n_tokens, const uint32_t* fmts, const uint32_t* owners, int32_t n) {
  if (!pool || n < 0 || (n > 0 && (!slots || !keys || !n_tokens || !fmts || !owners))) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  int32_t placed = 0;
  const uint64_t t = now_ns();
  for (int32_t i = 0; i < n; ++i) {
    const uint32_t s = slots[i];
    if (s >= pool->h->n_slots || pool->slots[s].state != kFree || n_tokens[i] <= 0 || pool->find(keys[i]) != kNone)
      continue;
    Slot& e = pool->slots[s];
    e.key = keys[i];
    e.state = kReady;
    e.fmt = fmts[i];
    e.n_tokens = n_tokens[i];
    e.owner = owners[i];
    e.pins = 0;
    e.lease_until_ns = 0;
    e.touched_ns = t;
    pool->table_insert(s);
    pool->lru_push_tail(s);
    ++pool->h->n_used;
    ++placed;
  }
  if (placed) {  // the free list skips the slots just taken
    pool->h->free_head = kNone;
    for (uint32_t s = pool->h->n_slots; s-- > 0;) {
      if (pool->slots[s].state != kFree) continue;
      pool->slots[s].free_next = pool->h->free_head;
      pool->h->free_head = s;
    }
  }
  return placed;
}

extern "C" int b200kv_pool_drop(b200kv_pool* pool, uint64_t key) {
  if (!pool) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  const uint32_t s = pool->find(key);
  if (s == kNone || pool->slots[s].state != kReady) return B200KV_ENOENT;
  if (pool->slots[s].pins) return B200KV_EBUSY;
  pool->lru_unlink(s);
  pool->free_slot(s);
  return B200KV_OK;
}

extern "C" int b200kv_pool_get_stats(b200kv_pool* pool, b200kv_pool_stats* out) {
  if (!pool || !out) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  *out = pool->h->stats;
  out->n_slots = pool->h->n_slots;
  out->n_used = pool->h->n_used;
  out->slot_bytes = pool->h->slot_bytes;
  return B200KV_OK;
}

extern "C" int b200kv_pool_check(b200kv_pool* pool) {
  if (!pool) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  const uint32_t n = pool->h->n_slots;
  uint32_t n_free = 0, n_ready = 0, n_writing = 0, walked = 0;
  for (uint32_t s = 0; s < n; ++s) {
    const uint32_t st = pool->slots[s].state;
    n_free += st == kFree;
    n_ready += st == kReady;
    n_writing += st == kWriting;
    if (st != kFree && pool->find(pool->slots[s].key) != s) return B200KV_EIO;  // not (uniquely) indexed
  }
  if (n_free + n_ready + n_writing != n || pool->h->n_used != n_ready + n_writing) return B200KV_EIO;
  for (uint32_t s = pool->h->free_head; s != kNone; s = pool->slots[s].free_next)
    if (++walked > n || pool->slots[s].state != kFree) return B200KV_EIO;
  if (walked != n_free) return B200KV_EIO;
  walked = 0;
  uint32_t prev = kNone;
  for (uint32_t s = pool->h->lru_head; s != kNone; prev = s, s = pool->slots[s].lru_next)
    if (++walked > n || pool->slots[s].state != kReady || pool->slots[s].lru_prev != prev) return B200KV_EIO;
  if (walked != n_ready || pool->h->lru_tail != prev) return B200KV_EIO;
  return B200KV_OK;
}

extern "C" int b200kv_pool_clear(b200kv_pool* pool) {
  if (!pool) return B200KV_EINVAL;
  b200kv_pool::Guard g(pool);
  int busy = 0;
  for (uint32_t s = 0; s < pool->h->n_slots; ++s) {
    Slot& e = pool->slots[s];
    if (e.state == kReady && e.pins == 0) {
      pool->lru_unlink(s);
      pool->free_slot(s);
    } else if (e.state != kFree) {
      ++busy;
    }
  }
  return busy ? B200KV_EBUSY : B200KV_OK;
}
