// Host-side race / memory check of the CPU parts of libb200kv (pool index, cache server + client, disk tier):
// built with -fsanitize=thread and again with -fsanitize=address,undefined by tools/sanitize_host.sh.
// Threads hammer one pool through the public C ABI (writers, pinned readers verifying the payload,
// lookups, clears) while other threads push and fetch chunks through a cache server, and others write
// chunks to and read them from one disk tier small enough to evict all the time; any chunk whose
// bytes do not match its key, or a failed b200kv_pool_check, is an error.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <thread>
#include <vector>

#include <stdlib.h>
#include <sys/stat.h>
#include <unistd.h>

#include "b200kv.h"

static constexpr uint64_t kSlot = 16 * 1024;
static std::atomic<long> g_errors{0}, g_ops{0};

static void fill(uint8_t* p, uint64_t key) {
  for (uint64_t i = 0; i < kSlot; i += 8) {
    const uint64_t v = key * 0x9e3779b97f4a7c15ull + i;
    memcpy(p + i, &v, 8);
  }
}
static bool verify(const uint8_t* p, uint64_t key) {
  for (uint64_t i = 0; i < kSlot; i += 8) {
    uint64_t v;
    memcpy(&v, p + i, 8);
    if (v != key * 0x9e3779b97f4a7c15ull + i) return false;
  }
  return true;
}

static b200kv_pool* open_pool(uint32_t n_slots) {
  b200kv_pool_config pc;
  memset(&pc, 0, sizeof(pc));
  pc.pool_bytes = n_slots * kSlot;
  pc.slot_bytes = kSlot;
  pc.flags = B200KV_POOL_CREATE;
  b200kv_pool* p = nullptr;
  if (b200kv_pool_open(&pc, &p) != 0) abort();
  return p;
}

static void pool_worker(b200kv_pool* pool, int seed, int iters) {
  std::mt19937_64 rng(seed);
  for (int i = 0; i < iters; ++i) {
    const uint64_t key = 1 + rng() % 48;
    switch (rng() % 8) {
      case 0: case 1: case 2: {
        uint32_t slot;
        if (b200kv_pool_reserve(pool, key, 256, 0, seed, &slot) == 0) {
          fill(static_cast<uint8_t*>(b200kv_pool_slot_ptr(pool, slot)), key);
          if (rng() % 16 == 0) b200kv_pool_abort(pool, key);
          else b200kv_pool_commit(pool, key);
        }
        break;
      }
      case 3: case 4: case 5: {
        uint32_t slot, fmt;
        int32_t n;
        if (b200kv_pool_acquire(pool, key, &slot, &n, &fmt) == 0) {
          if (!verify(static_cast<const uint8_t*>(b200kv_pool_slot_ptr(pool, slot)), key)) ++g_errors;
          b200kv_pool_release(pool, key);
        }
        break;
      }
      case 6: {
        uint64_t keys[4] = {key, key + 1, key + 2, key + 3};
        int32_t ct[4] = {256, 256, 256, 256}, hc;
        int64_t ht;
        uint32_t owners[4];
        b200kv_pool_lookup(pool, keys, ct, 4, i % 3 ? 0 : 1, &hc, &ht);
        b200kv_pool_lookup_owner(pool, keys, 4, &hc, owners);
        break;
      }
      default:
        if (rng() % 64 == 0) b200kv_pool_clear(pool);
        else { b200kv_pool_stats st; b200kv_pool_get_stats(pool, &st); }
    }
    ++g_ops;
  }
}

static void remote_worker(int port, int seed, int iters) {
  b200kv_pool* local = open_pool(8);
  b200kv_remote* r = nullptr;
  if (b200kv_remote_connect("127.0.0.1", port, 5000, &r) != 0) { ++g_errors; return; }
  std::mt19937_64 rng(seed);
  for (int i = 0; i < iters; ++i) {
    const uint64_t key = 1000 + rng() % 24;
    if (rng() % 2) {
      uint32_t slot;
      if (b200kv_pool_reserve(local, key, 256, 0, seed, &slot) == 0) {
        fill(static_cast<uint8_t*>(b200kv_pool_slot_ptr(local, slot)), key);
        b200kv_pool_commit(local, key);
      }
      const int rc = b200kv_remote_put(r, local, key, seed);
      if (rc != 0 && rc != B200KV_EEXIST && rc != B200KV_ENOENT && rc != B200KV_ENOSPC) ++g_errors;
    } else {
      const int rc = b200kv_remote_get(r, local, key, seed);
      if (rc == 0) {
        uint32_t slot, fmt;
        int32_t n;
        if (b200kv_pool_acquire(local, key, &slot, &n, &fmt) == 0) {
          if (!verify(static_cast<const uint8_t*>(b200kv_pool_slot_ptr(local, slot)), key)) ++g_errors;
          b200kv_pool_release(local, key);
        }
      } else if (rc != B200KV_ENOENT && rc != B200KV_ENOSPC) {
        ++g_errors;
      }
    }
    int32_t n_prefix;
    uint64_t ks[2] = {key, key + 1};
    if (b200kv_remote_exists(r, ks, 2, &n_prefix) != 0) ++g_errors;
    ++g_ops;
  }
  b200kv_remote_close(r);
  if (b200kv_pool_check(local) != 0) ++g_errors;
  b200kv_pool_close(local);
}

// Every disk thread has its own pool (as every engine has) and shares the disk handle and its index.
static void disk_worker(b200kv_disk* disk, int seed, int iters) {
  b200kv_pool* local = open_pool(8);
  std::mt19937_64 rng(seed);
  for (int i = 0; i < iters; ++i) {
    const uint64_t key = 5000 + rng() % 32;
    switch (rng() % 4) {
      case 0: {
        uint32_t slot;
        if (b200kv_pool_reserve(local, key, 256, 0, seed, &slot) == 0) {
          fill(static_cast<uint8_t*>(b200kv_pool_slot_ptr(local, slot)), key);
          b200kv_pool_commit(local, key);
        }
        const int rc = b200kv_disk_put(disk, local, key, seed);
        if (rc != 0 && rc != B200KV_EEXIST && rc != B200KV_ENOENT && rc != B200KV_ENOSPC) ++g_errors;
        break;
      }
      case 1: case 2: {
        const int rc = b200kv_disk_get(disk, local, key);
        if (rc == 0) {
          uint32_t slot, fmt;
          int32_t n;
          if (b200kv_pool_acquire(local, key, &slot, &n, &fmt) == 0) {
            if (!verify(static_cast<const uint8_t*>(b200kv_pool_slot_ptr(local, slot)), key)) ++g_errors;
            b200kv_pool_release(local, key);
          }
        } else if (rc != B200KV_ENOENT && rc != B200KV_ENOSPC) {
          ++g_errors;
        }
        break;
      }
      default: {
        uint64_t ks[3] = {key, key + 1, key + 2};
        int32_t n_prefix;
        if (b200kv_disk_lookup(disk, ks, 3, &n_prefix) != 0) ++g_errors;
        if (rng() % 256 == 0) b200kv_pool_clear(local);
        if (rng() % 512 == 0) b200kv_disk_clear(disk);
      }
    }
    ++g_ops;
  }
  if (b200kv_pool_check(local) != 0) ++g_errors;
  b200kv_pool_close(local);
}

int main(int argc, char** argv) {
  const int iters = argc > 1 ? atoi(argv[1]) : 20000;
  b200kv_pool* pool = open_pool(16);
  b200kv_server* srv = nullptr;
  if (b200kv_server_start("127.0.0.1", 0, 12 * kSlot, &srv) != 0) abort();
  const int port = b200kv_server_port(srv);
  std::vector<std::thread> ts;
  for (int t = 0; t < 6; ++t) ts.emplace_back(pool_worker, pool, 100 + t, iters);
  for (int t = 0; t < 4; ++t) ts.emplace_back(remote_worker, port, 200 + t, iters / 10);
  const char* tmp = getenv("TMPDIR");
  std::string dtmpl = std::string(tmp && *tmp ? tmp : "/tmp") + "/b200kv-sanitize-disk-XXXXXX";
  std::vector<char> dbuf(dtmpl.begin(), dtmpl.end());
  dbuf.push_back(0);
  if (!mkdtemp(dbuf.data())) abort();
  b200kv_disk* disk = nullptr;
  // 12 disk slots of 4 KiB header + 16 KiB chunk for 32 keys: evictions all the time
  if (b200kv_disk_open(dbuf.data(), 4096 + 12 * (4096 + kSlot), kSlot, &disk) != 0) abort();
  for (int t = 0; t < 4; ++t) ts.emplace_back(disk_worker, disk, 300 + t, iters / 10);
  for (auto& t : ts) t.join();
  b200kv_disk_stats ds;
  b200kv_disk_get_stats(disk, &ds);
  b200kv_disk_close(disk);
  if (ds.n_corrupt) ++g_errors;
  // remove the file and its index in shm, which is named after the file (b200kv_disk_open)
  char path[600], name[64];
  snprintf(path, sizeof(path), "%s/b200kv-disk-%llx.slots", dbuf.data(), (unsigned long long)kSlot);
  struct stat fst;
  if (stat(path, &fst) == 0) {
    const uint64_t id[3] = {(uint64_t)fst.st_dev, (uint64_t)fst.st_ino, kSlot};
    snprintf(name, sizeof(name), "/b200kv-disk-%016llx", (unsigned long long)b200kv_xxh64(id, sizeof(id), 0));
    b200kv_pool_unlink(name);
  }
  unlink(path);
  rmdir(dbuf.data());
  if (b200kv_pool_check(pool) != 0) ++g_errors;
  b200kv_pool_stats st;
  b200kv_pool_get_stats(pool, &st);
  uint64_t s5[5];
  b200kv_server_get_stats(srv, s5);
  b200kv_server_stop(srv);
  b200kv_pool_close(pool);
  printf("ops=%ld errors=%ld pool: stored=%llu evicted=%llu dropped=%llu server: put=%llu get=%llu miss=%llu "
         "disk: put=%llu get=%llu evicted=%llu corrupt=%llu\n",
         g_ops.load(), g_errors.load(), (unsigned long long)st.n_stored_chunks, (unsigned long long)st.n_evicted_chunks,
         (unsigned long long)st.n_dropped_chunks, (unsigned long long)s5[0], (unsigned long long)s5[1],
         (unsigned long long)s5[2], (unsigned long long)ds.n_put, (unsigned long long)ds.n_get,
         (unsigned long long)ds.n_evicted, (unsigned long long)ds.n_corrupt);
  return g_errors.load() ? 1 : 0;
}
