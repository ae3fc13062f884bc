// b200kv_disk.cpp — local-disk chunk tier (LMCACHE_LOCAL_DISK + LMCACHE_MAX_LOCAL_DISK_SIZE,
// helm/templates/deployment-vllm-multi.yaml:334-337): the tier below the pinned host pool.
//
// CPU only.  One preallocated file per (directory, chunk size), `<dir>/b200kv-disk-<chunk bytes hex>.slots`:
//
//   [file header, 4 KiB | slot 0 | slot 1 | ...]      slot = [slot header, 4 KiB | chunk, rounded up to 4 KiB]
//
// Which key sits in which file slot, LRU and pins are kept by an index-only b200kv_pool in shm (16-byte dummy
// slots; pool slot i <-> file slot i), shared by every process that opens the same file, exactly as the device
// tier indexes HBM.  The index pool's payload area is otherwise unused: its first 16 bytes hold the UUID of the
// file it describes.  An index that is new, or whose UUID differs from the file's, is rebuilt from the slot
// headers under an exclusive flock on the file, so a restarted replica hits what it wrote before.
//
// A put writes the payload, then the slot header; a get verifies the header and the payload's XXH64 before it
// commits the pool slot, so a slot torn by a crash is caught on read (dropped from the index, counted, never
// loaded).  A rebuild trusts headers and does not scan payloads.  b200kv_disk_clear gives the file a new UUID,
// which retires every header written before it.
//
// I/O is O_DIRECT, so disk traffic does not fill the page cache of a host whose memory is the pinned pool.  The
// 4 KiB-aligned part of a pool slot moves directly between the slot and the disk; a slot that does not start on
// 4 KiB, and the tail of one whose size is not a multiple of 4 KiB, go through a per-thread aligned bounce buffer.
// A filesystem that refuses O_DIRECT gets buffered I/O with the written range flushed and dropped from the page
// cache (posix_fadvise DONTNEED).
#include <errno.h>
#include <fcntl.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <sys/file.h>
#include <sys/random.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstddef>
#include <new>
#include <string>
#include <vector>

#include "b200kv.h"

namespace {

constexpr uint64_t kBlock = 4096;
constexpr uint64_t kFileMagic = 0x46444b5630303262ull;  // "b200VKDF"
constexpr uint64_t kSlotMagic = 0x53444b5630303262ull;  // "b200VKDS"
constexpr uint32_t kDiskVersion = 1;
constexpr uint64_t kIndexSlot = 16;
constexpr uint64_t kBounce = 4ull << 20;

struct FileHeader {
  uint64_t magic;
  uint32_t version;
  uint32_t pad;
  uint64_t chunk_bytes;
  uint64_t n_slots;
  uint64_t uuid[2];
  uint64_t hash;  // XXH64 of the bytes before it
};

struct SlotHeader {
  uint64_t magic;
  uint32_t version;
  uint32_t fmt;
  uint64_t key;
  int32_t n_tokens;
  uint32_t owner;
  uint64_t payload_len;
  uint64_t payload_hash;  // XXH64 of the payload
  uint64_t stamp_ns;      // wall clock of the write: a rebuild restores LRU order from it
  uint64_t uuid[2];       // the file's UUID when the slot was written
  uint64_t hash;          // XXH64 of the bytes before it
};
static_assert(sizeof(SlotHeader) <= kBlock && sizeof(FileHeader) <= kBlock, "headers fit their block");

uint64_t round_up(uint64_t x, uint64_t a) { return (x + a - 1) / a * a; }

uint64_t mono_ns() {
  timespec ts;
  clock_gettime(CLOCK_MONOTONIC, &ts);
  return static_cast<uint64_t>(ts.tv_sec) * 1000000000ull + static_cast<uint64_t>(ts.tv_nsec);
}

uint64_t wall_ns() {
  timespec ts;
  clock_gettime(CLOCK_REALTIME, &ts);
  return static_cast<uint64_t>(ts.tv_sec) * 1000000000ull + static_cast<uint64_t>(ts.tv_nsec);
}

template <typename T>
uint64_t header_hash(const T& h) { return b200kv_xxh64(&h, offsetof(T, hash), 0); }

// Per-thread 4 KiB-aligned bounce buffer (the prefetch runs several gets in parallel).
struct Bounce {
  uint8_t* p = nullptr;
  ~Bounce() { free(p); }
  uint8_t* get() {
    if (!p && posix_memalign(reinterpret_cast<void**>(&p), kBlock, kBounce) != 0) p = nullptr;
    return p;
  }
};
thread_local Bounce t_bounce;

}  // namespace

struct b200kv_disk {
  int fd = -1;
  bool direct = true;
  int fail_errno = 0;  // B200KV_DISK_TEST_WRITE_ERRNO: every chunk write fails with this errno (tests)
  b200kv_pool* index = nullptr;
  uint64_t chunk_bytes = 0, stride = 0, n_slots = 0;
  std::string path;
  std::atomic<uint64_t> n_put{0}, n_get{0}, n_get_miss{0}, n_corrupt{0}, bytes_written{0}, bytes_read{0};
  std::atomic<uint64_t> hash_ns{0}, copy_ns{0}, io_ns{0}, n_restored{0};
  std::atomic<int> last_errno{0};

  uint64_t* shm_uuid() { return static_cast<uint64_t*>(b200kv_pool_slot_ptr(index, 0)); }
  void get_uuid(uint64_t u[2]) {
    uint64_t* s = shm_uuid();
    u[0] = __atomic_load_n(&s[0], __ATOMIC_ACQUIRE);
    u[1] = __atomic_load_n(&s[1], __ATOMIC_ACQUIRE);
  }
  void set_uuid(const uint64_t u[2]) {
    uint64_t* s = shm_uuid();
    __atomic_store_n(&s[0], u[0], __ATOMIC_RELEASE);
    __atomic_store_n(&s[1], u[1], __ATOMIC_RELEASE);
  }
  off_t slot_off(uint32_t slot) const { return static_cast<off_t>(kBlock + slot * stride); }

  // 0 or an errno.  Whole blocks only when direct.
  int pio(bool write, void* buf, uint64_t n, off_t off) {
    const uint64_t t0 = mono_ns();
    uint8_t* p = static_cast<uint8_t*>(buf);
    while (n) {
      const ssize_t k = write ? ::pwrite(fd, p, n, off) : ::pread(fd, p, n, off);
      if (k < 0) {
        if (errno == EINTR) continue;
        return errno;
      }
      if (k == 0) return EIO;  // short file
      p += k;
      n -= static_cast<uint64_t>(k);
      off += k;
    }
    io_ns += mono_ns() - t0;
    return 0;
  }

  // The chunk of `len` bytes at `mem` <-> the file at `off` (4 KiB aligned).
  int payload_io(bool write, uint8_t* mem, uint64_t len, off_t off) {
    if (!direct) {
      const int e = pio(write, mem, len, off);
      if (!e && write) sync_file_range(fd, off, static_cast<off_t>(len), SYNC_FILE_RANGE_WAIT_BEFORE |
                                       SYNC_FILE_RANGE_WRITE | SYNC_FILE_RANGE_WAIT_AFTER);
      if (!e) posix_fadvise(fd, off, static_cast<off_t>(len), POSIX_FADV_DONTNEED);
      return e;
    }
    const uint64_t body = reinterpret_cast<uintptr_t>(mem) % kBlock == 0 ? len / kBlock * kBlock : 0;
    if (body) {
      if (const int e = pio(write, mem, body, off)) return e;
    }
    uint8_t* bb = t_bounce.get();
    if (body < len && !bb) return ENOMEM;
    for (uint64_t done = body; done < len;) {
      const uint64_t piece = std::min(kBounce, len - done), whole = round_up(piece, kBlock);
      if (write) {
        const uint64_t t0 = mono_ns();
        memcpy(bb, mem + done, piece);
        memset(bb + piece, 0, whole - piece);
        copy_ns += mono_ns() - t0;
        if (const int e = pio(true, bb, whole, off + static_cast<off_t>(done))) return e;
      } else {
        if (const int e = pio(false, bb, whole, off + static_cast<off_t>(done))) return e;
        const uint64_t t0 = mono_ns();
        memcpy(mem + done, bb, piece);
        copy_ns += mono_ns() - t0;
      }
      done += piece;
    }
    return 0;
  }

  int header_io(bool write, void* hdr, uint64_t size, off_t off) {
    uint8_t* bb = t_bounce.get();
    if (!bb) return ENOMEM;
    if (write) {
      memset(bb, 0, kBlock);
      memcpy(bb, hdr, size);
      return pio(true, bb, kBlock, off);
    }
    const int e = pio(false, bb, kBlock, off);
    if (!e) memcpy(hdr, bb, size);
    return e;
  }

  uint64_t hash(const void* p, uint64_t n) {
    const uint64_t t0 = mono_ns();
    const uint64_t h = b200kv_xxh64(p, n, 0);
    hash_ns += mono_ns() - t0;
    return h;
  }

  int write_file_header(const uint64_t uuid[2]) {
    FileHeader fh;
    memset(&fh, 0, sizeof(fh));
    fh.magic = kFileMagic;
    fh.version = kDiskVersion;
    fh.chunk_bytes = chunk_bytes;
    fh.n_slots = n_slots;
    fh.uuid[0] = uuid[0];
    fh.uuid[1] = uuid[1];
    fh.hash = header_hash(fh);
    return header_io(true, &fh, sizeof(fh), 0);
  }

  // Index from the slot headers (file locked exclusively, index empty).
  void rebuild(const uint64_t uuid[2]) {
    b200kv_pool_clear(index);
    struct Entry {
      uint64_t stamp, key;
      uint32_t slot, fmt, owner;
      int32_t n_tokens;
    };
    std::vector<Entry> found;
    for (uint32_t s = 0; s < n_slots; ++s) {
      SlotHeader h;
      if (header_io(false, &h, sizeof(h), slot_off(s)) != 0) break;
      if (h.magic == 0) continue;  // never written
      if (h.magic != kSlotMagic || h.version != kDiskVersion || h.hash != header_hash(h)) {
        ++n_corrupt;  // garbage: never indexed
        continue;
      }
      if (h.uuid[0] != uuid[0] || h.uuid[1] != uuid[1]) continue;  // written before a clear
      if (h.payload_len != chunk_bytes || h.n_tokens <= 0) {
        ++n_corrupt;
        continue;
      }
      found.push_back({h.stamp_ns, h.key, s, h.fmt, h.owner, h.n_tokens});
    }
    // a key written twice (dropped as corrupt, then stored again) is the newer copy; LRU order is write order
    std::sort(found.begin(), found.end(), [](const Entry& a, const Entry& b) {
      return a.key != b.key ? a.key < b.key : a.stamp > b.stamp;
    });
    found.erase(std::unique(found.begin(), found.end(), [](const Entry& a, const Entry& b) { return a.key == b.key; }),
                found.end());
    std::sort(found.begin(), found.end(), [](const Entry& a, const Entry& b) { return a.stamp < b.stamp; });
    const size_t n = found.size();
    std::vector<uint32_t> slots(n), fmts(n), owners(n);
    std::vector<uint64_t> keys(n);
    std::vector<int32_t> toks(n);
    for (size_t i = 0; i < n; ++i) {
      slots[i] = found[i].slot;
      keys[i] = found[i].key;
      toks[i] = found[i].n_tokens;
      fmts[i] = found[i].fmt;
      owners[i] = found[i].owner;
    }
    const int placed = b200kv_pool_place(index, slots.data(), keys.data(), toks.data(), fmts.data(), owners.data(),
                                         static_cast<int32_t>(n));
    n_restored = placed > 0 ? static_cast<uint64_t>(placed) : 0;
    set_uuid(uuid);
  }
};

namespace {

int new_uuid(uint64_t u[2]) {
  if (getrandom(u, 16, 0) != 16) return errno ? errno : EIO;
  if (!u[0] && !u[1]) u[0] = 1;  // all-zero is "no index yet"
  return 0;
}

int open_index(b200kv_disk* d, const struct stat& st, bool* created) {
  char name[96];
  const uint64_t id[3] = {static_cast<uint64_t>(st.st_dev), static_cast<uint64_t>(st.st_ino), d->chunk_bytes};
  snprintf(name, sizeof(name), "/b200kv-disk-%016llx",
           static_cast<unsigned long long>(b200kv_xxh64(id, sizeof(id), 0)));
  b200kv_pool_config pc;
  memset(&pc, 0, sizeof(pc));
  pc.shm_name = name;
  pc.pool_bytes = d->n_slots * kIndexSlot;
  pc.slot_bytes = kIndexSlot;
  for (int attempt = 0; attempt < 2; ++attempt) {
    pc.flags = B200KV_POOL_CREATE;
    int rc = b200kv_pool_open(&pc, &d->index);
    *created = rc == B200KV_OK;
    if (rc == B200KV_EEXIST) {
      pc.flags = B200KV_POOL_ATTACH;
      rc = b200kv_pool_open(&pc, &d->index);
      if (rc == B200KV_OK) {
        b200kv_pool_stats ps;
        b200kv_pool_get_stats(d->index, &ps);
        if (ps.n_slots == d->n_slots) return B200KV_OK;
        b200kv_pool_close(d->index);  // an index of another incarnation of the file
        d->index = nullptr;
        rc = B200KV_EINVAL;
      }
      if (rc == B200KV_EINVAL) {
        b200kv_pool_unlink(name);
        continue;
      }
    }
    return rc;
  }
  return B200KV_EINVAL;
}

}  // namespace

extern "C" int b200kv_disk_open(const char* dir, uint64_t disk_bytes, uint64_t chunk_bytes, b200kv_disk** out) {
  if (!dir || !*dir || !out || chunk_bytes == 0) return B200KV_EINVAL;
  *out = nullptr;
  const uint64_t stride = kBlock + round_up(chunk_bytes, kBlock);
  const uint64_t n_slots = disk_bytes > kBlock ? (disk_bytes - kBlock) / stride : 0;
  if (n_slots == 0 || n_slots > 0x7fffffffu) return B200KV_EINVAL;
  struct stat ds;
  if (stat(dir, &ds) != 0) return -errno;
  if (!S_ISDIR(ds.st_mode)) return -ENOTDIR;

  b200kv_disk* d = new (std::nothrow) b200kv_disk();
  if (!d) return B200KV_ENOMEM;
  d->chunk_bytes = chunk_bytes;
  d->stride = stride;
  d->n_slots = n_slots;
  char fname[64];
  snprintf(fname, sizeof(fname), "/b200kv-disk-%llx.slots", static_cast<unsigned long long>(chunk_bytes));
  d->path = std::string(dir) + fname;
  if (const char* e = getenv("B200KV_DISK_TEST_WRITE_ERRNO")) d->fail_errno = atoi(e);

  d->fd = ::open(d->path.c_str(), O_RDWR | O_CREAT | O_CLOEXEC | O_DIRECT, 0644);
  if (d->fd < 0 && errno == EINVAL) {  // the filesystem refuses O_DIRECT
    d->direct = false;
    d->fd = ::open(d->path.c_str(), O_RDWR | O_CREAT | O_CLOEXEC, 0644);
  }
  if (d->fd < 0) {
    const int e = errno;
    delete d;
    return -e;
  }
  flock(d->fd, LOCK_EX);  // one opener at a time sizes the file and (re)builds the index
  int rc = B200KV_OK;
  uint64_t uuid[2] = {0, 0};
  FileHeader fh;
  memset(&fh, 0, sizeof(fh));
  struct stat fs;
  if (fstat(d->fd, &fs) != 0) {
    rc = -errno;
  } else if (static_cast<uint64_t>(fs.st_size) >= kBlock && d->header_io(false, &fh, sizeof(fh), 0) == 0 &&
             fh.magic == kFileMagic && fh.version == kDiskVersion && fh.hash == header_hash(fh) &&
             fh.chunk_bytes == chunk_bytes && fh.n_slots > 0 && fh.n_slots <= 0x7fffffffu &&
             static_cast<uint64_t>(fs.st_size) >= kBlock + fh.n_slots * stride) {
    d->n_slots = fh.n_slots;  // an existing file keeps the size it was created with
    uuid[0] = fh.uuid[0];
    uuid[1] = fh.uuid[1];
  } else if (int e = new_uuid(uuid)) {
    rc = -e;
  } else if (int e = ftruncate(d->fd, 0) != 0 ? errno : posix_fallocate(d->fd, 0, static_cast<off_t>(kBlock + n_slots * stride))) {
    rc = (e == EFBIG || e == ENOSPC) ? B200KV_ENOSPC : -e;
    if (ftruncate(d->fd, 0) != 0) { /* best effort: give the space back */ }
  } else if (int e2 = d->write_file_header(uuid)) {
    rc = e2 == ENOSPC ? B200KV_ENOSPC : -e2;
  }
  bool created = false;
  if (rc == B200KV_OK) rc = open_index(d, fs, &created);
  if (rc == B200KV_OK) {
    uint64_t have[2];
    d->get_uuid(have);
    if (created || have[0] != uuid[0] || have[1] != uuid[1]) d->rebuild(uuid);
  }
  flock(d->fd, LOCK_UN);
  if (rc != B200KV_OK) {
    b200kv_disk_close(d);
    return rc;
  }
  *out = d;
  return B200KV_OK;
}

extern "C" int b200kv_disk_close(b200kv_disk* d) {
  if (!d) return B200KV_EINVAL;
  if (d->fd >= 0) ::close(d->fd);
  if (d->index) b200kv_pool_close(d->index);
  delete d;
  return B200KV_OK;
}

extern "C" int b200kv_disk_put(b200kv_disk* d, b200kv_pool* local, uint64_t key, uint32_t owner) {
  if (!d || !local) return B200KV_EINVAL;
  b200kv_pool_stats ls;
  if (b200kv_pool_get_stats(local, &ls) != B200KV_OK || ls.slot_bytes != d->chunk_bytes) return B200KV_EINVAL;
  uint32_t lslot = 0, fmt = 0, dslot = 0;
  int32_t n_tok = 0;
  int rc = b200kv_pool_acquire(local, key, &lslot, &n_tok, &fmt);
  if (rc != B200KV_OK) return rc;
  rc = b200kv_pool_reserve(d->index, key, n_tok, fmt, owner, &dslot);
  if (rc != B200KV_OK) {
    b200kv_pool_release(local, key);
    return rc;
  }
  uint8_t* mem = static_cast<uint8_t*>(b200kv_pool_slot_ptr(local, lslot));
  SlotHeader h;
  memset(&h, 0, sizeof(h));
  h.magic = kSlotMagic;
  h.version = kDiskVersion;
  h.fmt = fmt;
  h.key = key;
  h.n_tokens = n_tok;
  h.owner = owner;
  h.payload_len = d->chunk_bytes;
  h.payload_hash = d->hash(mem, d->chunk_bytes);
  h.stamp_ns = wall_ns();
  d->get_uuid(h.uuid);
  h.hash = header_hash(h);
  const off_t off = d->slot_off(dslot);
  int e = d->fail_errno ? d->fail_errno : d->payload_io(true, mem, d->chunk_bytes, off + static_cast<off_t>(kBlock));
  if (!e) e = d->header_io(true, &h, sizeof(h), off);  // payload first, then header
  b200kv_pool_release(local, key);
  if (e) {
    b200kv_pool_abort(d->index, key);
    d->last_errno = e;
    return B200KV_EIO;
  }
  ++d->n_put;
  d->bytes_written += d->chunk_bytes;
  return b200kv_pool_commit(d->index, key);
}

extern "C" int b200kv_disk_get(b200kv_disk* d, b200kv_pool* local, uint64_t key) {
  if (!d || !local) return B200KV_EINVAL;
  b200kv_pool_stats ls;
  if (b200kv_pool_get_stats(local, &ls) != B200KV_OK || ls.slot_bytes != d->chunk_bytes) return B200KV_EINVAL;
  uint32_t dslot = 0, fmt = 0, lslot = 0;
  int32_t n_tok = 0;
  if (b200kv_pool_acquire(d->index, key, &dslot, &n_tok, &fmt) != B200KV_OK) {  // pinned: not evictable now
    ++d->n_get_miss;
    return B200KV_ENOENT;
  }
  const off_t off = d->slot_off(dslot);
  SlotHeader h;
  int e = d->header_io(false, &h, sizeof(h), off);
  if (e) {
    b200kv_pool_release(d->index, key);
    d->last_errno = e;
    return B200KV_EIO;
  }
  bool bad = h.magic != kSlotMagic || h.version != kDiskVersion || h.hash != header_hash(h) || h.key != key ||
             h.n_tokens != n_tok || h.fmt != fmt || h.payload_len != d->chunk_bytes;
  int rc = B200KV_OK;
  if (!bad) {
    rc = b200kv_pool_reserve(local, key, n_tok, fmt, h.owner, &lslot);
    if (rc != B200KV_OK) {
      b200kv_pool_release(d->index, key);
      return rc == B200KV_EEXIST ? B200KV_OK : rc;
    }
    uint8_t* mem = static_cast<uint8_t*>(b200kv_pool_slot_ptr(local, lslot));
    e = d->payload_io(false, mem, d->chunk_bytes, off + static_cast<off_t>(kBlock));
    if (e) {
      b200kv_pool_abort(local, key);
      b200kv_pool_release(d->index, key);
      d->last_errno = e;
      return B200KV_EIO;
    }
    bad = d->hash(mem, d->chunk_bytes) != h.payload_hash;
    if (bad) b200kv_pool_abort(local, key);
  }
  if (bad) {  // torn or overwritten slot: never loaded, gone from the index, and its header retired (still pinned)
    ++d->n_corrupt;
    SlotHeader zero;
    memset(&zero, 0, sizeof(zero));
    if (d->header_io(true, &zero, sizeof(zero), off) != 0) { /* a restart finds it again and drops it again */ }
    b200kv_pool_release(d->index, key);
    b200kv_pool_drop(d->index, key);
    return B200KV_ENOENT;
  }
  b200kv_pool_release(d->index, key);
  ++d->n_get;
  d->bytes_read += d->chunk_bytes;
  return b200kv_pool_commit(local, key);
}

extern "C" int b200kv_disk_lookup(b200kv_disk* d, const uint64_t* keys, int32_t n_keys, int32_t* n_prefix) {
  if (!d || !n_prefix) return B200KV_EINVAL;
  return b200kv_pool_lookup_owner(d->index, keys, n_keys, n_prefix, nullptr);
}

extern "C" int b200kv_disk_get_stats(b200kv_disk* d, b200kv_disk_stats* out) {
  if (!d || !out) return B200KV_EINVAL;
  b200kv_pool_stats ps;
  const int rc = b200kv_pool_get_stats(d->index, &ps);
  if (rc != B200KV_OK) return rc;
  memset(out, 0, sizeof(*out));
  out->n_slots = ps.n_slots;
  out->n_used = ps.n_used;
  out->slot_bytes = d->stride;
  out->n_put = d->n_put;
  out->n_get = d->n_get;
  out->n_get_miss = d->n_get_miss;
  out->n_corrupt = d->n_corrupt;
  out->n_evicted = ps.n_evicted_chunks;
  out->n_dropped = ps.n_dropped_chunks;
  out->bytes_written = d->bytes_written;
  out->bytes_read = d->bytes_read;
  out->hash_ns = d->hash_ns;
  out->copy_ns = d->copy_ns;
  out->io_ns = d->io_ns;
  out->n_restored = d->n_restored;
  out->direct_io = d->direct ? 1 : 0;
  out->last_errno = d->last_errno;
  return B200KV_OK;
}

extern "C" int b200kv_disk_clear(b200kv_disk* d) {
  if (!d) return B200KV_EINVAL;
  uint64_t uuid[2];
  if (int e = new_uuid(uuid)) return -e;
  flock(d->fd, LOCK_EX);
  const int rc = b200kv_pool_clear(d->index);
  const int e = d->write_file_header(uuid);  // retires every slot header written so far
  if (!e) d->set_uuid(uuid);
  flock(d->fd, LOCK_UN);
  if (e) {
    d->last_errno = e;
    return B200KV_EIO;
  }
  return rc;
}
