// Rings in POSIX shared memory between a data rank without a GPU and the stages it feeds and collects from.
//
// A data rank outside the stage pipeline only loads micro-batches, sends them and receives the logits. Without a GPU it
// cannot own a peer link's ring (device memory, cudaIpc), so each of its two hops gets a ring in a shared-memory segment
// the data rank creates (shm_open + mmap): the slot layout of a peer link ([16 KiB header | payload], link.cuh) and its
// monotonic counters, full[s] and free[s], both in the segment (HostRing). Slot s carries payloads s, s + R, ...; the
// k-th use is published when full[s] == k + 1 and may be overwritten once free[s] == k + 1. The segment's name comes
// from the caller (MASTER_PORT and the hop's ranks, so that concurrent jobs stay apart); it is unlinked as soon as both
// ends have mapped it, or the handshake failed, so that a job that dies later leaves nothing in /dev/shm.
//
// The host end (pe_hostring_*, this file) never touches the CUDA runtime: it reads and writes the segment with acquire /
// release atomics and sends one ticket per payload on the hop's socket, as a peer link does. The stage's end is a
// pe_link of kind 3 (pe_link_open, link.cu): the segment registered with CUDA, results stored into it by the last
// stage's send kernel (zero-copy over PCIe), inputs copied out of it by the first stage's copy engine.
#include <errno.h>
#include <fcntl.h>
#include <math.h>
#include <poll.h>
#include <sched.h>
#include <stdlib.h>
#include <string.h>
#include <sys/mman.h>
#include <sys/socket.h>
#include <sys/stat.h>
#include <time.h>
#include <unistd.h>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"
#include "link.cuh"

namespace pe {

unsigned long long link_timeout_ns() {
  const char* e = getenv("PIPEEDGE_LINK_TIMEOUT_S");
  double s = e != nullptr ? atof(e) : 30.0;
  if (s < 0.01) s = 0.01;
  return static_cast<unsigned long long>(s * 1e9);
}

static unsigned long long now_ns() {
  struct timespec t;
  clock_gettime(CLOCK_MONOTONIC, &t);
  return static_cast<unsigned long long>(t.tv_sec) * 1000000000ull + static_cast<unsigned long long>(t.tv_nsec);
}

static size_t roundup4k(size_t x) { return (x + 4095) / 4096 * 4096; }

int hostring_map(const char* name, bool create, int n_slots, size_t slot_bytes, HostRing* r) {
  const size_t bytes = kShmCtlBytes + slot_bytes * static_cast<size_t>(n_slots);
  int fd = -1;
  if (create) {
    fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
    if (fd < 0 && errno == EEXIST) {
      // left by a job with the same port and ranks that died during its handshake: that job cannot still be running,
      // because a live one holds the port
      shm_unlink(name);
      fd = shm_open(name, O_CREAT | O_EXCL | O_RDWR, 0600);
    }
  } else {
    fd = shm_open(name, O_RDWR, 0);
  }
  if (fd < 0) {
    set_error("host ring: shm_open(%s): %s", name, strerror(errno));
    return PE_ERR_INVALID;
  }
  if (create && ftruncate(fd, static_cast<off_t>(bytes)) != 0) {   // zero-filled: every counter starts at 0
    set_error("host ring: ftruncate(%s, %zu): %s", name, bytes, strerror(errno));
    close(fd);
    shm_unlink(name);
    return PE_ERR_NOMEM;
  }
  if (!create) {
    struct stat st;
    if (fstat(fd, &st) != 0 || static_cast<size_t>(st.st_size) != bytes) {
      set_error("host ring: segment %s is not the %zu bytes its geometry names", name, bytes);
      close(fd);
      return PE_ERR_INVALID;
    }
  }
  void* p = mmap(nullptr, bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0);
  close(fd);
  if (p == MAP_FAILED) {
    set_error("host ring: mmap(%s, %zu): %s", name, bytes, strerror(errno));
    if (create) shm_unlink(name);
    return PE_ERR_NOMEM;
  }
  r->base = static_cast<uint8_t*>(p);
  r->map_bytes = bytes;
  r->slot_bytes = slot_bytes;
  r->n_slots = n_slots;
  r->seq = 0;
  r->timeout_ns = link_timeout_ns();
  return PE_OK;
}

void hostring_unmap(HostRing* r) {
  if (r->base != nullptr) munmap(r->base, r->map_bytes);
  r->base = nullptr;
  r->map_bytes = 0;
}

// Bounded: a dead or stalled peer ends in an error after the link timeout, never in a hang. Yields first (the flag is
// usually raised within microseconds of the ticket), then sleeps 50 us between polls.
static int wait_ge(const HostRing* r, const uint64_t* flag, uint64_t want, const char* what) {
  if (__atomic_load_n(flag, __ATOMIC_ACQUIRE) >= want) return PE_OK;
  const unsigned long long t0 = now_ns();
  unsigned spins = 0;
  while (__atomic_load_n(flag, __ATOMIC_ACQUIRE) < want) {
    if (++spins < 2000) {
      sched_yield();
    } else {
      const struct timespec pause = {0, 50000};
      nanosleep(&pause, nullptr);
    }
    if ((spins & 15) == 0 && now_ns() - t0 > r->timeout_ns) {
      set_error("host ring: %s within the link timeout (PIPEEDGE_LINK_TIMEOUT_S)", what);
      return PE_ERR_CUDA;
    }
  }
  return PE_OK;
}

int hostring_read(HostRing* r, int items, size_t bytes, const void** data) {
  const uint64_t n = static_cast<uint64_t>(r->n_slots);
  const uint64_t slot = r->seq % n, k = r->seq / n;
  int rc = wait_ge(r, r->full() + slot, k + 1, "the producer did not publish the announced payload");
  if (rc != PE_OK) return rc;
  LinkHeader h;
  memcpy(&h, r->slot(r->seq), sizeof(h));
  // the bytes the header describes: a raw payload names them; one raw f32 tensor (a last stage's results) has
  // items x n values
  size_t described = SIZE_MAX;
  if (h.n_tensors == kLinkRawKind && h.t[0].dtype == kLinkDtypeBytes) described = h.t[0].n;
  else if (h.n_tensors == 1 && h.t[0].bit == 0 && h.t[0].dtype == 0) described = static_cast<size_t>(h.items) * h.t[0].n * 4;
  if (h.magic != kLinkMagic || h.items != static_cast<uint32_t>(items) || described != bytes ||
      h.t[0].data_off != kLinkHeaderBytes || kLinkHeaderBytes + bytes > r->slot_bytes) {
    set_error("host ring: payload mismatch: magic %x kind %u items %u, %zu bytes (expected %d items, %zu bytes)", h.magic,
              h.n_tensors, h.items, described, items, bytes);
    return PE_ERR_INVALID;
  }
  *data = r->slot(r->seq) + kLinkHeaderBytes;
  return PE_OK;
}

int read_within(int fd, void* buf, size_t n, unsigned long long timeout_ns, const char* what) {
  char* p = static_cast<char*>(buf);
  const unsigned long long t0 = now_ns();
  while (n > 0) {
    const unsigned long long waited = now_ns() - t0;
    if (waited >= timeout_ns) {
      set_error("host ring: %s did not arrive within the link timeout (PIPEEDGE_LINK_TIMEOUT_S)", what);
      return PE_ERR_CUDA;
    }
    struct pollfd pfd = {fd, POLLIN, 0};
    const int ms = static_cast<int>((timeout_ns - waited + 999999) / 1000000);
    const int pr = poll(&pfd, 1, ms);
    if (pr < 0 && errno == EINTR) continue;
    if (pr < 0) {
      set_error("host ring: poll while waiting for %s: %s", what, strerror(errno));
      return PE_ERR_CUDA;
    }
    if (pr == 0) continue;
    const ssize_t got = recv(fd, p, n, 0);
    if (got == 0) {
      set_error("host ring: the peer closed the hop before %s", what);
      return PE_ERR_CUDA;
    }
    if (got < 0) {
      if (errno == EINTR) continue;
      set_error("host ring: socket read while waiting for %s: %s", what, strerror(errno));
      return PE_ERR_CUDA;
    }
    p += got;
    n -= static_cast<size_t>(got);
  }
  return PE_OK;
}

static void name_to_handle(const char* name, cudaIpcMemHandle_t* handle) {
  memset(handle, 0, sizeof(*handle));
  memcpy(handle, name, strlen(name));
}

}  // namespace pe

struct pe_hostring {
  int fd = -1;
  bool is_producer = false;
  pe::HostRing ring;
};

extern "C" {

// Data rank: create the segment of one hop and hand it to the stage at the other end of `fd` (see link.cuh: HelloMsg).
int pe_hostring_create(int fd, const char* name, int is_producer, size_t slot_payload_bytes, int n_slots,
                       pe_hostring** out) {
  using namespace pe;
  PE_REQUIRE(out != nullptr && fd >= 0 && name != nullptr && name[0] == '/' && strchr(name + 1, '/') == nullptr &&
                 strlen(name) < sizeof(cudaIpcMemHandle_t),
             "pe_hostring_create: bad arguments (the name is '/' and at most %zu more characters, no other '/')",
             sizeof(cudaIpcMemHandle_t) - 2);
  const unsigned long long timeout = link_timeout_ns();
  pe_hostring* r = new pe_hostring();
  r->fd = fd;
  r->is_producer = is_producer != 0;
  int rc = PE_OK;
  if (is_producer) {
    HelloMsg hello = {};
    if (n_slots < 2 || n_slots > kLinkMaxSlots || slot_payload_bytes == 0) {
      set_error("pe_hostring_create: n_slots=%d outside [2,%d] or empty slots", n_slots, kLinkMaxSlots);
      rc = PE_ERR_INVALID;
    } else {
      rc = hostring_map(name, true, n_slots, roundup4k(kLinkHeaderBytes + slot_payload_bytes), &r->ring);
    }
    hello.magic = rc == PE_OK ? kShmMagic : 0u;   // 0: tell the peer we failed, so that it does not block
    hello.n_slots = static_cast<uint32_t>(n_slots);
    hello.slot_bytes = r->ring.slot_bytes;
    name_to_handle(name, &hello.handle);
    const int w = write_all(fd, &hello, sizeof(hello));
    if (rc == PE_OK) {
      ReplyMsg reply = {};
      rc = w != 0 ? PE_ERR_CUDA : read_within(fd, &reply, sizeof(reply), timeout, "the consumer's reply");
      shm_unlink(name);   // both ends have mapped it, or the handshake failed
      if (w != 0) set_error("pe_hostring_create: socket write failed: %s", strerror(errno));
      else if (rc == PE_OK && (reply.magic != kShmMagic || reply.status != 0)) {
        set_error("pe_hostring_create: the consumer could not map the ring");
        rc = PE_ERR_CUDA;
      }
    }
  } else {
    HelloMsg hello = {};
    rc = read_within(fd, &hello, sizeof(hello), timeout, "the producer's hello");
    ReplyMsg reply = {};
    if (rc == PE_OK) {
      if (hello.magic != kLinkMagic || hello.n_slots < 2 || hello.n_slots > static_cast<uint32_t>(kLinkMaxSlots) ||
          hello.slot_bytes <= kLinkHeaderBytes || hello.slot_bytes % 4096 != 0) {
        set_error("pe_hostring_create: malformed hello from the producer");
        rc = PE_ERR_CUDA;
      } else {
        rc = hostring_map(name, true, static_cast<int>(hello.n_slots), hello.slot_bytes, &r->ring);
      }
      reply.magic = rc == PE_OK ? kShmMagic : 0u;
      reply.status = rc == PE_OK ? 0u : 1u;
      name_to_handle(name, &reply.handle);
      const int w = write_all(fd, &reply, sizeof(reply));
      if (rc == PE_OK) {
        ReplyMsg ack = {};
        rc = w != 0 ? PE_ERR_CUDA : read_within(fd, &ack, sizeof(ack), timeout, "the producer's acknowledgement");
        shm_unlink(name);
        if (w != 0) set_error("pe_hostring_create: socket write failed: %s", strerror(errno));
        else if (rc == PE_OK && (ack.magic != kShmMagic || ack.status != 0)) {
          set_error("pe_hostring_create: the producer could not map the ring");
          rc = PE_ERR_CUDA;
        }
      }
    }
  }
  if (rc != PE_OK) {
    hostring_unmap(&r->ring);
    delete r;
    return rc;
  }
  *out = r;
  return PE_OK;
}

// The other end of pe_hostring_create without a GPU: what a stage's pe_link_open does for such a hop, less the CUDA
// registration.
int pe_hostring_attach(int fd, int is_producer, size_t slot_payload_bytes, int n_slots, pe_hostring** out) {
  using namespace pe;
  PE_REQUIRE(out != nullptr && fd >= 0, "pe_hostring_attach: bad arguments");
  PE_REQUIRE(!is_producer || (n_slots >= 2 && n_slots <= kLinkMaxSlots && slot_payload_bytes > 0),
             "pe_hostring_attach: n_slots=%d outside [2,%d] or empty slots", n_slots, kLinkMaxSlots);
  const unsigned long long timeout = link_timeout_ns();
  pe_hostring* r = new pe_hostring();
  r->fd = fd;
  r->is_producer = is_producer != 0;
  int rc = PE_OK;
  if (is_producer) {
    HelloMsg hello = {};
    hello.magic = kLinkMagic;
    hello.n_slots = static_cast<uint32_t>(n_slots);
    hello.slot_bytes = roundup4k(kLinkHeaderBytes + slot_payload_bytes);
    ReplyMsg reply = {};
    if (write_all(fd, &hello, sizeof(hello)) != 0) {
      set_error("pe_hostring_attach: socket write failed: %s", strerror(errno));
      rc = PE_ERR_CUDA;
    }
    if (rc == PE_OK) rc = read_within(fd, &reply, sizeof(reply), timeout, "the consumer's reply");
    if (rc == PE_OK && (reply.magic != kShmMagic || reply.status != 0)) {
      set_error("pe_hostring_attach: the consumer did not offer a shared-memory ring");
      rc = PE_ERR_CUDA;
    }
    if (rc == PE_OK) {
      reply.handle.reserved[sizeof(reply.handle) - 1] = 0;
      rc = hostring_map(reply.handle.reserved, false, n_slots, hello.slot_bytes, &r->ring);
      ReplyMsg ack = {kShmMagic, rc == PE_OK ? 0u : 1u, {}};
      if (write_all(fd, &ack, sizeof(ack)) != 0 && rc == PE_OK) {
        set_error("pe_hostring_attach: socket write failed: %s", strerror(errno));
        rc = PE_ERR_CUDA;
      }
    }
  } else {
    HelloMsg hello = {};
    rc = read_within(fd, &hello, sizeof(hello), timeout, "the producer's hello");
    if (rc == PE_OK && (hello.magic != kShmMagic || hello.n_slots < 2 ||
                        hello.n_slots > static_cast<uint32_t>(kLinkMaxSlots))) {
      set_error("pe_hostring_attach: the producer did not offer a shared-memory ring");
      rc = PE_ERR_CUDA;
    }
    if (rc == PE_OK) {
      hello.handle.reserved[sizeof(hello.handle) - 1] = 0;
      rc = hostring_map(hello.handle.reserved, false, static_cast<int>(hello.n_slots), hello.slot_bytes, &r->ring);
      ReplyMsg reply = {kShmMagic, rc == PE_OK ? 0u : 1u, {}};
      if (write_all(fd, &reply, sizeof(reply)) != 0 && rc == PE_OK) {
        set_error("pe_hostring_attach: socket write failed: %s", strerror(errno));
        rc = PE_ERR_CUDA;
      }
    }
  }
  if (rc != PE_OK) {
    hostring_unmap(&r->ring);
    delete r;
    return rc;
  }
  *out = r;
  return PE_OK;
}

int pe_hostring_close(pe_hostring* r) {
  if (r == nullptr) return PE_OK;
  pe::hostring_unmap(&r->ring);
  delete r;
  return PE_OK;
}

size_t pe_hostring_slot_bytes(const pe_hostring* r) {
  return r == nullptr ? 0 : r->ring.slot_bytes - pe::kLinkHeaderBytes;
}

// Producer: wait (bounded) until the next slot is free, write a raw header and the payload, publish the slot (release
// store of full[s]) and send its ticket {items, dim1}. A payload larger than a slot is refused before anything is
// written.
int pe_hostring_publish(pe_hostring* r, const void* data, size_t bytes, int items, long long dim1) {
  using namespace pe;
  PE_REQUIRE(r != nullptr && r->is_producer && data != nullptr && bytes > 0 && items > 0 && items <= kLinkMaxItems,
             "pe_hostring_publish: bad arguments");
  PE_REQUIRE(kLinkHeaderBytes + bytes <= r->ring.slot_bytes, "pe_hostring_publish: %zu bytes exceed the ring's %zu-byte slots",
             bytes, r->ring.slot_bytes - kLinkHeaderBytes);
  HostRing& g = r->ring;
  const uint64_t n = static_cast<uint64_t>(g.n_slots);
  const uint64_t slot = g.seq % n, k = g.seq / n;
  int rc = wait_ge(&g, g.free_() + slot, k, "the consumer did not release a slot");
  if (rc != PE_OK) return rc;
  LinkHeader h = {};
  h.magic = kLinkMagic;
  h.n_tensors = kLinkRawKind;
  h.items = static_cast<uint32_t>(items);
  h.t[0].dtype = kLinkDtypeBytes;
  h.t[0].n = bytes;
  h.t[0].data_off = kLinkHeaderBytes;
  h.t[0].alpha = INFINITY;
  uint8_t* base = g.slot(g.seq);
  memcpy(base, &h, sizeof(h));
  memcpy(base + kLinkHeaderBytes, data, bytes);
  __atomic_store_n(g.full() + slot, k + 1, __ATOMIC_RELEASE);
  ++g.seq;
  const long long ticket[2] = {items, dim1};
  PE_REQUIRE(write_all(r->fd, ticket, sizeof(ticket)) == 0, "pe_hostring_publish: ticket write failed: %s", strerror(errno));
  return PE_OK;
}

// Producer: no more payloads (the closing ticket).
int pe_hostring_close_input(pe_hostring* r) {
  PE_REQUIRE(r != nullptr && r->is_producer, "pe_hostring_close_input: not the producer end of a host ring");
  const long long ticket[2] = {-1, 0};
  PE_REQUIRE(pe::write_all(r->fd, ticket, sizeof(ticket)) == 0, "pe_hostring_close_input: ticket write failed: %s",
             strerror(errno));
  return PE_OK;
}

// Consumer: the next ticket {items, dim1 or elements per item}; blocks until it arrives. 1: the producer closed.
int pe_hostring_next(pe_hostring* r, long long* ticket2) {
  using namespace pe;
  PE_REQUIRE(r != nullptr && !r->is_producer && ticket2 != nullptr, "pe_hostring_next: bad arguments");
  const int got = read_all(r->fd, ticket2, 2 * sizeof(long long));
  if (got == 1 || (got == 0 && ticket2[0] < 0)) return 1;
  PE_REQUIRE(got == 0, "pe_hostring_next: socket read failed: %s", strerror(errno));
  return PE_OK;
}

// Consumer: wait (bounded) for the payload the last ticket announced; its header must name `items` and `bytes`.
// *data stays valid until pe_hostring_release.
int pe_hostring_wait(pe_hostring* r, int items, size_t bytes, const void** data) {
  PE_REQUIRE(r != nullptr && !r->is_producer && data != nullptr, "pe_hostring_wait: bad arguments");
  return pe::hostring_read(&r->ring, items, bytes, data);
}

// Consumer: hand the slot back to the producer (release store of free[s]).
int pe_hostring_release(pe_hostring* r) {
  PE_REQUIRE(r != nullptr && !r->is_producer, "pe_hostring_release: not the consumer end of a host ring");
  pe::HostRing& g = r->ring;
  const uint64_t n = static_cast<uint64_t>(g.n_slots);
  __atomic_store_n(g.free_() + g.seq % n, g.seq / n + 1, __ATOMIC_RELEASE);
  ++g.seq;
  return PE_OK;
}

}  // extern "C"
