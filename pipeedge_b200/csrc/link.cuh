// Peer-memory links between pipeline stages: shared declarations of link.cu (rings, flags, put / get kernels) and
// pipe.cu (the per-rank stage loop built on them).
#pragma once
#include <stddef.h>
#include <stdint.h>

#include "common.cuh"

namespace pe {

constexpr int kLinkMaxSlots = 8;
constexpr int kLinkMaxItems = 512;                 // items (micro-batch size) a slot header has scale / shift room for
constexpr size_t kLinkHeaderBytes = 16384;         // slot = [header | payload]; payload starts here
constexpr size_t kLinkScaleOff = 256;              // + tensor * 4096: scale f32 [kLinkMaxItems], then shift f32 [kLinkMaxItems]
constexpr uint32_t kLinkMagic = 0x4b4c4550u;       // "PELK"

// error codes a kernel leaves in the link's host-mapped status word before it traps
enum : unsigned {
  kLinkErrNone = 0,
  kLinkErrWaitFull = 1,    // consumer: the producer never raised the slot's full flag
  kLinkErrWaitFree = 2,    // producer: the consumer never released the slot
  kLinkErrHeader = 3,      // consumer: payload description does not match what the stage expects
  kLinkErrBarrier = 4,     // fused quantise-and-send: grid barrier timed out
};

struct LinkTensorHdr {     // 32 bytes
  uint32_t bit;            // 0 = raw values, else QuantPipe bit-width
  uint32_t dtype;          // raw values: 0 = f32, 1 = f16
  uint64_t n;              // elements per item
  uint64_t data_off;       // byte offset of the tensor's data from the slot base
  float alpha;             // clamp threshold used (+inf when none)
  uint32_t pad;
};
struct LinkHeader {        // first bytes of every slot that carries activations
  uint32_t magic;
  uint32_t n_tensors;
  uint32_t items;
  uint32_t pad;
  LinkTensorHdr t[2];
};
// A raw payload (the data rank's input micro-batch relayed to the first stage, link_relay): n_tensors = kLinkRawKind,
// t[0].n = bytes, t[0].dtype = kLinkDtypeBytes, bit 0, the bytes at kLinkHeaderBytes, unconverted.
constexpr uint32_t kLinkRawKind = 0;
constexpr uint32_t kLinkDtypeBytes = 2;

// Receiver-side view of a link (what a get kernel dereferences). All flags are monotonic counters: slot s is used for
// payloads s, s + R, s + 2R, ...; its k-th use is complete when full[s] == k + 1 and may be overwritten when
// free[s] == k + 1.
struct LinkRx {
  uint8_t* ring;           // this device
  size_t slot_bytes;
  int n_slots;
  const uint64_t* full;    // this device; raised by the producer (peer store over NVLink, or a host-enqueued copy)
  uint64_t* free_;         // producer-visible: peer device memory (cudaIpc) or mapped host memory (host-fed link)
  uint64_t* seq;           // this device: payloads consumed so far
  unsigned* done_ctr;      // this device: CTAs of the running get kernel that have finished reading
  unsigned* status;        // mapped host memory
};
struct LinkTx {
  uint8_t* ring;           // the consumer's device (peer mapping)
  size_t slot_bytes;
  int n_slots;
  uint64_t* full;          // the consumer's device
  const uint64_t* free_;   // this device; advanced by the consumer
  uint64_t* seq;           // this device: payloads produced so far
  unsigned* done_ctr;      // this device
  unsigned* bar_count;     // this device: grid barrier of the fused quantise-and-send kernel
  unsigned* bar_gen;
  double* partials;        // this device: per-(item, chunk) statistics
  unsigned* status;        // mapped host memory
};

struct PutTensor {
  const float* a;          // [items, n] f32
  const float* b;          // nullable: the payload is a + b (a stage that ends on a projection defers its residual add)
  size_t n;                // elements per item
};

// The open handshake on a hop's socket. The producer writes a HelloMsg, the consumer answers with a ReplyMsg. A hop to or
// from a data rank without a GPU carries kShmMagic instead: the data rank has created the ring in POSIX shared memory and
// names it in `handle` (a NUL-terminated shm_open name). Data rank -> first stage: its HelloMsg carries the name, the
// stage maps the segment and replies. Last stage -> data rank: the data rank answers the stage's HelloMsg with the name,
// the stage maps the segment and acknowledges with a ReplyMsg of its own. magic 0 / status != 0: the sender failed.
constexpr uint32_t kShmMagic = 0x4853454bu;        // "KESH"
struct HelloMsg {
  uint32_t magic;
  uint32_t n_slots;
  uint32_t quant_hint;         // the bit-width the producer expects to send (sizes the consumer's receive grid)
  uint32_t pad;
  uint64_t slot_bytes;
  cudaIpcMemHandle_t handle;   // the producer's block (free flags), or the shared-memory segment's name
};
struct ReplyMsg {
  uint32_t magic;
  uint32_t status;             // 0 ok
  cudaIpcMemHandle_t handle;   // the consumer's block (full flags + ring), or the shared-memory segment's name
};

// A ring in POSIX shared memory between a data rank without a GPU and a stage (hostring.cu): the slot layout and the
// monotonic full / free counters of a peer link, both counters in the segment. The host end reads and writes it
// directly with acquire / release atomics; the stage's end registers it with CUDA (mapped, portable), so that link_put
// stores results into it and a copy engine reads inputs out of it.
constexpr size_t kShmCtlBytes = 4096;              // segment = [full u64[R] @0, free u64[R] @kShmFreeOff | R slots]
constexpr size_t kShmFreeOff = 2048;
struct HostRing {
  uint8_t* base = nullptr;     // host mapping
  size_t map_bytes = 0;
  size_t slot_bytes = 0;       // header included, a multiple of 4096
  int n_slots = 0;
  uint64_t seq = 0;            // payloads published (producer) / released (consumer) so far
  unsigned long long timeout_ns = 0;
  uint64_t* full() const { return reinterpret_cast<uint64_t*>(base); }
  uint64_t* free_() const { return reinterpret_cast<uint64_t*>(base + kShmFreeOff); }
  uint8_t* slot(uint64_t s) const { return base + kShmCtlBytes + (s % static_cast<uint64_t>(n_slots)) * slot_bytes; }
};

unsigned long long link_timeout_ns();   // PIPEEDGE_LINK_TIMEOUT_S (default 30 s)
// Map the segment `name` of R slots of `slot_bytes` (create: a new one, zeroed; else an existing one of that size).
int hostring_map(const char* name, bool create, int n_slots, size_t slot_bytes, HostRing* r);
void hostring_unmap(HostRing* r);
// Consumer: wait (bounded) for the next payload's full flag, check its header against `items` and `bytes`, *data = the
// payload. The slot stays owned until it is released.
int hostring_read(HostRing* r, int items, size_t bytes, const void** data);
// Read exactly n bytes within the link timeout: 0 ok, else an error is set.
int read_within(int fd, void* buf, size_t n, unsigned long long timeout_ns, const char* what);

}  // namespace pe

// Host-side handle. One object per END of a link; a loop-back link (both ends in one process) is one object.
struct pe_link {
  int fd = -1;               // ticket channel (Unix-domain stream socket); -1 for a host-fed link
  int fd_peer = -1;          // loop-back only: the other end of the socketpair
  int kind = 0;              // 0 = peer (cudaIpc), 1 = loop-back, 2 = host-fed, 3 = shared memory with a host data rank
  bool is_tx = false, is_rx = false;
  size_t slot_bytes = 0;
  int n_slots = 0;
  pe::LinkRx rx = {};
  pe::LinkTx tx = {};
  void* local_block = nullptr;     // cudaMalloc'ed by this end
  void* peer_block = nullptr;      // cudaIpcOpenMemHandle'd
  void* ctl_block = nullptr;       // this end's private counters (seq, done_ctr, barrier, partials)
  unsigned* status_host = nullptr; // cudaHostAlloc mapped
  uint64_t* host_flags = nullptr;  // host-fed: mapped [free x R | staged full values x R]
  uint64_t fed = 0;                // host-fed: payloads fed so far
  float* add_scratch = nullptr;    // generic-bit-width path: a + b materialised here
  size_t add_scratch_bytes = 0;
  void* quant_work = nullptr;
  size_t quant_work_bytes = 0;
  unsigned long long timeout_ns = 0;
  int wire_f16 = 0;
  int quant_hint = 0;              // bit-width the producer announced at open (0 = raw payloads)
  pe::HostRing shm;                // kind 3: the segment's host mapping (registered with CUDA)
  bool shm_registered = false;
  uint64_t* shm_free_dev = nullptr;   // kind 3 consumer: device alias of the segment's free flags
};

namespace pe {

// What a pipeline with timestamps (pipe.cu) asks of link_put: a launch between a staged put's stand-alone encode kernels
// and its shipping kernel, and a description of what the put wrote.
struct PutStamp {
  int (*encoded)(void* ctx, cudaStream_t stream) = nullptr;   // after the encode kernels of the last staged tensor
  void* ctx = nullptr;
  size_t bytes = 0;   // out: payload bytes written (see link_payload_bytes), summed over the tensors
  int paths = 0;      // out: OR of 1 << PE_LINK_PATH_* over the tensors
};

// Bytes a put of one [items, n] tensor at `bit` bits writes: the values (f32, or f16 with wire_f16), or the packed codes
// plus the per-item scale and shift. Equal to what the Python-thread path moves for the same tensor when wire_f16 == 0.
size_t link_payload_bytes(int items, size_t n, int bit, int wire_f16);

int link_put(pe_link* link, const PutTensor* t, int n_tensors, int items, int bit, int clamp, cudaStream_t stream,
             PutStamp* stamp = nullptr);
// prewait: park in the one-warp wait kernel first (consumers that may wait long while other streams compute)
int link_get(pe_link* link, void* dst0, void* dst1, int items, size_t n0, size_t n1, int n_tensors, cudaStream_t stream,
             bool prewait);
// items == 0: headerless (a host-fed link); items > 0: a raw payload relayed from a peer (link_relay) whose header must
// name `bytes` and `items`
int link_get_raw(pe_link* link, void* dst, size_t bytes, int items, cudaStream_t stream, bool prewait);
// Data rank outside the stage pipeline: the next host-fed payload of `in` (`bytes`, `items`) -> the peer ring of `out`
int link_relay(pe_link* in, pe_link* out, int items, size_t bytes, cudaStream_t stream);
int link_feed(pe_link* link, const void* src, size_t bytes, int src_is_host, cudaStream_t copy_stream);
int link_ticket_send(pe_link* link, long long a, long long b);
int link_ticket_recv(pe_link* link, long long* out2);   // 0 ok, 1 = peer closed
int link_check(pe_link* link);                          // PE_OK or the protocol error a kernel reported

}  // namespace pe
