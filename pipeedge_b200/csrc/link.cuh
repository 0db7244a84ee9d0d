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

}  // namespace pe

// Host-side handle. One object per END of a link; a loop-back link (both ends in one process) is one object.
struct pe_link {
  int fd = -1;               // ticket channel (Unix-domain stream socket); -1 for a host-fed link
  int fd_peer = -1;          // loop-back only: the other end of the socketpair
  int kind = 0;              // 0 = peer (cudaIpc), 1 = loop-back, 2 = host-fed
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
