// Inter-stage hop, native fast path: one C call per payload on each side (no Python in the steady state).
//
// A hop is a directed pair (sender rank -> receiver rank) on one node. Control data travels over the hop's
// Unix-domain socket (opened by the Python layer, `pipeedge_b200/comm/p2p`), device tensors over a dedicated
// 2-rank NCCL communicator (NVLink / NVSwitch P2P) on the caller's side stream:
//   sender  : write the 16-byte "same layout as before" envelope, wait for the producer's event on the hop
//             stream, ncclSend every device tensor in one group, record the "sent" event;
//   receiver: (the blocking read of the envelope is done by pe_hop_wait_envelope with the GIL released)
//             wait for the "consumer done" events of the destination buffers, ncclRecv in one group, record
//             the "ready" event the compute stream will wait on.
// NCCL is resolved at run time from the libnccl.so.2 the process already has loaded (PyTorch's), so the library
// itself carries no link-time NCCL dependency.
// Replaces TensorSendThread.run / TensorRecvThread.run + _send_tensor / _recv_tensor (p2p/__init__.py:96-258).
#include <dlfcn.h>
#include <mutex>
#include <errno.h>
#include <string.h>
#include <sys/socket.h>
#include <unistd.h>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"

namespace pe {

int require_sm90();

// minimal NCCL surface (ABI-stable since NCCL 2.x)
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { kNcclUint8 = 1 };   // ncclUint8 / ncclChar8

struct NcclApi {
  ncclResult_t (*GetUniqueId)(ncclUniqueId*);
  ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
  ncclResult_t (*CommDestroy)(ncclComm_t);
  ncclResult_t (*Send)(const void*, size_t, int, int, ncclComm_t, cudaStream_t);
  ncclResult_t (*Recv)(void*, size_t, int, int, ncclComm_t, cudaStream_t);
  ncclResult_t (*GroupStart)();
  ncclResult_t (*GroupEnd)();
  const char* (*GetErrorString)(ncclResult_t);
  bool ok = false;
};

static NcclApi load_nccl() {
  NcclApi api;
  void* h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (h == nullptr) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (h != nullptr) {
    api.GetUniqueId = reinterpret_cast<decltype(api.GetUniqueId)>(dlsym(h, "ncclGetUniqueId"));
    api.CommInitRank = reinterpret_cast<decltype(api.CommInitRank)>(dlsym(h, "ncclCommInitRank"));
    api.CommDestroy = reinterpret_cast<decltype(api.CommDestroy)>(dlsym(h, "ncclCommDestroy"));
    api.Send = reinterpret_cast<decltype(api.Send)>(dlsym(h, "ncclSend"));
    api.Recv = reinterpret_cast<decltype(api.Recv)>(dlsym(h, "ncclRecv"));
    api.GroupStart = reinterpret_cast<decltype(api.GroupStart)>(dlsym(h, "ncclGroupStart"));
    api.GroupEnd = reinterpret_cast<decltype(api.GroupEnd)>(dlsym(h, "ncclGroupEnd"));
    api.GetErrorString = reinterpret_cast<decltype(api.GetErrorString)>(dlsym(h, "ncclGetErrorString"));
    api.ok = api.GetUniqueId && api.CommInitRank && api.CommDestroy && api.Send && api.Recv && api.GroupStart &&
             api.GroupEnd && api.GetErrorString;
  }
  return api;
}

// function-local static: initialised exactly once even when the send and the receive thread race to the first call
static NcclApi& nccl() {
  static NcclApi api = load_nccl();
  return api;
}

// Communicator creation / destruction touch process-wide NCCL state (proxy service, shared resources): the send and
// receive threads of a stage close their hops at about the same time, so those calls are serialised per process.
static std::mutex& comm_lifecycle_mutex() {
  static std::mutex m;
  return m;
}

int write_all(int fd, const void* buf, size_t n) {
  const char* p = static_cast<const char*>(buf);
  while (n > 0) {
    const ssize_t w = send(fd, p, n, MSG_NOSIGNAL);
    if (w < 0) {
      if (errno == EINTR) continue;
      return -1;
    }
    p += w;
    n -= static_cast<size_t>(w);
  }
  return 0;
}

int read_all(int fd, void* buf, size_t n) {
  char* p = static_cast<char*>(buf);
  while (n > 0) {
    const ssize_t r = recv(fd, p, n, 0);
    if (r == 0) return 1;   // EOF
    if (r < 0) {
      if (errno == EINTR) continue;
      return -1;
    }
    p += r;
    n -= static_cast<size_t>(r);
  }
  return 0;
}

}  // namespace pe

struct pe_hop {
  int fd;
  int is_sender;
  pe::ncclComm_t comm;
};

#define PE_NCCL(call)                                                                      \
  do {                                                                                     \
    const pe::ncclResult_t _r = (call);                                                    \
    if (_r != 0) {                                                                         \
      pe::set_error("NCCL error %d (%s) in %s", _r, pe::nccl().GetErrorString(_r), #call); \
      return PE_ERR_CUDA;                                                                  \
    }                                                                                      \
  } while (0)

extern "C" {

int pe_hop_available(void) { return pe::nccl().ok ? 1 : 0; }

// Both ends call this once (it blocks until the peer has joined): the sender creates the NCCL id and ships it over
// the socket. `fd` stays owned by the caller.
int pe_hop_open(int fd, int is_sender, pe_hop** out) {
  using namespace pe;
  PE_REQUIRE(out != nullptr && fd >= 0, "pe_hop_open: bad arguments");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;
  NcclApi& api = nccl();
  PE_REQUIRE(api.ok, "pe_hop_open: libnccl.so.2 is not loadable in this process");
  ncclUniqueId id;
  if (is_sender) {
    PE_NCCL(api.GetUniqueId(&id));
    PE_REQUIRE(write_all(fd, &id, sizeof(id)) == 0, "pe_hop_open: socket write failed: %s", strerror(errno));
  } else {
    PE_REQUIRE(read_all(fd, &id, sizeof(id)) == 0, "pe_hop_open: socket read failed");
  }
  pe_hop* hop = new pe_hop();
  hop->fd = fd;
  hop->is_sender = is_sender;
  hop->comm = nullptr;
  ncclResult_t r;
  {
    // hops are opened one at a time per process, in the same global order on every rank (p2p/__init__.py), so holding
    // the lock across the blocking rendezvous cannot deadlock
    std::lock_guard<std::mutex> lock(comm_lifecycle_mutex());
    r = api.CommInitRank(&hop->comm, 2, id, is_sender ? 0 : 1);
  }
  if (r != 0) {
    set_error("ncclCommInitRank failed: %s", api.GetErrorString(r));
    delete hop;
    return PE_ERR_CUDA;
  }
  *out = hop;
  return PE_OK;
}

int pe_hop_close(pe_hop* hop) {
  if (hop == nullptr) return PE_OK;
  if (hop->comm != nullptr) {
    std::lock_guard<std::mutex> lock(pe::comm_lifecycle_mutex());
    pe::nccl().CommDestroy(hop->comm);
  }
  delete hop;
  return PE_OK;
}

// Sender, steady state. ptrs/bytes: the payload's device tensors in order. `ready_event` (may be NULL): recorded by the
// producer when the tensors are written; `done_event` (may be NULL): recorded here once the sends are enqueued behind
// everything on `stream`. If `write_envelope` the 16-byte (0, -1) header is written first.
int pe_hop_send(pe_hop* hop, const void* const* ptrs, const size_t* bytes, int n, void* ready_event, void* stream_v,
                void* done_event, int write_envelope) {
  using namespace pe;
  PE_REQUIRE(hop != nullptr && hop->is_sender && n >= 0, "pe_hop_send: bad arguments");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if (write_envelope) {
    const long long head[2] = {0, -1};
    PE_REQUIRE(write_all(hop->fd, head, sizeof(head)) == 0, "pe_hop_send: socket write failed: %s", strerror(errno));
  }
  if (ready_event != nullptr) PE_CUDA(cudaStreamWaitEvent(stream, static_cast<cudaEvent_t>(ready_event), 0));
  NcclApi& api = nccl();
  if (n > 1) PE_NCCL(api.GroupStart());
  for (int i = 0; i < n; ++i) PE_NCCL(api.Send(ptrs[i], bytes[i], kNcclUint8, 1, hop->comm, stream));
  if (n > 1) PE_NCCL(api.GroupEnd());
  if (done_event != nullptr) PE_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(done_event), stream));
  return PE_OK;
}

// Receiver: block (callers release the GIL) until the next 16-byte envelope header arrives. Returns 1 on EOF.
int pe_hop_wait_envelope(pe_hop* hop, long long* head2) {
  using namespace pe;
  PE_REQUIRE(hop != nullptr && head2 != nullptr, "pe_hop_wait_envelope: bad arguments");
  const int r = read_all(hop->fd, head2, 2 * sizeof(long long));
  if (r == 1) return 1;
  PE_REQUIRE(r == 0, "pe_hop_wait_envelope: socket read failed: %s", strerror(errno));
  return PE_OK;
}

// Receiver: free_events[i] (may be NULL) guards buffer i against its previous consumer; `ready_event` is recorded
// after the receives.
int pe_hop_recv(pe_hop* hop, void* const* ptrs, const size_t* bytes, void* const* free_events, int n, void* stream_v,
                void* ready_event) {
  using namespace pe;
  PE_REQUIRE(hop != nullptr && !hop->is_sender && n >= 0, "pe_hop_recv: bad arguments");
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  for (int i = 0; i < n; ++i)
    if (free_events != nullptr && free_events[i] != nullptr)
      PE_CUDA(cudaStreamWaitEvent(stream, static_cast<cudaEvent_t>(free_events[i]), 0));
  NcclApi& api = nccl();
  if (n > 1) PE_NCCL(api.GroupStart());
  for (int i = 0; i < n; ++i) PE_NCCL(api.Recv(ptrs[i], bytes[i], kNcclUint8, 0, hop->comm, stream));
  if (n > 1) PE_NCCL(api.GroupEnd());
  if (ready_event != nullptr) PE_CUDA(cudaEventRecord(static_cast<cudaEvent_t>(ready_event), stream));
  return PE_OK;
}

}  // extern "C"
