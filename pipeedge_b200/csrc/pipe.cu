// Per-rank pipeline stage loop: one CUDA graph per micro-batch, no Python and no GIL in the steady state.
//
// A stage's whole micro-batch - link get (wait for the upstream payload, copy / dequantise it into the stage's fixed
// input buffer) -> embeddings / encoder blocks / head kernels -> link put (quantise-and-send into the downstream ring) -
// is captured ONCE per (micro-batch size, sequence length, send bit-width) into a CUDA graph: the link kernels find
// their ring slot through device-resident sequence counters (link.cu), so the graph takes no per-payload arguments and
// the first replay is already the steady state. The host side of a stage is this loop:
//     read a 16-byte ticket from the upstream hop's socket (blocks) -> cudaGraphLaunch -> write the ticket downstream
// i.e. two system calls and one launch per micro-batch; ordering against the neighbours' GPUs is entirely on the
// devices (flags in peer memory). The data rank feeds its first stage through a host-fed link (pe_pipe_submit: H2D /
// D2D copy on a side stream + graph launch) and drains results through pe_pipe_next_result. A data rank outside the
// stage pipeline does the same with a graph of one relay kernel (pe_pipe_capture_relay) that forwards the fed input to
// the first stage, whose graph then starts with a raw receive from its peer link.
//
// Replaces TensorWorkThread.run + the queue hand-offs of DistP2pPipelineStage (p2p/__init__.py:261-295,373-394,442-450):
// FIFO per hop (tickets and flags are strictly ordered), back-pressure through the rings (a producer blocks - on the
// device - until the consumer has released the slot; enqueue blocks on the host-fed ring).
#include <limits.h>
#include <string.h>

#include <atomic>
#include <map>
#include <mutex>
#include <tuple>
#include <utility>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"
#include "link.cuh"

namespace pe {
void count_launches(int n);
uint64_t launch_count_now();
int require_sm90();
constexpr int kPipeWindow = 8;   // graph launches the host may run ahead of the device
static_assert(PE_PIPE_STAMP_DEPTH > kPipeWindow, "a record must outlive the launches the host may run ahead");

// One record of the timestamp ring (mapped host memory). `seq` is written last: index + 1 once the record is complete,
// 0 while its first stamp has started to overwrite it.
struct StampSlot {
  unsigned long long seq;
  pe_pipe_record rec;
};
}  // namespace pe

struct pe_pipe {
  pe_link* in = nullptr;
  pe_link* out = nullptr;
  pe_link* res = nullptr;
  cudaStream_t compute = nullptr, copy = nullptr, results = nullptr, put = nullptr;
  // Overlapped send (capture_end with overlap != 0): the stage writes its output into one of TWO buffer sets (parity =
  // micro-batch index mod 2); the link's send kernel runs as its own graph on the `put` stream and overlaps the next
  // micro-batch's receive / first kernels; events order main(i) -> put(i) -> main(i + 2).
  struct Graph {
    cudaGraphExec_t exec[2] = {nullptr, nullptr};       // get + stage kernels (+ put when not overlapped), per parity
    cudaGraphExec_t exec_put[2] = {nullptr, nullptr};   // the send on its own stream (overlapped mode)
    int n_par = 0;                                      // parities captured so far
    int want_par = 1;                                   // 1 (send inside the main graph) or 2 (overlapped)
    int kernels = 0;
    bool stamps = false;                                // captured with timestamp kernels
  };
  cudaEvent_t ev_main_done[2] = {nullptr, nullptr}, ev_put_done[2] = {nullptr, nullptr};
  bool put_pending[2] = {false, false};
  int cap_parity = 0;
  // (micro-batch size, dim1, send bit-width) -> graph. A stage whose bit-width changes between micro-batches keeps one
  // graph per bit-width and picks one per launch (send_bit); the kernels and graphs of each variant are those of a
  // fixed-bit stage at that bit-width.
  std::map<std::tuple<int, long long, int>, Graph> graphs;
  std::map<std::pair<int, long long>, int> latest_bit;   // bit-width of each shape's most recent capture
  std::atomic<int> send_bit{-1};   // pe_pipe_set_send_bit; -1: the shape's most recent capture, whatever its bit-width
  std::mutex graphs_mu;    // prepare() on the owner thread may insert while the stage thread looks a graph up
  bool capturing = false;
  int cap_ubatch = 0;
  long long cap_dim1 = 0;
  uint64_t cap_launch0 = 0;
  cudaEvent_t window[pe::kPipeWindow] = {};
  uint64_t launched = 0;
  // device-side timing of the current phase
  cudaEvent_t ev_first = nullptr, ev_last = nullptr, ev_res_last = nullptr;
  std::atomic<int> timing_reset{1};
  bool have_first = false, have_res = false;
  uint64_t timed_launches = 0, timed_kernels = 0;
  // results (data rank)
  void* res_dev = nullptr;
  void* res_host = nullptr;
  size_t res_cap = 0;
  // a ticket read by pe_pipe_run for which no graph exists yet
  bool pending = false;
  long long pend[2] = {0, 0};
  long long out_dim = 0;   // > 0: outgoing tickets carry it instead of the incoming dim (last stage: result elements per item)
  // per-micro-batch timestamps (pe_pipe_enable_stamps)
  std::atomic<bool> stamps_on{false};
  bool cap_stamps = false;                  // the capture in progress carries stamp kernels
  pe::StampSlot* stamp_host = nullptr;      // the ring, PE_PIPE_STAMP_DEPTH records (cudaHostAllocMapped)
  pe::StampSlot* stamp_dev = nullptr;       // ... its device alias
  unsigned long long* stamp_ctr = nullptr;  // device: next record of the main graph [0] and of the send graph [1]
  unsigned long long stamp_next = 0;        // drain: the next record to read
};

namespace pe {

// `bit`: the send bit-width of the variant (-1: the shape's most recent capture). `current`: the graph must also have been
// captured with the stamps setting now in force (a graph captured the other way counts as missing, so the next payload
// of its shape captures again)
static bool find_graph(pe_pipe* p, int ubatch, long long dim1, int bit, pe_pipe::Graph* out, bool current = true) {
  std::lock_guard<std::mutex> lock(p->graphs_mu);
  if (bit < 0) {
    auto lb = p->latest_bit.find(std::make_pair(ubatch, dim1));
    if (lb == p->latest_bit.end()) return false;
    bit = lb->second;
  }
  auto it = p->graphs.find(std::make_tuple(ubatch, dim1, bit));
  if (it == p->graphs.end() || it->second.n_par < it->second.want_par) return false;   // every parity captured?
  if (current && it->second.stamps != p->stamps_on.load()) return false;
  if (out != nullptr) *out = it->second;
  return true;
}

// ------------------------------------------------------------------------------------------------ timestamps
// Which fields a stamp writes. A micro-batch's record gets, in order: Start (graph start, before the receive), Got
// (receive done), Stage (the stage's last kernel done), SendStart, Encoded (staged sends only), SendEnd. With the send
// inside the main graph, Stage and SendStart are one stamp; with an overlapped send, the send graph's stamps find the
// record through their own counter, because send(i) runs while main(i + 1) already stamps record i + 1.
enum : int {
  kStampStart = 1, kStampGot = 2, kStampStage = 4, kStampSendStart = 8, kStampEncoded = 16, kStampSendEnd = 32,
};

struct StampArgs {
  StampSlot* ring;                // device alias of the mapped host ring
  unsigned long long* ctr;        // device counters: [0] main graph, [1] send graph
  int ctr_idx;                    // the counter that names this stamp's record
  int what;                       // kStamp* fields
  int bump;                       // bit i: advance ctr[i] past this record
  // kStampGot on a peer link: the receive's ring, whose slot header holds the payload's bit-width
  const uint8_t* in_ring;
  size_t in_slot_bytes;
  int in_slots;
  const uint64_t* in_seq;
  // kStampSendEnd: the record's remaining fields
  int items, bit_out, flags;
  unsigned long long bytes_out;
};

// One thread: %globaltimer into the micro-batch's record. Launched WITHOUT programmatic dependent launch, so it starts
// only after the kernel before it has completed; the PDL-launched stage kernel after it waits (griddepcontrol.wait) for
// the stamp's completion, which is ordered after everything before the stamp.
__global__ void __launch_bounds__(1) pipe_stamp_kernel(const StampArgs a) {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  const unsigned long long r = *reinterpret_cast<volatile unsigned long long*>(a.ctr + a.ctr_idx);
  StampSlot* s = a.ring + r % PE_PIPE_STAMP_DEPTH;
  volatile pe_pipe_record* rec = &s->rec;
  if (a.what & kStampStart) {
    *reinterpret_cast<volatile unsigned long long*>(&s->seq) = 0;   // a reader copying the old record sees it changed
    __threadfence_system();
    rec->t_start = t;
    rec->t_encoded = 0;
  }
  if (a.what & kStampGot) {
    rec->t_got = t;
    int bit = -1;
    if (a.in_ring != nullptr) {
      // The slot of the payload just consumed. Its producer may already be rewriting that slot for a payload a whole
      // ring later; the header's bit-width then changes only if the producer's own bit-width did in between.
      const uint64_t seq = *reinterpret_cast<const volatile uint64_t*>(a.in_seq) - 1;
      const LinkHeader* h = reinterpret_cast<const LinkHeader*>(a.in_ring + (seq % static_cast<uint64_t>(a.in_slots)) * a.in_slot_bytes);
      bit = static_cast<int>(*reinterpret_cast<const volatile uint32_t*>(&h->t[0].bit));
    }
    rec->bit_in = bit;
  }
  if (a.what & kStampStage) rec->t_stage = t;
  if (a.what & kStampSendStart) rec->t_send_start = t;
  if (a.what & kStampEncoded) rec->t_encoded = t;
  if (a.what & kStampSendEnd) {
    rec->t_send_end = t;
    rec->index = r;
    rec->items = a.items;
    rec->bit_out = a.bit_out;
    rec->flags = a.flags;
    rec->bytes_out = a.bytes_out;
    __threadfence_system();   // every field of the record (earlier stamps fenced theirs) before the publication
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(&s->seq), "l"(r + 1) : "memory");
  } else {
    __threadfence_system();
  }
  if (a.bump & 1) a.ctr[0] = r + 1;
  if (a.bump & 2) a.ctr[1] = r + 1;
}

static int launch_stamp(pe_pipe* p, StampArgs a, cudaStream_t stream) {
  a.ring = p->stamp_dev;
  a.ctr = p->stamp_ctr;
  pipe_stamp_kernel<<<1, 1, 0, stream>>>(a);
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  return PE_OK;
}

struct EncodedStamp {   // link_put's callback context on a staged send
  pe_pipe* p;
  int ctr_idx;
};

static int stamp_encoded(void* ctx, cudaStream_t stream) {
  const EncodedStamp* e = static_cast<const EncodedStamp*>(ctx);
  StampArgs a = {};
  a.ctr_idx = e->ctr_idx;
  a.what = kStampEncoded;
  return launch_stamp(e->p, a, stream);
}

// The send of a capture with stamps: [SendStart] put [Encoded inside a staged put] SendEnd (publishes the record).
static int put_stamped(pe_pipe* p, const PutTensor* t, int n_tensors, int items, int bit, int clamp, int overlap,
                       cudaStream_t stream) {
  const int ctr_idx = overlap != 0 ? 1 : 0;
  StampArgs a = {};
  a.ctr_idx = ctr_idx;
  if (overlap != 0) {
    a.what = kStampSendStart;
    const int rc = launch_stamp(p, a, stream);
    if (rc != PE_OK) return rc;
  }
  EncodedStamp ctx = {p, ctr_idx};
  PutStamp ps;
  ps.encoded = stamp_encoded;
  ps.ctx = &ctx;
  const int rc = link_put(p->out, t, n_tensors, items, bit, clamp, stream, &ps);
  if (rc != PE_OK) return rc;
  a.what = kStampSendEnd;
  a.bump = overlap != 0 ? 2 : 3;
  a.items = items;
  a.bit_out = bit;
  a.flags = (overlap != 0 ? PE_STAMP_OVERLAPPED : 0) | ((ps.paths & (1 << PE_LINK_PATH_FUSED)) ? PE_STAMP_FUSED : 0) |
            ((ps.paths & (1 << PE_LINK_PATH_STAGED)) ? PE_STAMP_STAGED : 0);
  a.bytes_out = ps.bytes;
  return launch_stamp(p, a, stream);
}

static void destroy_graph(pe_pipe::Graph& g) {
  for (int i = 0; i < 2; ++i) {
    if (g.exec[i] != nullptr) cudaGraphExecDestroy(g.exec[i]);
    if (g.exec_put[i] != nullptr) cudaGraphExecDestroy(g.exec_put[i]);
    g.exec[i] = g.exec_put[i] = nullptr;
  }
  g.n_par = 0;
}

// File a captured graph (one parity of it) under (ubatch, dim1, bit).
static void file_graph(pe_pipe* p, int ubatch, long long dim1, int bit, int par, cudaGraphExec_t exec_main,
                       cudaGraphExec_t exec_put, int want_par, int kernels, bool stamps) {
  std::lock_guard<std::mutex> lock(p->graphs_mu);
  pe_pipe::Graph& g = p->graphs[std::make_tuple(ubatch, dim1, bit)];
  if (par == 0) {   // a fresh capture of this key starts with parity 0
    destroy_graph(g);
    p->latest_bit[std::make_pair(ubatch, dim1)] = bit;
    if (p->send_bit.load() < 0) {
      // no bit-width selected: the capture replaces the shape's graph, whatever bit-width that one sent with
      for (auto it = p->graphs.lower_bound(std::make_tuple(ubatch, dim1, INT_MIN));
           it != p->graphs.end() && std::get<0>(it->first) == ubatch && std::get<1>(it->first) == dim1;) {
        if (std::get<2>(it->first) == bit) {
          ++it;
          continue;
        }
        destroy_graph(it->second);
        it = p->graphs.erase(it);
      }
    }
  }
  g.want_par = want_par;
  g.exec[par] = exec_main;
  g.exec_put[par] = exec_put;
  g.n_par = par + 1;
  g.kernels = kernels;
  g.stamps = stamps;
}

static int launch_graph(pe_pipe* p, int ubatch, long long dim1, int bit) {
  pe_pipe::Graph g;
  PE_REQUIRE(find_graph(p, ubatch, dim1, bit, &g, false),
             "pipe: no graph captured for micro-batch size %d / dim %lld / send bit-width %d", ubatch, dim1, bit);
  const int w = static_cast<int>(p->launched % kPipeWindow);
  if (p->launched >= static_cast<uint64_t>(kPipeWindow)) PE_CUDA(cudaEventSynchronize(p->window[w]));
  if (p->timing_reset.exchange(0) != 0) {
    PE_CUDA(cudaEventRecord(p->ev_first, p->compute));
    p->have_first = true;
    p->have_res = false;
    p->timed_launches = 0;
    p->timed_kernels = 0;
  }
  if (g.want_par == 2) {
    const int par = static_cast<int>(p->launched & 1);
    if (p->put_pending[par]) PE_CUDA(cudaStreamWaitEvent(p->compute, p->ev_put_done[par], 0));   // its buffers are free again
    PE_CUDA(cudaGraphLaunch(g.exec[par], p->compute));
    PE_CUDA(cudaEventRecord(p->ev_main_done[par], p->compute));
    PE_CUDA(cudaStreamWaitEvent(p->put, p->ev_main_done[par], 0));
    PE_CUDA(cudaGraphLaunch(g.exec_put[par], p->put));
    PE_CUDA(cudaEventRecord(p->ev_put_done[par], p->put));
    p->put_pending[par] = true;
    PE_CUDA(cudaEventRecord(p->ev_last, p->put));
    PE_CUDA(cudaEventRecord(p->window[w], p->put));
  } else {
    // a previous overlapped micro-batch may still be sending out of the buffers this graph writes
    for (int par = 0; par < 2; ++par)
      if (p->put_pending[par]) {
        PE_CUDA(cudaStreamWaitEvent(p->compute, p->ev_put_done[par], 0));
        p->put_pending[par] = false;
      }
    PE_CUDA(cudaGraphLaunch(g.exec[0], p->compute));
    PE_CUDA(cudaEventRecord(p->ev_last, p->compute));
    PE_CUDA(cudaEventRecord(p->window[w], p->compute));
  }
  ++p->launched;
  ++p->timed_launches;
  p->timed_kernels += static_cast<uint64_t>(g.kernels);
  count_launches(g.kernels);
  int rc = link_check(p->in);
  if (rc == PE_OK) rc = link_check(p->out);
  return rc;
}

}  // namespace pe

extern "C" {

// `in`: host-fed link (data rank) or the consumer end of the upstream hop; `out`: producer end of the downstream hop
// (or of a loop-back link on a one-rank pipeline); `res`: data rank only - the consumer end results arrive on (the hop
// from the last stage, or the same loop-back link). Links stay owned by the caller and must outlive the pipe.
int pe_pipe_create(pe_link* in, pe_link* out, pe_link* res, pe_pipe** out_pipe) {
  using namespace pe;
  PE_REQUIRE(out_pipe != nullptr && in != nullptr && out != nullptr, "pe_pipe_create: null link");
  PE_REQUIRE(in->is_rx && out->is_tx && (res == nullptr || res->is_rx), "pe_pipe_create: link ends do not match their roles");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;
  pe_pipe* p = new pe_pipe();
  p->in = in;
  p->out = out;
  p->res = res;
  cudaError_t e = cudaStreamCreateWithFlags(&p->compute, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->copy, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->results, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&p->put, cudaStreamNonBlocking);
  for (int i = 0; i < 2 && e == cudaSuccess; ++i) {
    e = cudaEventCreateWithFlags(&p->ev_main_done[i], cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventCreateWithFlags(&p->ev_put_done[i], cudaEventDisableTiming);
  }
  for (int i = 0; i < kPipeWindow && e == cudaSuccess; ++i) e = cudaEventCreateWithFlags(&p->window[i], cudaEventDisableTiming);
  if (e == cudaSuccess) e = cudaEventCreate(&p->ev_first);
  if (e == cudaSuccess) e = cudaEventCreate(&p->ev_last);
  if (e == cudaSuccess) e = cudaEventCreate(&p->ev_res_last);
  if (e == cudaSuccess && res != nullptr) {
    p->res_cap = res->slot_bytes;
    e = cudaMalloc(&p->res_dev, p->res_cap);
    if (e == cudaSuccess) e = cudaHostAlloc(&p->res_host, p->res_cap, cudaHostAllocDefault);
  }
  if (e != cudaSuccess) {
    check_cuda(e, "pe_pipe_create");
    pe_pipe_destroy(p);
    return PE_ERR_CUDA;
  }
  *out_pipe = p;
  return PE_OK;
}

int pe_pipe_destroy(pe_pipe* p) {
  if (p == nullptr) return PE_OK;
  if (p->compute != nullptr) cudaStreamSynchronize(p->compute);
  if (p->put != nullptr) cudaStreamSynchronize(p->put);
  if (p->results != nullptr) cudaStreamSynchronize(p->results);
  if (p->copy != nullptr) cudaStreamSynchronize(p->copy);
  for (auto& kv : p->graphs) pe::destroy_graph(kv.second);
  for (int i = 0; i < 2; ++i) {
    if (p->ev_main_done[i] != nullptr) cudaEventDestroy(p->ev_main_done[i]);
    if (p->ev_put_done[i] != nullptr) cudaEventDestroy(p->ev_put_done[i]);
  }
  if (p->put != nullptr) cudaStreamDestroy(p->put);
  for (int i = 0; i < pe::kPipeWindow; ++i)
    if (p->window[i] != nullptr) cudaEventDestroy(p->window[i]);
  if (p->ev_first != nullptr) cudaEventDestroy(p->ev_first);
  if (p->ev_last != nullptr) cudaEventDestroy(p->ev_last);
  if (p->ev_res_last != nullptr) cudaEventDestroy(p->ev_res_last);
  if (p->res_dev != nullptr) cudaFree(p->res_dev);
  if (p->res_host != nullptr) cudaFreeHost(p->res_host);
  if (p->stamp_host != nullptr) cudaFreeHost(p->stamp_host);
  if (p->stamp_ctr != nullptr) cudaFree(p->stamp_ctr);
  if (p->compute != nullptr) cudaStreamDestroy(p->compute);
  if (p->copy != nullptr) cudaStreamDestroy(p->copy);
  if (p->results != nullptr) cudaStreamDestroy(p->results);
  cudaGetLastError();
  delete p;
  return PE_OK;
}

// The stream the stage's kernels must be enqueued on between capture_begin and capture_end (a cudaStream_t).
void* pe_pipe_stream(pe_pipe* p) { return p == nullptr ? nullptr : p->compute; }
void* pe_pipe_copy_stream(pe_pipe* p) { return p == nullptr ? nullptr : p->copy; }

// For the send bit-width now in force (pe_pipe_set_send_bit).
int pe_pipe_has_graph(pe_pipe* p, int ubatch, long long dim1) {
  return (p != nullptr && pe::find_graph(p, ubatch, dim1, p->send_bit.load(), nullptr)) ? 1 : 0;
}

// For one send bit-width, whichever is in force (-1: the shape's most recent capture).
int pe_pipe_has_variant(pe_pipe* p, int ubatch, long long dim1, int bit) {
  return (p != nullptr && pe::find_graph(p, ubatch, dim1, bit, nullptr)) ? 1 : 0;
}

// The send bit-width whose graphs launch from the next launch on (-1, the initial value: each shape's most recent
// capture). An atomic store: legal while another thread sits in pe_pipe_run or pe_pipe_submit, which read it once per
// micro-batch. A bit-width without a graph for a payload's shape makes pe_pipe_run ask for a capture (and
// pe_pipe_submit fail) rather than launch another variant.
int pe_pipe_set_send_bit(pe_pipe* p, int bit) {
  PE_REQUIRE(p != nullptr && bit >= -1 && bit <= 16, "pe_pipe_set_send_bit: bit=%d outside [-1,16]", bit);
  p->send_bit.store(bit);
  return PE_OK;
}

// Start capturing the graph for micro-batches of `ubatch` items (`dim1`: sequence length, part of the key). The get
// kernel is enqueued first: from a host-fed link `raw_bytes` bytes land in dst0; from a hop the payload's one or two
// tensors ([ubatch, n0] / [ubatch, n1] f32 after decoding) land in dst0 / dst1, or, with raw_bytes > 0 (the first stage
// fed by a data rank outside the stage pipeline, pe_pipe_capture_relay), the relayed input's `raw_bytes` bytes.
int pe_pipe_capture_begin(pe_pipe* p, int ubatch, long long dim1, int parity, void* dst0, void* dst1, size_t n0, size_t n1,
                          size_t raw_bytes) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && !p->capturing && ubatch > 0 && (parity == 0 || parity == 1),
             "pe_pipe_capture_begin: bad state / arguments");
  PE_CUDA(cudaStreamSynchronize(p->compute));
  PE_CUDA(cudaStreamSynchronize(p->put));
  p->cap_parity = parity;
  p->cap_stamps = p->stamps_on.load();
  if (parity == 1) {   // parity 1 follows its graph's parity 0 (the shape's latest capture): both replay the same kernels
    std::lock_guard<std::mutex> lock(p->graphs_mu);
    auto lb = p->latest_bit.find(std::make_pair(ubatch, dim1));
    auto it = lb == p->latest_bit.end() ? p->graphs.end() : p->graphs.find(std::make_tuple(ubatch, dim1, lb->second));
    if (it != p->graphs.end() && it->second.n_par == 1) p->cap_stamps = it->second.stamps;
  }
  PE_CUDA(cudaStreamBeginCapture(p->compute, cudaStreamCaptureModeRelaxed));
  p->capturing = true;
  p->cap_ubatch = ubatch;
  p->cap_dim1 = dim1;
  p->cap_launch0 = launch_count_now();
  StampArgs st = {};
  st.what = kStampStart;
  int rc = p->cap_stamps ? launch_stamp(p, st, p->compute) : PE_OK;
  if (rc == PE_OK) {
    if (p->in->kind == 2) rc = link_get_raw(p->in, dst0, raw_bytes, 0, p->compute, false);
    else if (raw_bytes > 0) rc = link_get_raw(p->in, dst0, raw_bytes, ubatch, p->compute, false);   // from a relay
    else rc = link_get(p->in, dst0, dst1, ubatch, n0, n1, dst1 != nullptr ? 2 : 1, p->compute, false);
  }
  if (rc == PE_OK && p->cap_stamps) {
    st.what = kStampGot;
    if (p->in->kind != 2 && raw_bytes == 0) {   // a raw input was not quantised: bit_in stays -1
      st.in_ring = p->in->rx.ring;
      st.in_slot_bytes = p->in->rx.slot_bytes;
      st.in_slots = p->in->rx.n_slots;
      st.in_seq = p->in->rx.seq;
    }
    rc = launch_stamp(p, st, p->compute);
  }
  if (rc != PE_OK) pe_pipe_capture_abort(p);
  return rc;
}

int pe_pipe_capture_abort(pe_pipe* p) {
  if (p == nullptr || !p->capturing) return PE_OK;
  cudaGraph_t graph = nullptr;
  cudaStreamEndCapture(p->compute, &graph);
  if (graph != nullptr) cudaGraphDestroy(graph);
  cudaGetLastError();
  p->capturing = false;
  return PE_OK;
}

static int end_capture(cudaStream_t stream, cudaGraphExec_t* exec, const char* what) {
  cudaGraph_t graph = nullptr;
  const cudaError_t end = cudaStreamEndCapture(stream, &graph);
  if (end != cudaSuccess || graph == nullptr) {
    if (graph != nullptr) cudaGraphDestroy(graph);
    return pe::check_cuda(end != cudaSuccess ? end : cudaErrorUnknown, what);
  }
  const cudaError_t inst = cudaGraphInstantiate(exec, graph, 0);
  cudaGraphDestroy(graph);
  PE_CUDA(inst);
  PE_CUDA(cudaGraphUpload(*exec, stream));   // the first replay must not pay for moving the graph to the device
  PE_CUDA(cudaStreamSynchronize(stream));
  return PE_OK;
}

// Finish the capture started by pe_pipe_capture_begin for its parity: the put of the stage's output (x_i = a_i + b_i when
// b_i != NULL; QuantPipe `bit` / `clamp` as pe_link_put) goes into the same graph (overlap == 0; parity must be 0) or
// into a graph of its own on the send stream (overlap != 0: capture parity 0 AND 1, each over its own output buffers).
// The graph is filed under (ubatch, dim1, bit); parity 1 completes the parity 0 capture of the same bit-width.
// *kernels = kernels per micro-batch.
int pe_pipe_capture_end(pe_pipe* p, const void* a0, const void* b0, size_t n0, const void* a1, const void* b1, size_t n1,
                        int items, int bit, int clamp, int overlap, int* kernels) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && p->capturing, "pe_pipe_capture_end: no capture in progress");
  PE_REQUIRE(overlap != 0 || p->cap_parity == 0, "pe_pipe_capture_end: parity 1 exists only with an overlapped send");
  if (p->cap_parity == 1) {
    bool has_par0 = false;
    {
      std::lock_guard<std::mutex> lock(p->graphs_mu);
      auto it = p->graphs.find(std::make_tuple(p->cap_ubatch, p->cap_dim1, bit));
      has_par0 = it != p->graphs.end() && it->second.n_par == 1;
    }
    if (!has_par0) {
      pe_pipe_capture_abort(p);
      set_error("pe_pipe_capture_end: parity 1 of bit-width %d without its parity 0", bit);
      return PE_ERR_INVALID;
    }
  }
  PutTensor t[2] = {{static_cast<const float*>(a0), static_cast<const float*>(b0), n0},
                    {static_cast<const float*>(a1), static_cast<const float*>(b1), n1}};
  const int par = p->cap_parity;
  const bool stamps = p->cap_stamps;
  const int n_tensors = a1 != nullptr ? 2 : 1;
  cudaGraphExec_t exec_main = nullptr, exec_put = nullptr;
  int rc = PE_OK;
  if (stamps) {   // the stage's last kernel is done (and, with the send in this graph, the send starts)
    StampArgs st = {};
    st.what = overlap != 0 ? kStampStage : (kStampStage | kStampSendStart);
    st.bump = overlap != 0 ? 1 : 0;
    rc = launch_stamp(p, st, p->compute);
  }
  if (rc == PE_OK && overlap == 0) {
    rc = stamps ? put_stamped(p, t, n_tensors, items, bit, clamp, 0, p->compute)
                : link_put(p->out, t, n_tensors, items, bit, clamp, p->compute);
  }
  if (rc != PE_OK) {
    pe_pipe_capture_abort(p);
    return rc;
  }
  p->capturing = false;
  rc = end_capture(p->compute, &exec_main, "cudaStreamEndCapture (pipe)");
  if (rc != PE_OK) return rc;
  if (overlap != 0) {
    PE_CUDA(cudaStreamBeginCapture(p->put, cudaStreamCaptureModeRelaxed));
    rc = stamps ? put_stamped(p, t, n_tensors, items, bit, clamp, 1, p->put)
                : link_put(p->out, t, n_tensors, items, bit, clamp, p->put);
    if (rc != PE_OK) {
      cudaGraph_t graph = nullptr;
      cudaStreamEndCapture(p->put, &graph);
      if (graph != nullptr) cudaGraphDestroy(graph);
      cudaGetLastError();
      cudaGraphExecDestroy(exec_main);
      return rc;
    }
    rc = end_capture(p->put, &exec_put, "cudaStreamEndCapture (pipe, send)");
    if (rc != PE_OK) {
      cudaGraphExecDestroy(exec_main);
      return rc;
    }
  }
  const int captured = static_cast<int>(launch_count_now() - p->cap_launch0);
  file_graph(p, p->cap_ubatch, p->cap_dim1, bit, par, exec_main, exec_put, overlap != 0 ? 2 : 1, captured, stamps);
  if (kernels != nullptr) *kernels = captured;
  return PE_OK;
}

// Data rank outside the stage pipeline (in: host-fed link, out: the producer end of the hop to the first stage, res: the
// consumer end of the hop from the last stage): capture the relay graph of micro-batches of `ubatch` items whose input
// is `bytes` bytes, filed as (ubatch, dim1, bit-width 0). pe_pipe_submit / close_input / next_result / sync then serve
// it as they serve a data rank that owns the first stage. With stamps on, the graph's record has t_start, t_send_start,
// t_send_end, bytes_out = `bytes`, bit_out = 0 and bit_in = -1. *kernels = kernels per micro-batch.
int pe_pipe_capture_relay(pe_pipe* p, int ubatch, long long dim1, size_t bytes, int* kernels) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && !p->capturing, "pe_pipe_capture_relay: bad state");
  PE_REQUIRE(p->in->kind == 2, "pe_pipe_capture_relay: this pipe's input is not host-fed");
  PE_REQUIRE(ubatch > 0 && ubatch <= kLinkMaxItems && bytes > 0, "pe_pipe_capture_relay: %d items / %zu bytes", ubatch,
             bytes);
  PE_REQUIRE(kLinkHeaderBytes + bytes <= p->in->slot_bytes && kLinkHeaderBytes + bytes <= p->out->slot_bytes,
             "pe_pipe_capture_relay: %zu bytes exceed the input ring's %zu-byte or the link's %zu-byte slots", bytes,
             p->in->slot_bytes - kLinkHeaderBytes, p->out->slot_bytes - kLinkHeaderBytes);
  PE_CUDA(cudaStreamSynchronize(p->compute));
  const bool stamps = p->stamps_on.load();
  PE_CUDA(cudaStreamBeginCapture(p->compute, cudaStreamCaptureModeRelaxed));
  p->capturing = true;
  StampArgs st = {};
  st.what = kStampStart | kStampGot | kStampStage | kStampSendStart;   // no receive, no stage: one stamp
  int rc = stamps ? launch_stamp(p, st, p->compute) : PE_OK;
  if (rc == PE_OK) rc = link_relay(p->in, p->out, ubatch, bytes, p->compute);
  if (rc == PE_OK && stamps) {
    st = {};
    st.what = kStampSendEnd;
    st.bump = 3;
    st.items = ubatch;
    st.bit_out = 0;
    st.bytes_out = bytes;
    rc = launch_stamp(p, st, p->compute);
  }
  if (rc != PE_OK) {
    pe_pipe_capture_abort(p);
    return rc;
  }
  p->capturing = false;
  cudaGraphExec_t exec = nullptr;
  rc = end_capture(p->compute, &exec, "cudaStreamEndCapture (relay)");
  if (rc != PE_OK) return rc;
  // counted here, not from the process-wide launch counter: the results thread may launch receives meanwhile
  const int captured = stamps ? 3 : 1;
  file_graph(p, ubatch, dim1, 0, 0, exec, nullptr, 1, captured, stamps);
  if (kernels != nullptr) *kernels = captured;
  return PE_OK;
}

// Drop every captured graph (the stage's output quantisation changed).
int pe_pipe_invalidate(pe_pipe* p) {
  PE_REQUIRE(p != nullptr && !p->capturing, "pe_pipe_invalidate: bad state");
  PE_CUDA(cudaStreamSynchronize(p->compute));
  PE_CUDA(cudaStreamSynchronize(p->put));
  std::lock_guard<std::mutex> lock(p->graphs_mu);
  for (auto& kv : p->graphs) pe::destroy_graph(kv.second);
  p->graphs.clear();
  p->latest_bit.clear();
  return PE_OK;
}

// Data rank: feed one micro-batch (`bytes` at `src`, host or device memory) and launch its graph. Blocks while the input
// ring is full. The source must stay valid until the copy has run (callers keep the last n_slots sources alive).
int pe_pipe_submit(pe_pipe* p, const void* src, size_t bytes, int src_is_host, int ubatch, long long dim1) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && p->in->kind == 2, "pe_pipe_submit: this pipe's input is not host-fed");
  const int bit = p->send_bit.load();
  // refused before the input is fed: a micro-batch without its graph must not occupy the input ring
  PE_REQUIRE(find_graph(p, ubatch, dim1, bit, nullptr, false),
             "pipe: no graph captured for micro-batch size %d / dim %lld / send bit-width %d", ubatch, dim1, bit);
  int rc = link_feed(p->in, src, bytes, src_is_host, p->copy);
  if (rc != PE_OK) return rc;
  rc = launch_graph(p, ubatch, dim1, bit);
  if (rc != PE_OK) return rc;
  return link_ticket_send(p->out, ubatch, p->out_dim > 0 ? p->out_dim : dim1);
}

// Last stage: what its outgoing tickets say in their second word - the elements per item of the result tensor, which
// the data rank needs to drain it (it does not own the last shard).
int pe_pipe_set_out_dim(pe_pipe* p, long long n) {
  PE_REQUIRE(p != nullptr && n >= 0, "pe_pipe_set_out_dim: bad arguments");
  p->out_dim = n;
  return PE_OK;
}

// Data rank: no more inputs - the closing ticket travels down the pipeline and comes back on the results link.
int pe_pipe_close_input(pe_pipe* p) {
  PE_REQUIRE(p != nullptr, "pe_pipe_close_input: null pipe");
  return pe::link_ticket_send(p->out, -1, 0);
}

// Downstream ranks: serve tickets until the upstream closes (returns 1, after forwarding the close and draining the
// device) or a ticket arrives for which no graph exists (returns 2 with need2 = {ubatch, dim1}; capture it and call
// again - the ticket is kept). Call with the GIL released.
int pe_pipe_run(pe_pipe* p, long long* need2) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && need2 != nullptr && p->in->kind != 2, "pe_pipe_run: bad arguments");
  for (;;) {
    if (!p->pending) {
      const int r = link_ticket_recv(p->in, p->pend);
      if (r < 0) return r;
      if (r == 1 || p->pend[0] < 0) {
        link_ticket_send(p->out, -1, 0);
        PE_CUDA(cudaStreamSynchronize(p->compute));
        PE_CUDA(cudaStreamSynchronize(p->put));
        const int rc = link_check(p->in);
        return rc != PE_OK ? rc : 1;
      }
    }
    const int ubatch = static_cast<int>(p->pend[0]);
    const int bit = p->send_bit.load();   // one read per micro-batch: the check and the launch agree
    if (!find_graph(p, ubatch, p->pend[1], bit, nullptr)) {
      p->pending = true;
      need2[0] = p->pend[0];
      need2[1] = p->pend[1];
      return 2;
    }
    p->pending = false;
    int rc = launch_graph(p, ubatch, p->pend[1], bit);
    if (rc != PE_OK) return rc;
    rc = link_ticket_send(p->out, p->pend[0], p->out_dim > 0 ? p->out_dim : p->pend[1]);
    if (rc != PE_OK) return rc;
  }
}

// Data rank: block until the next result has reached host memory. Returns 1 when the pipeline has closed; otherwise
// *host_ptr (f32 [*items, *n], valid until the next call).
int pe_pipe_next_result(pe_pipe* p, void** host_ptr, int* items, size_t* n_out) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && p->res != nullptr && host_ptr != nullptr && items != nullptr && n_out != nullptr,
             "pe_pipe_next_result: bad arguments");
  long long t[2];
  const int r = link_ticket_recv(p->res, t);
  if (r < 0) return r;
  if (r == 1 || t[0] < 0) return 1;
  const int ubatch = static_cast<int>(t[0]);
  PE_REQUIRE(t[1] > 0, "pe_pipe_next_result: the last stage did not announce its result size");
  const size_t n = static_cast<size_t>(t[1]);
  *n_out = n;
  const size_t bytes = static_cast<size_t>(ubatch) * n * sizeof(float);
  PE_REQUIRE(bytes <= p->res_cap, "pe_pipe_next_result: result of %zu bytes exceeds the results link's slots", bytes);
  int rc = link_get(p->res, p->res_dev, nullptr, ubatch, n, 0, 1, p->results, true);
  if (rc != PE_OK) return rc;
  PE_CUDA(cudaMemcpyAsync(p->res_host, p->res_dev, bytes, cudaMemcpyDeviceToHost, p->results));
  PE_CUDA(cudaEventRecord(p->ev_res_last, p->results));
  p->have_res = true;
  const cudaError_t e = cudaStreamSynchronize(p->results);
  rc = link_check(p->res);
  if (rc != PE_OK) return rc;
  PE_CUDA(e);
  *host_ptr = p->res_host;
  *items = ubatch;
  return PE_OK;
}

int pe_pipe_sync(pe_pipe* p) {
  using namespace pe;
  PE_REQUIRE(p != nullptr, "pe_pipe_sync: null pipe");
  PE_CUDA(cudaStreamSynchronize(p->copy));
  PE_CUDA(cudaStreamSynchronize(p->compute));
  PE_CUDA(cudaStreamSynchronize(p->put));
  int rc = link_check(p->in);
  if (rc == PE_OK) rc = link_check(p->out);
  return rc;
}

// The next graph launch starts a new timed phase.
int pe_pipe_timing_reset(pe_pipe* p) {
  PE_REQUIRE(p != nullptr, "pe_pipe_timing_reset: null pipe");
  p->timing_reset.store(1);
  return PE_OK;
}

// Device time of the current phase (call after the phase has drained): compute_ms = first graph launch -> end of the last
// graph on this rank's compute stream; results_ms = first graph launch -> last result copied out (data rank, else -1).
int pe_pipe_timing(pe_pipe* p, float* compute_ms, float* results_ms, unsigned long long* launches,
                   unsigned long long* kernels) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && compute_ms != nullptr && results_ms != nullptr, "pe_pipe_timing: null pointer");
  *compute_ms = -1.f;
  *results_ms = -1.f;
  if (p->have_first && p->timed_launches > 0) {
    PE_CUDA(cudaEventSynchronize(p->ev_last));
    PE_CUDA(cudaEventElapsedTime(compute_ms, p->ev_first, p->ev_last));
    if (p->have_res) {
      PE_CUDA(cudaEventSynchronize(p->ev_res_last));
      PE_CUDA(cudaEventElapsedTime(results_ms, p->ev_first, p->ev_res_last));
    }
  }
  if (launches != nullptr) *launches = p->timed_launches;
  if (kernels != nullptr) *kernels = p->timed_kernels;
  return PE_OK;
}

// Capture the next graphs with (on != 0) or without timestamp kernels. The ring is allocated on first use and kept.
int pe_pipe_enable_stamps(pe_pipe* p, int on) {
  using namespace pe;
  PE_REQUIRE(p != nullptr, "pe_pipe_enable_stamps: null pipe");
  if (on != 0 && p->stamp_host == nullptr) {
    const size_t bytes = sizeof(StampSlot) * PE_PIPE_STAMP_DEPTH;
    void* host = nullptr;
    void* ctr = nullptr;
    cudaError_t e = cudaHostAlloc(&host, bytes, cudaHostAllocMapped);
    if (e == cudaSuccess) {
      memset(host, 0, bytes);
      e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&p->stamp_dev), host, 0);
    }
    if (e == cudaSuccess) e = cudaMalloc(&ctr, 2 * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaMemset(ctr, 0, 2 * sizeof(unsigned long long));
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) {   // load the kernel's module now: inside a stream capture a first-use load could be refused
      cudaFuncAttributes attr;
      e = cudaFuncGetAttributes(&attr, pipe_stamp_kernel);
    }
    if (e != cudaSuccess) {
      if (host != nullptr) cudaFreeHost(host);
      if (ctr != nullptr) cudaFree(ctr);
      p->stamp_dev = nullptr;
      return check_cuda(e, "pe_pipe_enable_stamps");
    }
    p->stamp_ctr = static_cast<unsigned long long*>(ctr);
    p->stamp_host = static_cast<StampSlot*>(host);
  }
  p->stamps_on.store(on != 0);
  return PE_OK;
}

// A seqlock read of each record: its sequence word before and after the copy must both name it.
int pe_pipe_drain_stamps(pe_pipe* p, pe_pipe_record* out, int max, int* n, unsigned long long* dropped) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && (out != nullptr || max == 0) && max >= 0 && n != nullptr && dropped != nullptr,
             "pe_pipe_drain_stamps: bad arguments");
  *n = 0;
  if (p->stamp_host == nullptr) return PE_OK;
  constexpr unsigned long long kDepth = PE_PIPE_STAMP_DEPTH;
  while (*n < max) {
    const unsigned long long want = p->stamp_next + 1;
    StampSlot* s = p->stamp_host + p->stamp_next % kDepth;
    const unsigned long long s1 = __atomic_load_n(&s->seq, __ATOMIC_ACQUIRE);
    if (s1 < want) break;   // not complete yet
    if (s1 > want) {
      // the slot already holds record s1 - 1 >= stamp_next + depth: every record older than s1 - depth is gone
      *dropped += s1 - kDepth - p->stamp_next;
      p->stamp_next = s1 - kDepth;
      continue;
    }
    memcpy(&out[*n], &s->rec, sizeof(pe_pipe_record));
    std::atomic_thread_fence(std::memory_order_acquire);
    if (__atomic_load_n(&s->seq, __ATOMIC_RELAXED) == s1) ++*n;
    else ++*dropped;   // overwritten while it was copied
    ++p->stamp_next;
  }
  return PE_OK;
}

}  // extern "C"
