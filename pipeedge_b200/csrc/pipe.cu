// Per-rank pipeline stage loop: one CUDA graph per micro-batch, no Python and no GIL in the steady state.
//
// A stage's whole micro-batch - link get (wait for the upstream payload, copy / dequantise it into the stage's fixed
// input buffer) -> embeddings / encoder blocks / head kernels -> link put (quantise-and-send into the downstream ring) -
// is captured ONCE per (micro-batch size, sequence length) into a CUDA graph: the link kernels find their ring slot
// through device-resident sequence counters (link.cu), so the graph takes no per-payload arguments and the first
// replay is already the steady state. The host side of a stage is this loop:
//     read a 16-byte ticket from the upstream hop's socket (blocks) -> cudaGraphLaunch -> write the ticket downstream
// i.e. two system calls and one launch per micro-batch; ordering against the neighbours' GPUs is entirely on the
// devices (flags in peer memory). The data rank feeds its first stage through a host-fed link (pe_pipe_submit: H2D /
// D2D copy on a side stream + graph launch) and drains results through pe_pipe_next_result.
//
// Replaces TensorWorkThread.run + the queue hand-offs of DistP2pPipelineStage (p2p/__init__.py:261-295,373-394,442-450):
// FIFO per hop (tickets and flags are strictly ordered), back-pressure through the rings (a producer blocks - on the
// device - until the consumer has released the slot; enqueue blocks on the host-fed ring).
#include <atomic>
#include <map>
#include <mutex>
#include <utility>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"
#include "link.cuh"

namespace pe {
void count_launches(int n);
uint64_t launch_count_now();
int require_sm90();
constexpr int kPipeWindow = 8;   // graph launches the host may run ahead of the device
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
  };
  cudaEvent_t ev_main_done[2] = {nullptr, nullptr}, ev_put_done[2] = {nullptr, nullptr};
  bool put_pending[2] = {false, false};
  int cap_parity = 0;
  std::map<std::pair<int, long long>, Graph> graphs;
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
};

namespace pe {

static bool find_graph(pe_pipe* p, int ubatch, long long dim1, pe_pipe::Graph* out) {
  std::lock_guard<std::mutex> lock(p->graphs_mu);
  auto it = p->graphs.find(std::make_pair(ubatch, dim1));
  if (it == p->graphs.end() || it->second.n_par < it->second.want_par) return false;   // every parity captured?
  if (out != nullptr) *out = it->second;
  return true;
}

static void destroy_graph(pe_pipe::Graph& g) {
  for (int i = 0; i < 2; ++i) {
    if (g.exec[i] != nullptr) cudaGraphExecDestroy(g.exec[i]);
    if (g.exec_put[i] != nullptr) cudaGraphExecDestroy(g.exec_put[i]);
    g.exec[i] = g.exec_put[i] = nullptr;
  }
  g.n_par = 0;
}

static int launch_graph(pe_pipe* p, int ubatch, long long dim1) {
  pe_pipe::Graph g;
  PE_REQUIRE(find_graph(p, ubatch, dim1, &g), "pipe: no graph captured for micro-batch size %d / dim %lld", ubatch, dim1);
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

int pe_pipe_has_graph(pe_pipe* p, int ubatch, long long dim1) {
  return (p != nullptr && pe::find_graph(p, ubatch, dim1, nullptr)) ? 1 : 0;
}

// Start capturing the graph for micro-batches of `ubatch` items (`dim1`: sequence length, part of the key). The get
// kernel is enqueued first: from a host-fed link `raw_bytes` bytes land in dst0; from a hop the payload's one or two
// tensors ([ubatch, n0] / [ubatch, n1] f32 after decoding) land in dst0 / dst1.
int pe_pipe_capture_begin(pe_pipe* p, int ubatch, long long dim1, int parity, void* dst0, void* dst1, size_t n0, size_t n1,
                          size_t raw_bytes) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && !p->capturing && ubatch > 0 && (parity == 0 || parity == 1),
             "pe_pipe_capture_begin: bad state / arguments");
  PE_CUDA(cudaStreamSynchronize(p->compute));
  PE_CUDA(cudaStreamSynchronize(p->put));
  p->cap_parity = parity;
  PE_CUDA(cudaStreamBeginCapture(p->compute, cudaStreamCaptureModeRelaxed));
  p->capturing = true;
  p->cap_ubatch = ubatch;
  p->cap_dim1 = dim1;
  p->cap_launch0 = launch_count_now();
  int rc;
  if (p->in->kind == 2) rc = link_get_raw(p->in, dst0, raw_bytes, p->compute, false);
  else rc = link_get(p->in, dst0, dst1, ubatch, n0, n1, dst1 != nullptr ? 2 : 1, p->compute, false);
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
// *kernels = kernels per micro-batch.
int pe_pipe_capture_end(pe_pipe* p, const void* a0, const void* b0, size_t n0, const void* a1, const void* b1, size_t n1,
                        int items, int bit, int clamp, int overlap, int* kernels) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && p->capturing, "pe_pipe_capture_end: no capture in progress");
  PE_REQUIRE(overlap != 0 || p->cap_parity == 0, "pe_pipe_capture_end: parity 1 exists only with an overlapped send");
  PutTensor t[2] = {{static_cast<const float*>(a0), static_cast<const float*>(b0), n0},
                    {static_cast<const float*>(a1), static_cast<const float*>(b1), n1}};
  const int par = p->cap_parity;
  cudaGraphExec_t exec_main = nullptr, exec_put = nullptr;
  int rc;
  if (overlap == 0) {
    rc = link_put(p->out, t, a1 != nullptr ? 2 : 1, items, bit, clamp, p->compute);
    if (rc != PE_OK) {
      pe_pipe_capture_abort(p);
      return rc;
    }
  }
  p->capturing = false;
  rc = end_capture(p->compute, &exec_main, "cudaStreamEndCapture (pipe)");
  if (rc != PE_OK) return rc;
  if (overlap != 0) {
    PE_CUDA(cudaStreamBeginCapture(p->put, cudaStreamCaptureModeRelaxed));
    rc = link_put(p->out, t, a1 != nullptr ? 2 : 1, items, bit, clamp, p->put);
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
  int total = captured;
  {
    std::lock_guard<std::mutex> lock(p->graphs_mu);
    pe_pipe::Graph& g = p->graphs[std::make_pair(p->cap_ubatch, p->cap_dim1)];
    if (par == 0) destroy_graph(g);   // a fresh capture of this key starts with parity 0
    g.want_par = overlap != 0 ? 2 : 1;
    g.exec[par] = exec_main;
    g.exec_put[par] = exec_put;
    g.n_par = par + 1;
    g.kernels = captured;
    total = g.kernels;
  }
  if (kernels != nullptr) *kernels = total;
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
  return PE_OK;
}

// Data rank: feed one micro-batch (`bytes` at `src`, host or device memory) and launch its graph. Blocks while the input
// ring is full. The source must stay valid until the copy has run (callers keep the last n_slots sources alive).
int pe_pipe_submit(pe_pipe* p, const void* src, size_t bytes, int src_is_host, int ubatch, long long dim1) {
  using namespace pe;
  PE_REQUIRE(p != nullptr && p->in->kind == 2, "pe_pipe_submit: this pipe's input is not host-fed");
  int rc = link_feed(p->in, src, bytes, src_is_host, p->copy);
  if (rc != PE_OK) return rc;
  rc = launch_graph(p, ubatch, dim1);
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
    if (!find_graph(p, ubatch, p->pend[1], nullptr)) {
      p->pending = true;
      need2[0] = p->pend[0];
      need2[1] = p->pend[1];
      return 2;
    }
    p->pending = false;
    int rc = launch_graph(p, ubatch, p->pend[1]);
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

}  // extern "C"
