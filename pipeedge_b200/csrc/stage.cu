// Stage executor: runs the encoder-block sub-layers [layer_start, layer_end] of one pipeline stage as
// a fixed sequence of the kernels in this library, optionally captured once into a CUDA graph and
// replayed (the per-micro-batch sequence is launch-bound: ~7 kernels of a few microseconds per block).
//
// Data layout in HBM (per stage, sized for max_ubatch items of S tokens; M = ubatch * S rows):
//   residual stream   f32 [M, H]   caller-owned (in0 / out0 / out1); updated in place after the first write
//   a16               f16 [M, H]   LayerNorm output / f16 copy of the residual = A operand of QKV and FC1
//   qkv16             f16 [M, 3H]  [Q | K | V], head-major inside each third
//   ctx16             f16 [M, H]   merged-head attention context = A operand of the output projection
//   inter16           f16 [M, I]   GELU(FC1) = A operand of FC2
//   t32               f32 [M, H]   output projection / FC2 result before the residual add, which is folded into
//                                  the LayerNorm that follows (or a small add kernel when the stage ends there)
// Replaces {ViT,DeiT,Bert}ModelShard.forward's block loop (vit.py:161-170, deit.py:158-167, bert.py:142-151).
#include <cstdlib>
#include <map>
#include <tuple>
#include <vector>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"

namespace pe {

void count_launches(int n);
int require_sm90();
int linear_impl(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n, int k,
                int epilogue, int rows_per_item, int out_item_rows, int out_row_offset, int resid_per_item,
                int static_w, cudaStream_t stream);
int linear_ln_impl(const void* a, const void* w, const void* bias, const void* resid, const void* gamma, const void* beta,
                   float eps, void* out_f32, int f32_is_ln, void* out_f16, int m, int n, int k, int static_w,
                   cudaStream_t stream);
int linear_ln_cluster(int n);
bool fuse_ln_enabled();
int layernorm_impl(const void* x, const void* resid, const void* gamma, const void* beta, float eps, void* sum_out,
                   void* out_f32, void* out_f16, int rows, int hidden, cudaStream_t stream);
int add_impl(const void* a, const void* b, void* out, size_t n, cudaStream_t stream);
int attention_impl(const void* qkv, void* ctx, int batch, int tokens, int heads, int head_dim, cudaStream_t stream);
int cast_impl(const void* src, void* dst, size_t n, bool to_half, cudaStream_t stream);
int spin_impl(float ms, cudaStream_t stream);

struct SubRange {
  int block;  // index into stage->blocks
  int s0, s1; // sub-layers 0..3 inclusive
};

}  // namespace pe

struct pe_stage {
  pe_stage_desc d;
  std::vector<pe_block_weights> blocks;
  std::vector<pe::SubRange> ranges;
  __half* a16 = nullptr;
  __half* qkv16 = nullptr;
  __half* ctx16 = nullptr;
  __half* inter16 = nullptr;
  float* t32 = nullptr;
  int kernels_last = 0;
  const void* defer_a = nullptr;   // PE_STAGE_DEFER_ADD: the stage's output is defer_a + defer_b, left to the consumer
  const void* defer_b = nullptr;
  cudaStream_t capture_stream = nullptr;  // private stream the kernel sequence is captured on
  typedef std::tuple<int, const void*, const void*, void*, void*> Key;
  struct Cached {
    cudaGraphExec_t exec = nullptr;
    bool warmed = false;
  };
  std::map<Key, Cached> graphs;
};

namespace pe {

#define PE_TRY(call)              \
  do {                            \
    int _rc = (call);             \
    if (_rc != PE_OK) return _rc; \
  } while (0)

// Optional per-kernel timing of one eager forward: an event is recorded after every launch.
struct Prof {
  std::vector<cudaEvent_t> events;  // events[0] precedes the first kernel
  std::vector<int> kinds;           // PE_KERNEL_* of kernel i, timed by events[i] -> events[i+1]
  cudaStream_t stream;
};
static int prof_mark(Prof* prof, int kind) {
  if (prof == nullptr) return PE_OK;
  cudaEvent_t e;
  PE_CUDA(cudaEventCreate(&e));
  PE_CUDA(cudaEventRecord(e, prof->stream));
  prof->events.push_back(e);
  if (kind >= 0) prof->kinds.push_back(kind);
  return PE_OK;
}
// launch + count + (optional) mark
#define PE_K(kind, call)                 \
  do {                                   \
    PE_TRY(call);                        \
    ++n_k;                               \
    PE_TRY(prof_mark(prof, kind));       \
  } while (0)

static int lin(const void* a, const void* w, const void* b, const void* resid, void* out, int m, int n, int k, int epi,
               cudaStream_t s) {
  return linear_impl(a, w, b, resid, out, m, n, k, epi, 0, 0, 0, 0, /*static_w=*/1, s);
}

// Enqueue the kernel sequence of one forward on `stream`. Returns the number of kernels in *count.
static int enqueue(pe_stage* st, const void* in0, const void* in1, void* out0, void* out1, int ubatch,
                   cudaStream_t stream, int* count, Prof* prof = nullptr, bool defer_add = false) {
  const pe_stage_desc& d = st->d;
  const int H = d.hidden, I = d.inter, S = d.tokens;
  const int M = ubatch * S;
  const bool post_ln = d.family == PE_FAMILY_BERT;
  const int first_sub = st->ranges.front().s0, last_sub = st->ranges.back().s1;
  const bool in_tuple = first_sub == 1 || first_sub == 3;
  const bool out_tuple = last_sub == 0 || last_sub == 2;
  PE_REQUIRE(in0 && out0, "pe_stage_forward: null payload");
  PE_REQUIRE(!in_tuple || in1, "pe_stage_forward: stage starts mid-block and needs the (data, skip) tuple");
  PE_REQUIRE(!out_tuple || out1, "pe_stage_forward: stage ends mid-block and produces a (data, skip) tuple");
  int n_k = 0;

  // every residual-stream write lands in the buffer that finally carries it out of the stage
  float* resid_dest = static_cast<float*>(out_tuple ? out1 : out0);
  const float* x = nullptr;     // current fp32 residual stream, when materialised
  const float* skip = nullptr;  // skip tensor of a pending (data, skip) tuple
  bool pending = false;         // residual stream = t32 + skip, not yet added (pre-LN only)
  bool a16_valid = false;       // a16 holds the f16 copy of x (post-LN only)

  // Projection + residual add + LayerNorm as ONE kernel (cluster epilogue, gemm_wgmma.cu) wherever the LayerNorm that
  // follows an output projection / FC2 belongs to this stage and the width splits into <= 8 slices of <= 128 columns.
  const bool fuse_ln = fuse_ln_enabled() && linear_ln_cluster(H) > 0;
  bool a16_ready = false;       // pre-LN: a16 already holds LayerNorm(x) for the sub-layer about to run

  if (first_sub == 0 || first_sub == 2) {
    x = static_cast<const float*>(in0);
  } else if (first_sub == 1) {
    PE_K(PE_KERNEL_CAST, cast_impl(in0, st->ctx16, static_cast<size_t>(M) * H, true, stream));
    skip = static_cast<const float*>(in1);
  } else {
    PE_K(PE_KERNEL_CAST, cast_impl(in0, st->inter16, static_cast<size_t>(M) * I, true, stream));
    skip = static_cast<const float*>(in1);
  }

  for (size_t ri = 0; ri < st->ranges.size(); ++ri) {
    const SubRange& r = st->ranges[ri];
    const pe_block_weights& w = st->blocks[r.block];
    for (int sub = r.s0; sub <= r.s1; ++sub) {
      const bool has_next = sub < r.s1 || ri + 1 < st->ranges.size();   // another sub-layer of this stage follows
      const bool attn_half = sub == 0;
      switch (sub) {
        case 0:
        case 2: {
          const void* ln_w = attn_half ? w.ln1_w : w.ln2_w;
          const void* ln_b = attn_half ? w.ln1_b : w.ln2_b;
          if (post_ln) {
            if (!a16_valid) { PE_K(PE_KERNEL_CAST, cast_impl(x, st->a16, static_cast<size_t>(M) * H, true, stream)); }
          } else if (a16_ready) {
            a16_ready = false;   // the producing projection already wrote x and a16 = LayerNorm(x)
          } else if (pending) {
            // residual add of the previous sub-layer + this LayerNorm in one pass; the sum becomes the stream
            PE_K(PE_KERNEL_LAYERNORM, layernorm_impl(st->t32, skip, ln_w, ln_b, d.eps, resid_dest, nullptr, st->a16, M, H, stream));
            x = resid_dest;
            pending = false;
          } else {
            PE_K(PE_KERNEL_LAYERNORM, layernorm_impl(x, nullptr, ln_w, ln_b, d.eps, nullptr, nullptr, st->a16, M, H, stream));
          }
          if (attn_half) {
            PE_K(PE_KERNEL_GEMM_QKV, lin(st->a16, w.w_qkv, w.b_qkv, nullptr, st->qkv16, M, 3 * H, H, PE_EPI_F16, stream));
            PE_K(PE_KERNEL_ATTENTION, attention_impl(st->qkv16, st->ctx16, ubatch, S, d.heads, H / d.heads, stream));
          } else {
            PE_K(PE_KERNEL_GEMM_FC1, lin(st->a16, w.w_fc1, w.b_fc1, nullptr, st->inter16, M, I, H, PE_EPI_GELU_F16, stream));
          }
          skip = x; x = nullptr; a16_valid = false;
          break;
        }
        default: {   // 1: output projection, 3: FC2 - both produce t32 = A @ W^T + b, residual add deferred
          const void* a_op = sub == 1 ? static_cast<const void*>(st->ctx16) : static_cast<const void*>(st->inter16);
          const void* w_op = sub == 1 ? w.w_o : w.w_fc2;
          const void* b_op = sub == 1 ? w.b_o : w.b_fc2;
          const int k_op = sub == 1 ? H : I;
          const int kind = sub == 1 ? PE_KERNEL_GEMM_OUT : PE_KERNEL_GEMM_FC2;
          if (fuse_ln && post_ln) {
            // BertSelfOutput / BertOutput: LayerNorm(dense(a) + input) -> fp32 stream and fp16 operand in one kernel
            const void* ln_w = sub == 1 ? w.ln1_w : w.ln2_w;
            const void* ln_b = sub == 1 ? w.ln1_b : w.ln2_b;
            PE_K(kind, linear_ln_impl(a_op, w_op, b_op, skip, ln_w, ln_b, d.eps, resid_dest, 1, st->a16, M, H, k_op, 1, stream));
            a16_valid = true;
            x = resid_dest; skip = nullptr;
            break;
          }
          if (fuse_ln && !post_ln && has_next) {
            // ViT: x = dense(a) + skip -> the residual stream, and LayerNorm(x) of the sub-layer that follows -> a16
            const pe_block_weights& wn = sub == 1 ? w : st->blocks[st->ranges[ri + 1].block];
            const void* ln_w = sub == 1 ? wn.ln2_w : wn.ln1_w;
            const void* ln_b = sub == 1 ? wn.ln2_b : wn.ln1_b;
            PE_K(kind, linear_ln_impl(a_op, w_op, b_op, skip, ln_w, ln_b, d.eps, resid_dest, 0, st->a16, M, H, k_op, 1, stream));
            x = resid_dest; skip = nullptr;
            a16_ready = true;
            break;
          }
          if (sub == 1) {
            PE_K(PE_KERNEL_GEMM_OUT, lin(st->ctx16, w.w_o, w.b_o, nullptr, st->t32, M, H, H, PE_EPI_F32, stream));
          } else {
            PE_K(PE_KERNEL_GEMM_FC2, lin(st->inter16, w.w_fc2, w.b_fc2, nullptr, st->t32, M, H, I, PE_EPI_F32, stream));
          }
          if (post_ln) {
            const void* ln_w = sub == 1 ? w.ln1_w : w.ln2_w;
            const void* ln_b = sub == 1 ? w.ln1_b : w.ln2_b;
            PE_K(PE_KERNEL_LAYERNORM, layernorm_impl(st->t32, skip, ln_w, ln_b, d.eps, nullptr, resid_dest, st->a16, M, H, stream));
            a16_valid = true;
            x = resid_dest; skip = nullptr;
          } else {
            pending = true;   // x = t32 + skip
          }
          break;
        }
      }
    }
  }
  st->defer_a = st->defer_b = nullptr;
  if (pending && defer_add && !out_tuple) {
    // the stage ends on an output projection / FC2 and its consumer (the link's send kernel) adds while it reads
    st->defer_a = st->t32;
    st->defer_b = skip;
    pending = false;
  } else if (pending) {   // ... otherwise materialise the sum
    PE_K(PE_KERNEL_CAST, add_impl(st->t32, skip, resid_dest, static_cast<size_t>(M) * H, stream));
    x = resid_dest; skip = nullptr; pending = false;
  }

  if (out_tuple) {
    // (ctx | inter, skip): the f16 operand is widened for the fp32 wire format of the boundary payload
    if (last_sub == 0) { PE_K(PE_KERNEL_CAST, cast_impl(st->ctx16, out0, static_cast<size_t>(M) * H, false, stream)); }
    else { PE_K(PE_KERNEL_CAST, cast_impl(st->inter16, out0, static_cast<size_t>(M) * I, false, stream)); }
    if (skip != static_cast<const float*>(out1)) {
      PE_CUDA(cudaMemcpyAsync(out1, skip, static_cast<size_t>(M) * H * sizeof(float), cudaMemcpyDeviceToDevice, stream));
    }
  }
  *count = n_k;
  return PE_OK;
}

static int build_ranges(pe_stage* st) {
  // same walk as ViTModelShard._build_shard (vit.py:99-113): 1-based sub-layer l -> block ceil(l/4)-1
  const int ls = st->d.layer_start, le = st->d.layer_end;
  const int first_block = (ls + 3) / 4 - 1, last_block = (le + 3) / 4 - 1;
  int cur = ls;
  while (cur <= le) {
    const int block = (cur + 3) / 4 - 1;
    const int s0 = (cur - 1) % 4;
    const int s1 = block == last_block ? (le - 1) % 4 : 3;
    st->ranges.push_back({block - first_block, s0, s1});
    cur += s1 - s0 + 1;
  }
  return last_block - first_block + 1;
}

}  // namespace pe

extern "C" {

int pe_stage_create(const pe_stage_desc* desc, const pe_block_weights* blocks, int n_blocks, pe_stage** out) {
  using namespace pe;
  PE_REQUIRE(desc && blocks && out, "pe_stage_create: null pointer");
  PE_REQUIRE(desc->family >= PE_FAMILY_VIT && desc->family <= PE_FAMILY_BERT, "pe_stage_create: bad family %d",
             desc->family);
  PE_REQUIRE(desc->layer_start >= 1 && desc->layer_end >= desc->layer_start, "pe_stage_create: bad layer range [%d,%d]",
             desc->layer_start, desc->layer_end);
  PE_REQUIRE(desc->hidden > 0 && desc->heads > 0 && desc->hidden % desc->heads == 0 &&
                 (desc->hidden / desc->heads == 64 || desc->hidden / desc->heads == 80),
             "pe_stage_create: hidden=%d heads=%d (head_dim must be 64 or 80)", desc->hidden, desc->heads);
  PE_REQUIRE(desc->hidden % 8 == 0 && desc->inter % 8 == 0 && desc->inter > 0, "pe_stage_create: bad hidden/inter");
  PE_REQUIRE(desc->tokens > 0 && desc->max_ubatch > 0, "pe_stage_create: bad tokens/max_ubatch");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;
  pe_stage* st = new pe_stage();
  st->d = *desc;
  const int need = build_ranges(st);
  if (need != n_blocks) {
    set_error("pe_stage_create: layers [%d,%d] touch %d blocks but %d weight sets were given", desc->layer_start,
              desc->layer_end, need, n_blocks);
    delete st;
    return PE_ERR_INVALID;
  }
  st->blocks.assign(blocks, blocks + n_blocks);
  for (const SubRange& r : st->ranges) {
    const pe_block_weights& w = st->blocks[r.block];
    bool ok = true;
    for (int s = r.s0; s <= r.s1; ++s) {
      if (s == 0) ok = ok && w.w_qkv && w.b_qkv && (desc->family == PE_FAMILY_BERT || (w.ln1_w && w.ln1_b));
      if (s == 1) ok = ok && w.w_o && w.b_o && (desc->family != PE_FAMILY_BERT || (w.ln1_w && w.ln1_b));
      if (s == 2) ok = ok && w.w_fc1 && w.b_fc1 && (desc->family == PE_FAMILY_BERT || (w.ln2_w && w.ln2_b));
      if (s == 3) ok = ok && w.w_fc2 && w.b_fc2 && (desc->family != PE_FAMILY_BERT || (w.ln2_w && w.ln2_b));
    }
    if (!ok) {
      set_error("pe_stage_create: missing weights for block %d sub-layers %d-%d", r.block, r.s0, r.s1);
      delete st;
      return PE_ERR_INVALID;
    }
  }
  const size_t M = static_cast<size_t>(desc->max_ubatch) * desc->tokens;
  const size_t H = desc->hidden, I = desc->inter;
  cudaError_t e = cudaSuccess;
  if (e == cudaSuccess) e = cudaMalloc(&st->a16, M * H * sizeof(__half));
  if (e == cudaSuccess) e = cudaMalloc(&st->qkv16, M * 3 * H * sizeof(__half));
  if (e == cudaSuccess) e = cudaMalloc(&st->ctx16, M * H * sizeof(__half));
  if (e == cudaSuccess) e = cudaMalloc(&st->inter16, M * I * sizeof(__half));
  if (e == cudaSuccess) e = cudaMalloc(&st->t32, M * H * sizeof(float));
  if (e != cudaSuccess) {
    set_error("pe_stage_create: workspace allocation failed: %s", cudaGetErrorString(e));
    pe_stage_destroy(st);
    return PE_ERR_NOMEM;
  }
  *out = st;
  return PE_OK;
}

int pe_stage_destroy(pe_stage* st) {
  if (st == nullptr) return PE_OK;
  for (auto& kv : st->graphs)
    if (kv.second.exec != nullptr) cudaGraphExecDestroy(kv.second.exec);
  if (st->capture_stream != nullptr) cudaStreamDestroy(st->capture_stream);
  cudaFree(st->a16);
  cudaFree(st->qkv16);
  cudaFree(st->ctx16);
  cudaFree(st->inter16);
  cudaFree(st->t32);
  delete st;
  return PE_OK;
}

int pe_stage_forward(pe_stage* st, const void* in0, const void* in1, void* out0, void* out1, int ubatch, int use_graph,
                     void* stream_v) {
  using namespace pe;
  PE_REQUIRE(st != nullptr, "pe_stage_forward: null stage");
  PE_REQUIRE(ubatch > 0 && ubatch <= st->d.max_ubatch, "pe_stage_forward: ubatch=%d outside [1,%d]", ubatch,
             st->d.max_ubatch);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  if ((use_graph & 1) == 0)
    return enqueue(st, in0, in1, out0, out1, ubatch, stream, &st->kernels_last, nullptr, (use_graph & PE_STAGE_DEFER_ADD) != 0);

  pe_stage::Cached& c = st->graphs[pe_stage::Key(ubatch, in0, in1, out0, out1)];
  if (c.exec != nullptr) {
    PE_CUDA(cudaGraphLaunch(c.exec, stream));
    count_launches(st->kernels_last);
    return PE_OK;
  }
  if (!c.warmed) {
    // first use: run eagerly (one-time cudaFuncSetAttribute / driver entry-point lookups happen here)
    c.warmed = true;
    return enqueue(st, in0, in1, out0, out1, ubatch, stream, &st->kernels_last);
  }
  // second use: capture the same sequence on the stage's private stream (the caller's stream may be the
  // legacy default stream, which cannot be captured), instantiate, then launch into the caller's stream
  if (st->graphs.size() > 64) {  // pointers that never repeat would grow the cache without bound: start over
    const pe_stage::Key mine(ubatch, in0, in1, out0, out1);
    for (auto it = st->graphs.begin(); it != st->graphs.end();) {
      if (it->first == mine) { ++it; continue; }
      if (it->second.exec != nullptr) cudaGraphExecDestroy(it->second.exec);
      it = st->graphs.erase(it);
    }
  }
  if (st->capture_stream == nullptr) PE_CUDA(cudaStreamCreateWithFlags(&st->capture_stream, cudaStreamNonBlocking));
  cudaGraph_t graph = nullptr;
  PE_CUDA(cudaStreamBeginCapture(st->capture_stream, cudaStreamCaptureModeThreadLocal));
  int n_k = 0;
  const int rc = enqueue(st, in0, in1, out0, out1, ubatch, st->capture_stream, &n_k);
  const cudaError_t end = cudaStreamEndCapture(st->capture_stream, &graph);
  if (rc != PE_OK) {
    if (graph != nullptr) cudaGraphDestroy(graph);
    return rc;
  }
  PE_CUDA(end);
  const cudaError_t inst = cudaGraphInstantiate(&c.exec, graph, 0);
  cudaGraphDestroy(graph);
  PE_CUDA(inst);
  st->kernels_last = n_k;
  PE_CUDA(cudaGraphLaunch(c.exec, stream));
  return PE_OK;  // kernels were already counted by enqueue() during capture
}

int pe_stage_profile(pe_stage* st, const void* in0, const void* in1, void* out0, void* out1, int ubatch,
                     void* stream_v, float* ms_out, int* kinds_out, int capacity, int* n_out) {
  using namespace pe;
  PE_REQUIRE(st && ms_out && kinds_out && n_out, "pe_stage_profile: null pointer");
  PE_REQUIRE(ubatch > 0 && ubatch <= st->d.max_ubatch, "pe_stage_profile: bad ubatch %d", ubatch);
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  Prof prof;
  prof.stream = stream;
  // Back-log the stream first so that every event and kernel below is already queued when the GPU reaches it
  // (otherwise host launch gaps would be charged to the kernels).
  int rc = spin_impl(4.0f, stream);
  if (rc != PE_OK) return rc;
  rc = prof_mark(&prof, -1);
  int n_k = 0;
  if (rc == PE_OK) rc = enqueue(st, in0, in1, out0, out1, ubatch, stream, &n_k, &prof);
  if (rc == PE_OK) rc = check_cuda(cudaStreamSynchronize(stream), "cudaStreamSynchronize");
  int n = 0;
  if (rc == PE_OK) {
    n = static_cast<int>(prof.kinds.size());
    for (int i = 0; i < n && i < capacity; ++i) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, prof.events[i], prof.events[i + 1]);
      ms_out[i] = ms;
      kinds_out[i] = prof.kinds[i];
    }
  }
  for (cudaEvent_t e : prof.events) cudaEventDestroy(e);
  *n_out = n;
  return rc;
}

int pe_stage_kernel_count(const pe_stage* st) { return st == nullptr ? 0 : st->kernels_last; }

int pe_stage_deferred(const pe_stage* st, const void** a, const void** b) {
  using namespace pe;
  PE_REQUIRE(st != nullptr && a != nullptr && b != nullptr, "pe_stage_deferred: null pointer");
  *a = st->defer_a;
  *b = st->defer_b;
  return PE_OK;
}

}  // extern "C"
