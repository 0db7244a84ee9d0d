/* pipeedge_b200 - C-ABI of the H100-native PipeEdge hot path.
 *
 * The reference (usc-isi/PipeEdge @ 1a68bbb) has no C/FFI boundary on this path: it sits behind three
 * PYTHON contracts (SURVEY.md 8b). This header is the boundary we define beneath them; each entry
 * point names the reference interface it replaces. The Python classes in `pipeedge_b200/` (same names
 * and signatures as the reference's) are the only callers; INTEGRATION.md shows the ctypes binding a
 * reference maintainer would add.
 *
 * Conventions
 *  - every function returns 0 on success or a negative PE_ERR_* code; `pe_last_error()` returns a
 *    thread-local message for the last failure on the calling thread;
 *  - all tensor arguments are DEVICE pointers owned by the caller, row-major, contiguous;
 *    "f32" = IEEE binary32, "f16" = IEEE binary16, "u8" = bytes;
 *  - `stream` is a `cudaStream_t` passed as `void*`; calls only enqueue work and never synchronise;
 *  - no global mutable state besides per-handle state; callable with the Python GIL released;
 *  - the library targets sm_90a (H100) only and refuses to run elsewhere (PE_ERR_DEVICE).
 */
#ifndef PIPEEDGE_B200_H
#define PIPEEDGE_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PE_OK 0
#define PE_ERR_INVALID (-1) /* bad argument / unsupported shape */
#define PE_ERR_CUDA (-2)    /* a CUDA runtime or driver call failed */
#define PE_ERR_DEVICE (-3)  /* no sm_90 device */
#define PE_ERR_NOMEM (-4)

#define PE_ABI_VERSION 2

/* Model family: selects pre-LN (ViT/DeiT: reference `vit.py:55-70`, `deit.py:54-69`) or post-LN
 * (BERT: `bert.py:41-52`) block structure. */
#define PE_FAMILY_VIT 0
#define PE_FAMILY_DEIT 1
#define PE_FAMILY_BERT 2

/* Epilogues of pe_linear (what follows `A @ W^T + bias`). */
#define PE_EPI_F16 0        /* out f16                                   (QKV projections)          */
#define PE_EPI_GELU_F16 1   /* out f16 = gelu_erf(.)                     (ViTIntermediate/BertIntermediate) */
#define PE_EPI_RESID_F32 2  /* out f32 = . + resid(f32)                  (ViTSelfOutput+skip, ViTOutput; BERT pre-LN sums) */
#define PE_EPI_F32 3        /* out f32                                   (classifier heads)         */
#define PE_EPI_TANH_F32 4   /* out f32 = tanh(.)                         (BertPooler)               */
#define PE_EPI_RESID_LN 5   /* internal to pe_linear_residual_layernorm */
/* OR-able into `epilogue`: W is not written by any work still pending on `stream` (model weights). The kernel may then
 * stream W into shared memory / L2 before its programmatic dependency on the preceding kernel resolves. */
#define PE_EPI_STATIC_W 0x100

int pe_abi_version(void);
const char* pe_last_error(void);
/* Number of kernels this library has launched since load (all threads); bench.py reports it. */
uint64_t pe_launch_count(void);

/* ---- LayerNorm over the last dim -------------------------------------------------------------
 * Replaces `nn.LayerNorm` at `vit.py:59,66,168`, the LayerNorm inside `BertSelfOutput`/`BertOutput`
 * (HF modeling_bert.py:294-298,352-356) and `BertEmbeddings.LayerNorm`.
 * x f32 [rows, hidden]; gamma/beta f32 [hidden]; writes out_f32 and/or out_f16 (either may be NULL).
 * Statistics in fp32, two-pass (mean, then centred variance); eps added in fp32. */
int pe_layernorm(const void* x, const void* gamma, const void* beta, float eps, void* out_f32, void* out_f16,
                 int rows, int hidden, void* stream);

/* Same with the residual add folded in: t = y + resid; sum_out (f32, may be NULL, may alias resid) = t;
 * outputs = LayerNorm(t). Replaces `data += skip` + `layernorm_after` (`vit.py:62-66`), the `+ input_tensor`
 * inside `ViTOutput` followed by the next block's `layernorm_before`, and `LayerNorm(dense + input)` in
 * `BertSelfOutput` / `BertOutput`. */
int pe_residual_layernorm(const void* y, const void* resid, const void* gamma, const void* beta, float eps,
                          void* sum_out, void* out_f32, void* out_f16, int rows, int hidden, void* stream);

/* ---- Dense contraction `out = epilogue(A @ W^T + bias)` on wgmma tensor cores ---------------
 * Replaces every `nn.Linear` on the path (`ViTSelfAttention.query/key/value`, `ViTSelfOutput.dense`,
 * `ViTIntermediate.dense`, `ViTOutput.dense` and the Bert equivalents; reference call sites
 * `vit.py:60-69`, `bert.py:45-51`).
 * a f16 [m, k]; w f16 [n, k] (the `nn.Linear.weight` layout); bias f32 [n] or NULL;
 * resid f32 [m, n] (PE_EPI_RESID_F32 only; may alias `out`); out [m, n] f16 or f32 per epilogue.
 * Requires k % 8 == 0 (16-byte TMA row pitch). fp32 accumulation in registers. */
int pe_linear(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n, int k,
              int epilogue, void* stream);

/* Projection + residual add + LayerNorm in ONE kernel: v = a @ w^T + bias + resid (f32 [m, n], may alias out_f32), then
 * LayerNorm(v) over the row. Replaces `ViTSelfOutput.dense` + `data += skip` + `layernorm_after` (`vit.py:62-66`),
 * `ViTOutput` + the next block's `layernorm_before`, and `LayerNorm(dense(x) + input)` of `BertSelfOutput` /
 * `BertOutput` (HF modeling_bert.py:294-298,352-356). The CTAs that own one row's column slices form a thread-block
 * cluster and exchange per-row (mean, M2) through distributed shared memory.
 *   out_f32 (nullable) = v (f32_is_ln == 0: the pre-LN residual stream) or LayerNorm(v) (f32_is_ln != 0: post-LN)
 *   out_f16 (nullable) = LayerNorm(v), the next GEMM's A operand
 * n must split into 1, 2, 4 or 8 column slices of a multiple of 32 and at most 128 columns (pe_linear_ln_cluster(n)
 * > 0: 768, 1024, 384, 192, 128 ...); other widths use pe_linear + pe_residual_layernorm. */
int pe_linear_residual_layernorm(const void* a, const void* w, const void* bias, const void* resid, const void* gamma,
                                 const void* beta, float eps, void* out_f32, int f32_is_ln, void* out_f16, int m, int n,
                                 int k, int static_w, void* stream);
int pe_linear_ln_cluster(int n);

/* ---- Unmasked multi-head self-attention --------------------------------------------------------
 * Replaces HF `eager_attention_forward` as invoked by `ViTSelfAttention`/`BertSelfAttention`
 * (reference passes no mask: `vit.py:60`, `bert.py:45`): softmax(Q K^T * head_dim^-0.5) V.
 * qkv f16 [batch*tokens, 3*heads*head_dim], columns = [Q | K | V], each head-major;
 * ctx f16 [batch*tokens, heads*head_dim] (heads merged, as `context_layer.reshape`). head_dim 64 or 80 (ViT-Huge). */
int pe_attention(const void* qkv, void* ctx, int batch, int tokens, int heads, int head_dim, void* stream);

/* ---- f32 -> f16 cast (boundary payloads entering a mid-block stage) --------------------------- */
int pe_cast_f32_to_f16(const void* src, void* dst, size_t n, void* stream);
int pe_cast_f16_to_f32(const void* src, void* dst, size_t n, void* stream);

/* ---- QuantPipe --------------------------------------------------------------------------------
 * pe_quant_encode replaces `forward_hook_quant_encode` (`runtime.py:73-91`) for one tensor:
 * optional Banner-2019 clamp (`clamp_op.py:11-33`; Laplace if min(x) < 0.2 else GeLU, threshold from
 * the whole micro-batch) followed by `tensor_encode_outerdim` (`basic_op.py:114-170`): per item
 * shift = min, scale = max - shift, code = rint((x - shift) / scale * (2^bit - 1)) in fp32 with IEEE
 * sub/div/mul (no FMA contraction), packed LSB-first floor(32/bit) codes per little-endian uint32.
 *   x      f32 [items, n]            codes  u8  [items, 4 * pe_quant_words(n, bit)]
 *   scale  f32 [items]               shift  f32 [items]
 *   alpha  f32 [1] (out, may be NULL): the clamp threshold used (+inf when clamp == 0)
 *   work   scratch of at least pe_quant_workspace_bytes(items, n) bytes
 * bit in [1,16]; clamp: 0 = none (bare tensor_encode_outerdim), 1 = runtime hook rule. */
#define PE_CLAMP_NONE 0
#define PE_CLAMP_AUTO 1
#define PE_CLAMP_LAPLACE 2 /* force `clamp_banner2019_laplace` */
#define PE_CLAMP_GELU 3    /* force `clamp_banner2019_gelu` */
size_t pe_quant_words(size_t n, int bit);
size_t pe_quant_workspace_bytes(int items, size_t n);
int pe_quant_encode(const void* x, int items, size_t n, int bit, int clamp, void* codes, void* scale, void* shift,
                    void* alpha, void* work, void* stream);
/* Threshold only: the alpha that `clamp_banner2019_{laplace,gelu}(x, bit)` would clamp to
 * (`clamp_op.py:11-33`), written to alpha f32 [1]; scale/shift f32 [items] receive the per-item
 * parameters of the clamped tensor. Two kernels, no codes produced. */
int pe_quant_alpha(const void* x, int items, size_t n, int bit, int clamp, void* scale, void* shift, void* alpha,
                   void* work, void* stream);
/* pe_quant_decode replaces `forward_pre_hook_quant_decode` / `tensor_decode_outerdim`
 * (`runtime.py:93-119`, `basic_op.py:146-176`): out = f32(code / (2^bit - 1)) * scale + shift
 * (float64 divide rounded to f32, then two fp32 roundings). out f32 [items, n]. */
int pe_quant_decode(const void* codes, int items, size_t n, int bit, const void* scale, const void* shift, void* out,
                    void* stream);
/* The Lambert-W clamp factor `_clamp_factor_{laplace,gelu}` (`clamp_op.py:6-8,22-24`), as f32. */
float pe_quant_clamp_factor(int bit, int gelu);

/* ---- Stage executor ---------------------------------------------------------------------------
 * Replaces `{ViT,DeiT,Bert}ModelShard.forward`'s loop over `{ViT,DeiT,Bert}LayerShard.forward`
 * (`vit.py:161-170`, `deit.py:158-167`, `bert.py:142-151`) for the encoder blocks of one stage.
 * Embeddings / final LayerNorm / pooler / classifier are separate calls (pe_* above) driven by the
 * Python shard class. */
typedef struct pe_block_weights {
  /* f16 matrices in `nn.Linear.weight` layout [out, in]; f32 vectors. NULL for sub-layers this stage
   * does not own. */
  const void* w_qkv;  /* [3H, H] rows = [Wq; Wk; Wv] */
  const void* b_qkv;  /* [3H] */
  const void* w_o;    /* [H, H] */
  const void* b_o;    /* [H] */
  const void* w_fc1;  /* [I, H] */
  const void* b_fc1;  /* [I] */
  const void* w_fc2;  /* [H, I] */
  const void* b_fc2;  /* [H] */
  const void* ln1_w;  /* pre-LN: LayerNorm_before; post-LN: attention.output.LayerNorm */
  const void* ln1_b;
  const void* ln2_w;  /* pre-LN: LayerNorm_after;  post-LN: output.LayerNorm */
  const void* ln2_b;
} pe_block_weights;

typedef struct pe_stage_desc {
  int family;      /* PE_FAMILY_* */
  int hidden;      /* H */
  int heads;
  int inter;       /* I */
  int tokens;      /* S: tokens per item */
  float eps;
  int layer_start; /* 1-based inclusive sub-layer range, as `ModuleShardConfig` (`models/__init__.py:9-22`) */
  int layer_end;
  int max_ubatch;  /* workspace is sized for this many items */
} pe_stage_desc;

typedef struct pe_stage pe_stage;

/* `blocks` has one entry per transformer block touched by [layer_start, layer_end], first to last. */
int pe_stage_create(const pe_stage_desc* desc, const pe_block_weights* blocks, int n_blocks, pe_stage** out);
int pe_stage_destroy(pe_stage* stage);
/* Payloads follow SURVEY.md 8a-A2. in0/out0: f32 [ubatch, S, H] (or [ubatch, S, I] after sub-layer 2);
 * in1/out1: the f32 skip tensor of a tuple payload, NULL otherwise. out0 may alias in0 only when the
 * stage starts and ends on block boundaries. If `use_graph` != 0 the kernel sequence for this
 * (ubatch, pointers) tuple is captured into a CUDA graph on first use and replayed afterwards. */
int pe_stage_forward(pe_stage* stage, const void* in0, const void* in1, void* out0, void* out1, int ubatch,
                     int use_graph, void* stream);
/* OR-able into `use_graph` (eager launches only, i.e. bit 0 clear): a stage that ends on an output projection / FC2
 * (`vit.py:62-64,69`) leaves its final residual add to the consumer; pe_stage_deferred then returns the two addends
 * (f32 [ubatch, S, H] each, library / caller owned, valid until the next forward), or NULLs when nothing was deferred
 * and the result is in out0 as usual. The link's send kernel (pe_link_put) adds while it reads. */
#define PE_STAGE_DEFER_ADD 2
int pe_stage_deferred(const pe_stage* stage, const void** a, const void** b);
/* One EAGER forward with a CUDA event after every kernel: ms_out[i] = device time of kernel i,
 * kinds_out[i] = PE_KERNEL_* (up to `capacity` entries, *n_out = kernels launched). Synchronises `stream`. */
#define PE_KERNEL_CAST 0
#define PE_KERNEL_LAYERNORM 1
#define PE_KERNEL_GEMM_QKV 2
#define PE_KERNEL_ATTENTION 3
#define PE_KERNEL_GEMM_OUT 4
#define PE_KERNEL_GEMM_FC1 5
#define PE_KERNEL_GEMM_FC2 6
int pe_stage_profile(pe_stage* stage, const void* in0, const void* in1, void* out0, void* out1, int ubatch,
                     void* stream, float* ms_out, int* kinds_out, int capacity, int* n_out);
/* Number of kernels one pe_stage_forward enqueues for `ubatch` items (for bench.py's gpu_launches). */
int pe_stage_kernel_count(const pe_stage* stage);

/* ---- Stage-0 edges (SURVEY.md 8a-A13) ------------------------------------------------------------
 * pe_patch_embed replaces HF `ViTEmbeddings` / `DeiTEmbeddings` as used at `vit.py:96,165`, `deit.py:95,161`:
 * Conv2d(C, H, P, stride P) as an im2col + wgmma GEMM whose epilogue adds the conv bias and position
 * rows and scatters into token rows n_prefix.. of each item; rows 0..n_prefix-1 are copied from `prefix`.
 *   pixels f32 [B, C, img, img]; w f16 [H, kpad] (Conv2d weight flattened [H, C*P*P], zero-padded to
 *   kpad = roundup(C*P*P, 8)); bias f32 [H]; pos f32 [S, H] with S = (img/P)^2 + n_prefix;
 *   prefix f32 [n_prefix, H] = cls (and distillation) token + their position rows;
 *   out f32 [B, S, H]; patches_work f16 [B * (img/P)^2, kpad] scratch. */
int pe_patch_embed(const void* pixels, const void* w, const void* bias, const void* pos, const void* prefix, void* out,
                   void* patches_work, int batch, int channels, int img, int patch, int hidden, int n_prefix,
                   void* stream);
/* pe_bert_embed replaces HF `BertEmbeddings` (eval mode) as used at `bert.py:78,146`:
 * out = LayerNorm(word[ids] + type0 + pos[pos_ids[s]]).  ids i64 [B, S]; pos_ids i64 [S];
 * word f32 [V, H]; type0 f32 [H] (token type 0 row); pos f32 [P, H]; out f32 [B, S, H]. */
int pe_bert_embed(const void* ids, const void* pos_ids, const void* word, const void* type0, const void* pos,
                  const void* gamma, const void* beta, float eps, void* out, int batch, int seq, int hidden,
                  void* stream);

/* ---- Peer-memory links: the inter-stage hop as NVLink stores + device-polled flags -------------------
 * Replaces `TensorSendThread.run` / `TensorRecvThread.run` + `_send_tensor` / `_recv_tensor`
 * (`p2p/__init__.py:96-258`) and, on quantised hops, `forward_hook_quant_encode` /
 * `forward_pre_hook_quant_decode` (`runtime.py:73-119`) around them. A link is a ring of slots in the CONSUMER's
 * HBM, mapped into the producer with cudaIpc; per slot a `full` counter (raised by the producer's kernel after its
 * stores) and a `free` counter (raised by the consumer's kernel after its reads), both polled on the devices. The
 * kernels find their slot through device-resident sequence counters, so they take no per-payload arguments and a
 * stage's get -> blocks -> put sequence replays as one CUDA graph. Host side: one 16-byte ticket per payload on the
 * hop's Unix-domain socket `fd` (owned by the caller). Wire format per tensor: f32 values (f16 with
 * PIPEEDGE_WIRE_F16=1) or, for bit > 0, the reference's packed codes (`basic_op.py:38-55`: floor(32/bit) codes per
 * little-endian uint32, LSB first) + per-item f32 scale / shift in the slot header. */
typedef struct pe_link pe_link;
/* Peer link over `fd`; blocks until the other end has called it too. The producer picks the geometry
 * (`slot_payload_bytes` per slot, `n_slots` in [2,8]) and announces the QuantPipe bit-width it expects to send
 * (`quant_hint`, 0 = raw; it only sizes the consumer's receive grid - every payload describes itself); the consumer
 * passes 0, 0, 0. */
int pe_link_open(int fd, int is_producer, size_t slot_payload_bytes, int n_slots, int quant_hint, pe_link** out);
/* Both ends in this process (one-rank pipelines, tests). */
int pe_link_open_local(size_t slot_payload_bytes, int n_slots, int quant_hint, pe_link** out);
/* Consumer end fed by the host with pe_link_feed (the data rank's inputs, `devices.forward_pre_hook_to_device`). */
int pe_link_open_host(size_t slot_payload_bytes, int n_slots, pe_link** out);
int pe_link_close(pe_link* link);
size_t pe_link_slot_bytes(const pe_link* link);
/* Producer: ship a payload of one or two tensors, x_i = a_i (+ b_i), each f32 [items, n_i]; a1 == NULL for one tensor.
 * bit == 0: raw values; bit in [1,16]: QuantPipe (`clamp` = PE_CLAMP_*). For bit in {2,4,8,16} and n % 16 == 0 this
 * is ONE kernel per tensor: statistics -> grid barrier -> thresholds -> quantise + pack + peer stores, the fp32 slice
 * held in shared memory in between; other widths run the stand-alone quant kernels and one shipping kernel. */
int pe_link_put(pe_link* link, const void* a0, const void* b0, size_t n0, const void* a1, const void* b1, size_t n1,
                int items, int bit, int clamp, void* stream);
/* The fused encode-and-send of one tensor under the name SURVEY.md 8(b) gives it (= pe_link_put with bit > 0). */
int pe_quant_encode_send(pe_link* link, const void* x, const void* skip, int items, size_t n, int bit, int clamp,
                         void* stream);
/* Consumer: wait for the next payload (on the device), copy / dequantise (`tensor_decode_outerdim`,
 * `basic_op.py:146-176`) it into dst0 (/ dst1) as f32 [items, n0] (/ [items, n1]) and release the slot. The payload's
 * description must match (items, n0, n1) or the kernel traps and pe_link_check reports it. */
int pe_link_get(pe_link* link, void* dst0, void* dst1, int items, size_t n0, size_t n1, void* stream);
int pe_link_get_raw(pe_link* link, void* dst, size_t bytes, void* stream);   /* host-fed links */
/* Host-fed link: copy the next payload into the ring on `copy_stream` (blocks on the host while the ring is full). */
int pe_link_feed(pe_link* link, const void* src, size_t bytes, int src_is_host, void* copy_stream);
int pe_link_ticket_send(pe_link* link, long long a, long long b);
int pe_link_ticket_recv(pe_link* link, long long* out2);   /* blocks; 1 = the peer closed */
int pe_link_check(pe_link* link);                          /* PE_OK, or the protocol error a link kernel reported */
int pe_link_debug_read(pe_link* link, unsigned long long seq, size_t offset, void* host_dst, size_t bytes);
#define PE_LINK_HEADER_BYTES 16384   /* slot = [header | payload]; scale f32[512] of tensor t at 256 + 4096 t, shift 2048 later */

/* ---- Host rings: the hops of a data rank without a GPU ------------------------------------------------
 * A data rank outside the stage pipeline that has no CUDA device (`runtime.py -d cpu`, or no visible GPU) moves its
 * inputs and results through rings in POSIX shared memory that it creates: R slots of [16 KiB header | payload] and a
 * monotonic full[s] / free[s] counter pair per slot, both in the segment (4 KiB of counters, then the slots). A
 * producer publishes a slot's k-th use with a release store full[s] = k + 1 and a ticket {items, dim1} on the hop's
 * socket; the consumer acquires full[s], checks the header and releases the slot with a release store free[s] = k + 1.
 * Every wait is bounded by PIPEEDGE_LINK_TIMEOUT_S. The segment is named by the caller (`/name`, at most 62 more
 * characters) and unlinked as soon as both ends have mapped it or the handshake failed.
 *
 * Host-only entry points (pe_hostring_*) never touch the CUDA runtime. The stage at the other end of such a hop opens
 * it with pe_link_open as usual: the handshake tells it that the peer is a host ring, and it maps the segment and
 * registers it with CUDA (cudaHostRegisterMapped | Portable). A last stage's send kernel then stores raw f32 results
 * straight into the mapped slots; a first stage waits for each input with pe_link_shm_wait, feeds it to its host-fed
 * ring with pe_pipe_submit (a copy-engine transfer out of the registered slot) and hands the slot back with
 * pe_link_shm_release. */
typedef struct pe_hostring pe_hostring;
/* Data rank: create the segment `name` for the hop on `fd` and hand it to the stage. Producer (inputs): the geometry is
 * `slot_payload_bytes` per slot and `n_slots` in [2,8]. Consumer (results): pass 0, 0; the last stage's hello names it. */
int pe_hostring_create(int fd, const char* name, int is_producer, size_t slot_payload_bytes, int n_slots,
                       pe_hostring** out);
/* The stage's side of pe_hostring_create without a GPU (tests; what pe_link_open does less the CUDA registration). */
int pe_hostring_attach(int fd, int is_producer, size_t slot_payload_bytes, int n_slots, pe_hostring** out);
int pe_hostring_close(pe_hostring* ring);   /* unmaps; `fd` stays the caller's */
size_t pe_hostring_slot_bytes(const pe_hostring* ring);
/* Producer: wait for a free slot, write a raw header and `bytes` of payload, publish it and send the ticket
 * {items, dim1}. A payload larger than a slot is refused before anything is written. */
int pe_hostring_publish(pe_hostring* ring, const void* data, size_t bytes, int items, long long dim1);
int pe_hostring_close_input(pe_hostring* ring);   /* producer: the closing ticket */
/* Consumer: the next ticket (blocks; 1 = the producer closed), then its payload - the header must name `items` and
 * `bytes` (a raw payload, or one raw f32 tensor of items x n values) - valid until pe_hostring_release. */
int pe_hostring_next(pe_hostring* ring, long long* ticket2);
int pe_hostring_wait(pe_hostring* ring, int items, size_t bytes, const void** data);
int pe_hostring_release(pe_hostring* ring);
/* The stage's end of a host ring (a pe_link from pe_link_open whose peer is a data rank without a GPU). */
int pe_link_is_shm(const pe_link* link);
/* First stage: wait on the host for the payload the last ticket (pe_link_ticket_recv) announced; *src = the payload in
 * registered host memory, a pinned source for pe_pipe_submit. */
int pe_link_shm_wait(pe_link* link, int items, size_t bytes, const void** src);
/* ... then hand its slot back behind the copy on `stream` (the pipe's copy stream): a one-thread kernel stores free[s]
 * with st.release.sys into mapped host memory. */
int pe_link_shm_release(pe_link* link, void* stream);

/* ---- Per-rank stage loop ---------------------------------------------------------------------------
 * Replaces `TensorWorkThread.run` and the queue hand-offs of `DistP2pPipelineStage` (`p2p/__init__.py:261-295,
 * 373-394,442-450`): a stage's micro-batch (link get -> kernels -> link put) is captured once into a CUDA graph;
 * per micro-batch the host reads a ticket, launches the graph and writes a ticket - in C, GIL released. */
typedef struct pe_pipe pe_pipe;
int pe_pipe_create(pe_link* in, pe_link* out, pe_link* res, pe_pipe** out_pipe);
int pe_pipe_destroy(pe_pipe* pipe);
void* pe_pipe_stream(pe_pipe* pipe);
void* pe_pipe_copy_stream(pe_pipe* pipe);
int pe_pipe_has_graph(pe_pipe* pipe, int ubatch, long long dim1);
/* Graphs are filed per (ubatch, dim1, send bit-width): pe_pipe_capture_end's `bit`. The send bit-width set here picks the
 * variant that pe_pipe_run / pe_pipe_submit launch and pe_pipe_has_graph reports, from the next launch on (an atomic
 * store, legal while another thread runs the pipe). A bit-width without a graph for a payload's shape makes pe_pipe_run
 * ask for a capture instead of launching another variant. -1, the initial value: each shape's most recent capture, and
 * while it is in force a capture replaces the shape's graph of any other bit-width - a pipe that never calls this keeps
 * and launches exactly what it did before. Set a bit-width before capturing to keep one graph per bit-width. */
int pe_pipe_set_send_bit(pe_pipe* pipe, int bit);
/* Whether the graph of (ubatch, dim1) for send bit-width `bit` is captured (with the stamps setting now in force). */
int pe_pipe_has_variant(pe_pipe* pipe, int ubatch, long long dim1, int bit);
/* Capture for buffer parity 0 (and, with an overlapped send, 1): begin enqueues the receive into dst0 / dst1, the caller
 * then enqueues the stage's kernels on pe_pipe_stream(), end adds the send - inside the same graph (overlap == 0) or as
 * a graph of its own on a second stream that overlaps the NEXT micro-batch's receive and first kernels (overlap != 0:
 * the stage must write its output into a different buffer set per parity; micro-batch i uses parity i mod 2). */
/* raw_bytes > 0 on a hop input: the first stage fed by a data rank outside the stage pipeline - the relayed input
 * (pe_pipe_capture_relay) lands unchanged in dst0, after its header was checked against raw_bytes and ubatch. */
int pe_pipe_capture_begin(pe_pipe* pipe, int ubatch, long long dim1, int parity, void* dst0, void* dst1, size_t n0,
                          size_t n1, size_t raw_bytes);
/* Data rank outside the stage pipeline (pe_pipe_create(host-fed link, producer end of the hop to the first stage,
 * consumer end of the hop from the last stage)): capture the graph that relays each input micro-batch of `ubatch` items
 * and `bytes` bytes from the host-fed ring into the first stage's ring (one kernel; plus two stamp kernels with stamps
 * on), filed as (ubatch, dim1, bit-width 0). pe_pipe_submit, pe_pipe_close_input, pe_pipe_next_result and pe_pipe_sync
 * then work as for a data rank that owns the first stage. */
int pe_pipe_capture_relay(pe_pipe* pipe, int ubatch, long long dim1, size_t bytes, int* kernels);
int pe_pipe_capture_end(pe_pipe* pipe, const void* a0, const void* b0, size_t n0, const void* a1, const void* b1,
                        size_t n1, int items, int bit, int clamp, int overlap, int* kernels);
int pe_pipe_capture_abort(pe_pipe* pipe);
int pe_pipe_invalidate(pe_pipe* pipe);
int pe_pipe_submit(pe_pipe* pipe, const void* src, size_t bytes, int src_is_host, int ubatch, long long dim1);
int pe_pipe_close_input(pe_pipe* pipe);
int pe_pipe_run(pe_pipe* pipe, long long* need2);   /* 1 = closed, 2 = graph needed for need2 = {ubatch, dim1} */
int pe_pipe_set_out_dim(pe_pipe* pipe, long long n);   /* last stage: result elements per item, sent with its tickets */
int pe_pipe_next_result(pe_pipe* pipe, void** host_ptr, int* items, size_t* n);   /* 1 = closed */
int pe_pipe_sync(pe_pipe* pipe);
int pe_pipe_timing_reset(pe_pipe* pipe);
int pe_pipe_timing(pe_pipe* pipe, float* compute_ms, float* results_ms, unsigned long long* launches,
                   unsigned long long* kernels);

/* Per-micro-batch device timestamps. With stamps on, graphs captured from then on carry one-thread kernels that read
 * %globaltimer (ns) into a ring of PE_PIPE_STAMP_DEPTH records in mapped host memory; the graphs still take no per-launch
 * arguments (device-resident counters pick the record). Turning them on or off makes every graph captured the other
 * way count as missing: the next payload of its shape captures again. Graphs captured without stamps are exactly the
 * graphs of a pipe that never had them. */
#define PE_PIPE_STAMP_DEPTH 256
#define PE_STAMP_OVERLAPPED 1   /* the send ran as its own graph, overlapping the next micro-batch */
#define PE_STAMP_FUSED 2        /* a tensor went through the fused quantise-and-send kernel */
#define PE_STAMP_STAGED 4       /* a tensor went through the stand-alone encode kernels + a shipping kernel */
typedef struct pe_pipe_record {
  unsigned long long index;        /* records of this pipe before this one */
  unsigned long long t_start;      /* graph start, before the receive */
  unsigned long long t_got;        /* receive (and dequantise) done */
  unsigned long long t_stage;      /* the stage's last kernel done */
  unsigned long long t_send_start; /* send start (= t_stage when the send is inside the main graph) */
  unsigned long long t_encoded;    /* staged send: its stand-alone encode kernels done; else 0 */
  unsigned long long t_send_end;   /* send done: the payload is published to the consumer */
  unsigned long long bytes_out;    /* payload bytes the send wrote (pe_link_payload_bytes, summed over its tensors) */
  int items;                       /* micro-batch size */
  int bit_out;                     /* bit-width the send quantised to (0 = raw values) */
  int bit_in;                      /* bit-width of the payload the receive consumed, from its slot header; -1: host-fed */
  int flags;                       /* PE_STAMP_* */
} pe_pipe_record;
int pe_pipe_enable_stamps(pe_pipe* pipe, int on);
/* Non-blocking: copy up to `max` records completed since the previous call into `out` (oldest first; *n of them) and add
 * to *dropped the records that were overwritten before they could be read (a reader a whole ring behind). */
int pe_pipe_drain_stamps(pe_pipe* pipe, pe_pipe_record* out, int max, int* n, unsigned long long* dropped);

/* ---- Inter-stage hop over NCCL (generic payloads) -----------------------------------------------
 * Replaces `TensorSendThread.run` / `TensorRecvThread.run` + `_send_tensor` / `_recv_tensor`
 * (`p2p/__init__.py:96-258`) for the device tensors of a payload: one call per payload and side, over a
 * dedicated 2-rank NCCL communicator per directed hop; `fd` is the hop's connected Unix-domain socket (owned by
 * the caller) carrying the 16-byte envelope headers. Events are `cudaEvent_t`, streams `cudaStream_t`. */
typedef struct pe_hop pe_hop;
int pe_hop_available(void);
int pe_hop_open(int fd, int is_sender, pe_hop** out);
int pe_hop_close(pe_hop* hop);
int pe_hop_send(pe_hop* hop, const void* const* ptrs, const size_t* bytes, int n, void* ready_event, void* stream,
                void* done_event, int write_envelope);
int pe_hop_wait_envelope(pe_hop* hop, long long* head2);
int pe_hop_recv(pe_hop* hop, void* const* ptrs, const size_t* bytes, void* const* free_events, int n, void* stream,
                void* ready_event);

/* ---- Debug / bring-up ------------------------------------------------------------------------
 * Reference GEMM on CUDA cores (fp16 inputs, fp32 accumulate, same epilogues). Used ONLY by tests to
 * localise a failure to the wgmma kernel; never selected by the product path. */
int pe_debug_linear_simt(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n,
                         int k, int epilogue, void* stream);

/* While `buf` (device, >= 32 * 8 * grid bytes) is set, every pe_linear launch stores a per-CTA clock64 timeline
 * (start, setup done, first operands landed, last MMA issued, accumulator ready, epilogue done, exit, epilogue and
 * steady-state main-loop detail; 32 slots per CTA). Slots 2, 3 and 5 (first operands landed, last MMA retired, epilogue
 * done) are stamped for a CTA's first tile, slots 7, 8 and 10 the same for its second (scripts/gemm_phases.py). */
int pe_debug_gemm_trace(void* buf);

/* Host-only (no device needed): the tile plan and launch geometry pe_linear would use for an [m, k] x [n, k]^T product
 * with `epilogue`: out6 = {cluster_m, cluster_n, block_n, ring stages, tiles, CTAs}. */
int pe_debug_gemm_plan(int m, int n, int k, int epilogue, int* out6);

/* Host-only: how pe_link_put would ship one tensor of `items` x `n` f32 values at `bit` bits (`aligned`: its a / b are
 * 16-byte aligned) on the current device (132 SMs without one): out5 = {path, CTAs, chunks per item, elements per
 * chunk, slice cached}. FUSED = the one-kernel quantise-and-send; its CTA keeps its fp32 slice in shared memory when it
 * fits in 160 KiB (cached = 1), else pass 2 re-reads it from HBM. STAGED = stand-alone quant kernels + a copy kernel. */
#define PE_LINK_PATH_COPY 0
#define PE_LINK_PATH_FUSED 1
#define PE_LINK_PATH_STAGED 2
int pe_debug_link_put_plan(int items, size_t n, int bit, int aligned, int* out5);
/* Host-only: bytes a put of one [items, n] tensor at `bit` bits writes - the f32 values (f16 with `wire_f16`), or the
 * packed codes plus the per-item f32 scale and shift. With wire_f16 == 0 it equals what the Python-thread path moves for
 * the same tensor (its CUDA tensors: the values, or codes + scale + shift). 0 for invalid arguments. */
size_t pe_link_payload_bytes(int items, size_t n, int bit, int wire_f16);

#ifdef __cplusplus
}
#endif
#endif /* PIPEEDGE_B200_H */
