// Peer-memory links: the inter-stage hop as device-to-device stores over NVLink, synchronised by flags the GPUs
// themselves poll - no NCCL rendezvous kernel, no host round trip per payload.
//
// A link is a directed (producer -> consumer) ring of R slots that lives in the CONSUMER's HBM and is mapped into the
// producer's address space with cudaIpc (one process per GPU). Per slot there are two monotonic counters:
//   full[s]  in the consumer's memory, raised by the producer after the payload of the slot's k-th use has landed
//            (peer stores, __threadfence_system, st.release.sys);
//   free[s]  in the producer's memory, raised by the consumer once it has read that payload.
// Both sides poll LOCAL memory only. A slot is [16 KiB header (payload description, per-item scale / shift) | data].
//
//   put (producer stage's last kernel)   waits for free[s], writes header + data straight into the peer slot and raises
//                                        full[s]. With bit > 0 it is the fused QuantPipe kernel: statistics of a (+ b)
//                                        -> grid barrier -> clamp threshold, per-item scale / shift -> codes packed and
//                                        stored into the peer slot, the fp32 slice kept in shared memory in between;
//   get (consumer stage's first kernel)  waits for full[s], copies / dequantises the payload into the stage's fixed input
//                                        buffer, raises free[s];
//   relay (a data rank outside the       waits for its host-fed input slot and the first stage's free[s], copies the
//   stage pipeline: its whole graph)     input bytes unchanged into that slot behind a raw header, raises full[s] and
//                                        releases the host-fed slot.
// Which slot a kernel works on comes from a device-resident sequence counter, so the kernels take no per-payload
// arguments: a stage's whole micro-batch (get -> blocks -> put) is ONE CUDA graph replayed unchanged (pipe.cu).
// The host side of a link is only a "ticket" per payload on the hop's Unix-domain socket, telling the consumer's host
// loop that one more graph launch is due.
//
// Replaces TensorSendThread.run / TensorRecvThread.run + _send_tensor / _recv_tensor (p2p/__init__.py:96-258) and, for
// quantised hops, forward_hook_quant_encode / forward_pre_hook_quant_decode (runtime.py:73-119) around them.
#include <errno.h>
#include <sched.h>
#include <stdlib.h>
#include <string.h>
#include <sys/socket.h>
#include <time.h>
#include <unistd.h>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"
#include "link.cuh"
#include "quant_dev.cuh"

namespace pe {

void count_launches(int n);
int require_sm90();
int add_impl(const void* a, const void* b, void* out, size_t n, cudaStream_t stream);

constexpr int kPutThreads = 512;
constexpr int kGetThreads = 256;
constexpr size_t kQuantCacheBytes = 160 * 1024;   // fp32 slice a CTA of the fused kernel keeps between its two passes
constexpr int kFlagsBytes = 256;                  // R x 8 bytes, padded

// ------------------------------------------------------------------------------------------------ device helpers
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ uint64_t ld_acquire_sys(const uint64_t* p) {
  uint64_t v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_sys(uint64_t* p, uint64_t v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned ld_acquire_gpu_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fail(unsigned* status, unsigned code) {
  *reinterpret_cast<volatile unsigned*>(status) = code;
  __threadfence_system();
  __trap();
}
// Bounded: a protocol bug or a dead peer ends in a trap (the launch fails, the host sees an error), never in a hang.
// Between polls the back-off doubles from kMinNs up to kMaxNs.
template <unsigned kMinNs, unsigned kMaxNs>
__device__ __forceinline__ void spin_until_ge(const uint64_t* flag, uint64_t want, unsigned long long timeout_ns,
                                              unsigned* status, unsigned code) {
  if (ld_acquire_sys(flag) >= want) return;
  const unsigned long long t0 = globaltimer_ns();
  unsigned ns = kMinNs;
  while (ld_acquire_sys(flag) < want) {
    __nanosleep(ns);
    if (ns < kMaxNs) ns <<= 1;
    if (globaltimer_ns() - t0 > timeout_ns) {
      printf("pipeedge_b200: link wait timed out (code %u, block %d)\n", code, blockIdx.x);
      fail(status, code);
    }
  }
}

// ------------------------------------------------------------------------------------------------ get
struct GetArgs {
  LinkRx rx;
  void* dst0;
  void* dst1;
  size_t n0, n1;        // elements per item the stage expects (raw mode: n0 = bytes to copy)
  int items;
  int n_tensors;
  int raw;              // copy n0 bytes: 1 = host-fed link (no header), 2 = relayed raw payload (header checked)
  unsigned long long timeout_ns;
};

__device__ __forceinline__ LinkHeader load_header(const uint8_t* base) {
  LinkHeader h;
  const uint4* src = reinterpret_cast<const uint4*>(base);
  uint4* d = reinterpret_cast<uint4*>(&h);
#pragma unroll
  for (int i = 0; i < static_cast<int>(sizeof(LinkHeader) / 16); ++i) d[i] = __ldcg(src + i);
  return h;
}

// Grid-stride copy with kU independent 16-byte loads in flight per thread (a lone load per trip left these kernels
// latency-bound: ncu r02b measured 0.5 TB/s for a 4.8 MB payload).
template <typename Load, typename Store>
__device__ __forceinline__ void stream4(size_t n, size_t tid, size_t stride, Load load, Store store) {
  constexpr int kU = 4;
  size_t i = tid;
  for (; i + (kU - 1) * stride < n; i += kU * stride) {
    uint4 v[kU];
#pragma unroll
    for (int u = 0; u < kU; ++u) v[u] = load(i + u * stride);
#pragma unroll
    for (int u = 0; u < kU; ++u) store(i + u * stride, v[u]);
  }
  for (; i < n; i += stride) store(i, load(i));
}

__device__ void get_tensor(const uint8_t* slot, const LinkTensorHdr& th, int ti, int items, float* dst, float* lut) {
  const size_t n = th.n;
  const size_t total = static_cast<size_t>(items) * n;
  const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const uint8_t* data = slot + th.data_off;
  if (th.bit == 0) {
    if (th.dtype == 0) {
      const size_t n4 = total >> 2;
      const uint4* s4 = reinterpret_cast<const uint4*>(data);
      uint4* d4 = reinterpret_cast<uint4*>(dst);
      stream4(n4, tid, stride, [&](size_t i) { return __ldcg(s4 + i); }, [&](size_t i, uint4 v) { d4[i] = v; });
      for (size_t i = (n4 << 2) + tid; i < total; i += stride) dst[i] = __ldcg(reinterpret_cast<const float*>(data) + i);
    } else {
      const size_t n8 = total >> 3;   // 8 halves (16 bytes) in, 32 bytes out
      const uint4* s4 = reinterpret_cast<const uint4*>(data);
      stream4(n8, tid, stride, [&](size_t i) { return __ldcg(s4 + i); },
              [&](size_t i, uint4 v) {
                const __half2* h = reinterpret_cast<const __half2*>(&v);
                const float2 a = __half22float2(h[0]), b = __half22float2(h[1]), c = __half22float2(h[2]), d = __half22float2(h[3]);
                reinterpret_cast<float4*>(dst)[2 * i] = make_float4(a.x, a.y, b.x, b.y);
                reinterpret_cast<float4*>(dst)[2 * i + 1] = make_float4(c.x, c.y, d.x, d.y);
              });
      for (size_t i = (n8 << 3) + tid; i < total; i += stride) dst[i] = __half2float(reinterpret_cast<const __half*>(data)[i]);
    }
    return;
  }
  // QuantPipe decode (tensor_decode_outerdim, basic_op.py:146-176)
  const QDecoder dec = fill_dequant_lut(lut, static_cast<int>(th.bit));
  const int ratio = dec.ratio;
  const float* scale = reinterpret_cast<const float*>(slot + kLinkScaleOff + static_cast<size_t>(ti) * 4096);
  const float* shift = scale + kLinkMaxItems;
  const size_t wpi = (n + ratio - 1) / ratio;
  const size_t words = static_cast<size_t>(items) * wpi;
  const uint32_t* codes = reinterpret_cast<const uint32_t*>(data);
  if ((ratio % 4 == 0) && (n % ratio == 0) && (wpi % 4 == 0) && words < (1ull << 32)) {
    // fast path: a thread turns 16 bytes of codes (4 words) into 4 * ratio values; 32-bit index arithmetic
    const uint32_t wpi4 = static_cast<uint32_t>(wpi >> 2), total4 = static_cast<uint32_t>(words >> 2);
    const uint4* c4 = reinterpret_cast<const uint4*>(codes);
    constexpr int kU = 2;
    const uint32_t t32 = static_cast<uint32_t>(tid), s32 = static_cast<uint32_t>(stride);
    for (uint32_t g0 = t32; g0 < total4; g0 += kU * s32) {
      uint4 w[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u)
        if (g0 + u * s32 < total4) w[u] = __ldcg(c4 + g0 + u * s32);
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const uint32_t g = g0 + u * s32;
        if (g >= total4) break;
        const uint32_t item = g / wpi4, in_item = g - item * wpi4;
        const float sc = __ldcg(scale + item), sh = __ldcg(shift + item);
        float* oi = dst + static_cast<size_t>(item) * n + static_cast<size_t>(in_item) * 4 * ratio;
        const uint32_t ww[4] = {w[u].x, w[u].y, w[u].z, w[u].w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          for (int j = 0; j < ratio; j += 4) {
            float v[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) v[q] = dec.value(ww[k], j + q, sc, sh);
            *reinterpret_cast<float4*>(oi + k * ratio + j) = make_float4(v[0], v[1], v[2], v[3]);
          }
        }
      }
    }
    return;
  }
  for (size_t w = tid; w < words; w += stride) {
    const size_t item = w / wpi;
    const size_t wi = w - item * wpi;
    const uint32_t word = __ldcg(codes + w);
    const float sc = __ldcg(scale + item), sh = __ldcg(shift + item);
    dec.word(word, wi * ratio, n, sc, sh, dst + item * n + wi * ratio);
  }
}

// The wait itself: ONE warp, no shared memory, long back-off. A consumer may sit here for a whole pipeline latency (the
// data rank waiting for a result) while the same GPU runs another stream's GEMMs, which need every SM's entire shared
// memory: a waiting CTA that held shared memory (or many waiting CTAs) would push a GEMM CTA into a second wave.
__global__ void __launch_bounds__(32) link_wait_kernel(const LinkRx rx, unsigned long long timeout_ns) {
  if (threadIdx.x == 0) {
    const uint64_t seq = *reinterpret_cast<volatile uint64_t*>(rx.seq);
    const uint64_t slot = seq % static_cast<uint64_t>(rx.n_slots), k = seq / static_cast<uint64_t>(rx.n_slots);
    spin_until_ge<64, 2048>(rx.full + slot, k + 1, timeout_ns, rx.status, kLinkErrWaitFull);
  }
}

__global__ void __launch_bounds__(kGetThreads) link_get_kernel(const GetArgs g) {
  extern __shared__ float get_lut[];
  __shared__ uint64_t s_seq;
  if (threadIdx.x == 0) {
    const uint64_t seq = *reinterpret_cast<volatile uint64_t*>(g.rx.seq);
    const uint64_t slot = seq % static_cast<uint64_t>(g.rx.n_slots), k = seq / static_cast<uint64_t>(g.rx.n_slots);
    spin_until_ge<32, 512>(g.rx.full + slot, k + 1, g.timeout_ns, g.rx.status, kLinkErrWaitFull);
    s_seq = seq;
  }
  __syncthreads();
  const uint64_t seq = s_seq;
  const uint64_t slot = seq % static_cast<uint64_t>(g.rx.n_slots), k = seq / static_cast<uint64_t>(g.rx.n_slots);
  const uint8_t* base = g.rx.ring + slot * g.rx.slot_bytes;
  if (g.raw) {
    if (g.raw == 2) {
      const LinkHeader h = load_header(base);
      if (h.magic != kLinkMagic || h.n_tensors != kLinkRawKind || h.t[0].dtype != kLinkDtypeBytes ||
          h.items != static_cast<uint32_t>(g.items) || h.t[0].n != g.n0) {
        if (threadIdx.x == 0)
          printf("pipeedge_b200: raw payload mismatch: magic %x kind %u items %u bytes %llu (expected %d / %llu)\n",
                 h.magic, h.n_tensors, h.items, static_cast<unsigned long long>(h.t[0].n), g.items,
                 static_cast<unsigned long long>(g.n0));
        fail(g.rx.status, kLinkErrHeader);
      }
    }
    const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
    const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
    const uint8_t* data = base + kLinkHeaderBytes;
    const size_t n16 = g.n0 >> 4;
    const uint4* s4 = reinterpret_cast<const uint4*>(data);
    uint4* d4 = reinterpret_cast<uint4*>(g.dst0);
    stream4(n16, tid, stride, [&](size_t i) { return __ldcg(s4 + i); }, [&](size_t i, uint4 v) { d4[i] = v; });
    for (size_t i = (n16 << 4) + tid; i < g.n0; i += stride)
      reinterpret_cast<uint8_t*>(g.dst0)[i] = __ldcg(data + i);
  } else {
    const LinkHeader h = load_header(base);
    const bool ok = h.magic == kLinkMagic && h.n_tensors == static_cast<uint32_t>(g.n_tensors) &&
                    h.items == static_cast<uint32_t>(g.items) && h.t[0].n == g.n0 &&
                    (g.n_tensors < 2 || h.t[1].n == g.n1);
    if (!ok) {
      if (threadIdx.x == 0)
        printf("pipeedge_b200: link payload mismatch: magic %x tensors %u items %u n0 %llu (expected %d / %d / %llu)\n",
               h.magic, h.n_tensors, h.items, static_cast<unsigned long long>(h.t[0].n), g.n_tensors, g.items,
               static_cast<unsigned long long>(g.n0));
      fail(g.rx.status, kLinkErrHeader);
    }
    get_tensor(base, h.t[0], 0, g.items, static_cast<float*>(g.dst0), get_lut);
    if (g.n_tensors > 1) {
      __syncthreads();   // the LUT may be rebuilt for a different bit-width
      get_tensor(base, h.t[1], 1, g.items, static_cast<float*>(g.dst1), get_lut);
    }
  }
  // every CTA has finished reading -> hand the slot back to the producer. One GPU-scope fence per CTA, after its barrier
  // (the fence is cumulative over what the barrier ordered before it); the CTA that arrives last releases the slot with
  // a system-scope fence and st.release.sys, which are cumulative over everything the arrival counter ordered before
  // them. A system-scope fence in every thread made these kernels 3-4x longer than their copy (ncu r02c), and one in
  // every CTA makes each CTA wait for its own accesses to become visible system-wide.
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(g.rx.done_ctr, 1u);
    if (prev == gridDim.x - 1) {
      *g.rx.done_ctr = 0;
      *reinterpret_cast<volatile uint64_t*>(g.rx.seq) = seq + 1;
      __threadfence_system();
      st_release_sys(g.rx.free_ + slot, k + 1);
    }
  }
}

// ------------------------------------------------------------------------------------------------ put
struct PutArgs {
  LinkTx tx;
  PutTensor t;
  int ti, n_tensors, items;
  int bit, clamp;
  int wire_f16;
  int is_last;            // this launch completes the payload: raise full[s], advance the sequence
  uint64_t data_off;
  float factor_laplace, factor_gelu;
  int chunks;             // fused quantise: segments per item
  size_t per;             // ... elements per segment (multiple of 16)
  int cache;              // ... keep the fp32 slice in shared memory between the passes
  unsigned long long timeout_ns;
  // staged path (generic bit-widths): codes / scale / shift already computed into local memory
  const uint8_t* staged_codes;
  const float* staged_scale;
  const float* staged_shift;
  const float* staged_alpha;
  size_t staged_bytes;
};

__device__ __forceinline__ void put_begin(const PutArgs& p, uint64_t* s_seq) {
  if (threadIdx.x == 0) {
    const uint64_t seq = *reinterpret_cast<volatile uint64_t*>(p.tx.seq);
    const uint64_t slot = seq % static_cast<uint64_t>(p.tx.n_slots), k = seq / static_cast<uint64_t>(p.tx.n_slots);
    spin_until_ge<32, 512>(p.tx.free_ + slot, k, p.timeout_ns, p.tx.status, kLinkErrWaitFree);   // (k-1)-th use consumed
    *s_seq = seq;
  }
  __syncthreads();
}

__device__ __forceinline__ void put_header(const PutArgs& p, uint8_t* base, float alpha) {
  LinkHeader* h = reinterpret_cast<LinkHeader*>(base);
  if (p.ti == 0) {
    h->magic = kLinkMagic;
    h->n_tensors = static_cast<uint32_t>(p.n_tensors);
    h->items = static_cast<uint32_t>(p.items);
    h->pad = 0;
  }
  LinkTensorHdr th;
  th.bit = static_cast<uint32_t>(p.bit);
  th.dtype = (p.bit == 0 && p.wire_f16) ? 1u : 0u;
  th.n = p.t.n;
  th.data_off = p.data_off;
  th.alpha = alpha;
  th.pad = 0;
  h->t[p.ti] = th;
}

__device__ __forceinline__ void put_end(const PutArgs& p, uint64_t seq) {
  // this CTA's peer stores are ordered before its arrival (barrier, then ONE GPU-scope fence); the last CTA to arrive
  // publishes the slot with a system-scope fence and st.release.sys, cumulative over what the arrival counter ordered
  // before them (see the end of link_get_kernel)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(p.tx.done_ctr, 1u);
    if (prev == gridDim.x - 1) {
      *p.tx.done_ctr = 0;
      if (p.is_last) {
        const uint64_t slot = seq % static_cast<uint64_t>(p.tx.n_slots), k = seq / static_cast<uint64_t>(p.tx.n_slots);
        *reinterpret_cast<volatile uint64_t*>(p.tx.seq) = seq + 1;
        __threadfence_system();
        st_release_sys(p.tx.full + slot, k + 1);
      }
    }
  }
}

// bit == 0: payload = a (+ b) as f32 (or f16 on the wire)
__global__ void __launch_bounds__(kPutThreads) link_put_copy_kernel(const PutArgs p) {
  __shared__ uint64_t s_seq;
  put_begin(p, &s_seq);
  const uint64_t seq = s_seq;
  uint8_t* base = p.tx.ring + (seq % static_cast<uint64_t>(p.tx.n_slots)) * p.tx.slot_bytes;
  if (blockIdx.x == 0 && threadIdx.x == 0) put_header(p, base, INFINITY);
  const size_t total = static_cast<size_t>(p.items) * p.t.n;
  const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t n4 = total >> 2;
  const float4* a4 = reinterpret_cast<const float4*>(p.t.a);
  const float4* b4 = reinterpret_cast<const float4*>(p.t.b);
  uint8_t* data = base + p.data_off;
  {
    constexpr int kU = 4;   // independent loads in flight per thread (see stream4)
    for (size_t i0 = tid; i0 < n4; i0 += kU * stride) {
      float4 va[kU], vb[kU];
#pragma unroll
      for (int u = 0; u < kU; ++u)
        if (i0 + u * stride < n4) va[u] = a4[i0 + u * stride];
      if (b4 != nullptr) {
#pragma unroll
        for (int u = 0; u < kU; ++u)
          if (i0 + u * stride < n4) vb[u] = b4[i0 + u * stride];
      }
#pragma unroll
      for (int u = 0; u < kU; ++u) {
        const size_t i = i0 + u * stride;
        if (i >= n4) break;
        float4 v = va[u];
        if (b4 != nullptr) { v.x += vb[u].x; v.y += vb[u].y; v.z += vb[u].z; v.w += vb[u].w; }
        if (p.wire_f16) {
          uint2 pk;
          *reinterpret_cast<__half2*>(&pk.x) = __floats2half2_rn(v.x, v.y);
          *reinterpret_cast<__half2*>(&pk.y) = __floats2half2_rn(v.z, v.w);
          reinterpret_cast<uint2*>(data)[i] = pk;
        } else {
          reinterpret_cast<float4*>(data)[i] = v;
        }
      }
    }
  }
  for (size_t i = (n4 << 2) + tid; i < total; i += stride) {
    float v = p.t.a[i];
    if (p.t.b != nullptr) v += p.t.b[i];
    if (p.wire_f16) reinterpret_cast<__half*>(data)[i] = __float2half_rn(v);
    else reinterpret_cast<float*>(data)[i] = v;
  }
  put_end(p, seq);
}

// generic bit-widths: codes / scale / shift were produced by the stand-alone quant kernels into local memory
__global__ void __launch_bounds__(kPutThreads) link_put_staged_kernel(const PutArgs p) {
  __shared__ uint64_t s_seq;
  put_begin(p, &s_seq);
  const uint64_t seq = s_seq;
  uint8_t* base = p.tx.ring + (seq % static_cast<uint64_t>(p.tx.n_slots)) * p.tx.slot_bytes;
  if (blockIdx.x == 0) {
    if (threadIdx.x == 0) put_header(p, base, *p.staged_alpha);
    float* scale = reinterpret_cast<float*>(base + kLinkScaleOff + static_cast<size_t>(p.ti) * 4096);
    float* shift = scale + kLinkMaxItems;
    for (int i = threadIdx.x; i < p.items; i += blockDim.x) {
      scale[i] = p.staged_scale[i];
      shift[i] = p.staged_shift[i];
    }
  }
  const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t n4 = p.staged_bytes >> 2;   // whole uint32 words
  const uint32_t* src = reinterpret_cast<const uint32_t*>(p.staged_codes);
  uint32_t* dst = reinterpret_cast<uint32_t*>(base + p.data_off);
  for (size_t i = tid; i < n4; i += stride) dst[i] = src[i];
  put_end(p, seq);
}

// ---- the fused QuantPipe send: bit in {2, 4, 8, 16}, n % 16 == 0 ------------------------------------------------------
// Grid G <= SMs - 8, one CTA per SM (the fp32 slice lives in shared memory), all CTAs co-resident (grid barrier).
//   pass 1  x = a (+ b) for this CTA's (item, chunk) segments: min / max / sum / sum of squares (fp64) -> partials,
//           x kept in shared memory (XOR-swizzled float4s: conflict-free for both passes);
//   barrier
//   pass 2  every CTA reduces the partials in the same fixed order (= quant_finalize_kernel) -> alpha, scale, shift;
//           quantises its slice out of shared memory and stores the packed words into the peer's slot.
__device__ __forceinline__ uint32_t swz(uint32_t f) { return f ^ ((f >> 3) & 7u); }

template <int BIT>
__global__ void __launch_bounds__(kPutThreads, 1) link_put_quant_kernel(const PutArgs p) {
  extern __shared__ float4 cache4[];
  __shared__ uint64_t s_seq;
  __shared__ double red[kPutThreads / 32][kQPartialDoubles];
  __shared__ QStats s_item[kLinkMaxItems];
  __shared__ float s_alpha;
  constexpr int kWords = 16 * BIT / 32;
  constexpr int kRatio = 32 / BIT;

  put_begin(p, &s_seq);
  const uint64_t seq = s_seq;
  uint8_t* base = p.tx.ring + (seq % static_cast<uint64_t>(p.tx.n_slots)) * p.tx.slot_bytes;
  const int segs = p.items * p.chunks;
  const size_t n = p.t.n;
  const uint32_t per4 = static_cast<uint32_t>(p.per >> 2);

  // ---------------------------------------------------------------- pass 1
  int local = 0;
  for (int seg = blockIdx.x; seg < segs; seg += gridDim.x, ++local) {
    const int item = seg / p.chunks, chunk = seg - item * p.chunks;
    const size_t begin = static_cast<size_t>(chunk) * p.per;
    const size_t end = begin + p.per < n ? begin + p.per : n;
    QStats st = QStats::empty();
    if (begin < end) {
      const uint32_t len4 = static_cast<uint32_t>((end - begin) >> 2);
      const float4* a4 = reinterpret_cast<const float4*>(p.t.a + static_cast<size_t>(item) * n + begin);
      const float4* b4 = p.t.b != nullptr ? reinterpret_cast<const float4*>(p.t.b + static_cast<size_t>(item) * n + begin) : nullptr;
      const uint32_t off4 = static_cast<uint32_t>(local) * per4;
      constexpr int kU = 4;   // independent 16-byte loads in flight per thread and operand
      for (uint32_t i0 = threadIdx.x; i0 < len4; i0 += kU * kPutThreads) {
        float4 va[kU], vb[kU];
#pragma unroll
        for (int u = 0; u < kU; ++u)
          if (i0 + u * kPutThreads < len4) va[u] = a4[i0 + u * kPutThreads];
        if (b4 != nullptr) {
#pragma unroll
          for (int u = 0; u < kU; ++u)
            if (i0 + u * kPutThreads < len4) vb[u] = b4[i0 + u * kPutThreads];
        }
#pragma unroll
        for (int u = 0; u < kU; ++u) {
          const uint32_t i = i0 + u * kPutThreads;
          if (i >= len4) break;
          float4 v = va[u];
          if (b4 != nullptr) { v.x += vb[u].x; v.y += vb[u].y; v.z += vb[u].z; v.w += vb[u].w; }
          if (p.cache) cache4[swz(off4 + i)] = v;
          st.add(v);
        }
      }
    }
    stats_to_partial(st, red, p.tx.partials + static_cast<size_t>(seg) * kQPartialDoubles);
  }
  // ---------------------------------------------------------------- grid barrier
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();   // the partials written above (by thread 0 of this CTA) are visible before the arrival
    const unsigned gen = ld_acquire_gpu_u32(p.tx.bar_gen);
    const unsigned prev = atomicAdd(p.tx.bar_count, 1u);
    if (prev == gridDim.x - 1) {
      *p.tx.bar_count = 0;
      __threadfence();
      atomicAdd(p.tx.bar_gen, 1u);
    } else {
      const unsigned long long t0 = globaltimer_ns();
      while (ld_acquire_gpu_u32(p.tx.bar_gen) == gen) {
        __nanosleep(64);
        if (globaltimer_ns() - t0 > p.timeout_ns) fail(p.tx.status, kLinkErrBarrier);
      }
    }
  }
  __syncthreads();
  // ---------------------------------------------------------------- thresholds (same fixed order as quant_finalize_kernel)
  for (int i = threadIdx.x; i < p.items; i += kPutThreads) s_item[i] = fold_item<true>(p.tx.partials, i, p.chunks);
  __syncthreads();
  if (threadIdx.x == 0)
    s_alpha = fold_items_alpha(p.items, [&](int i) { return s_item[i]; }, n, p.clamp, p.factor_laplace, p.factor_gelu);
  __syncthreads();
  const float alpha = s_alpha;
  if (blockIdx.x == 0 && threadIdx.x == 0) put_header(p, base, alpha);
  float* scale_out = reinterpret_cast<float*>(base + kLinkScaleOff + static_cast<size_t>(p.ti) * 4096);
  float* shift_out = scale_out + kLinkMaxItems;
  // ---------------------------------------------------------------- pass 2
  const size_t wpi = n / kRatio;   // n % 16 == 0
  uint32_t* codes = reinterpret_cast<uint32_t*>(base + p.data_off);
  local = 0;
  for (int seg = blockIdx.x; seg < segs; seg += gridDim.x, ++local) {
    const int item = seg / p.chunks, chunk = seg - item * p.chunks;
    const size_t begin = static_cast<size_t>(chunk) * p.per;
    const size_t end = begin + p.per < n ? begin + p.per : n;
    float sc, sh;
    item_scale_shift(s_item[item].mn, s_item[item].mx, alpha, sc, sh);
    if (chunk == 0 && threadIdx.x == 0) {
      scale_out[item] = sc;
      shift_out[item] = sh;
    }
    if (begin >= end) continue;
    const uint32_t units = static_cast<uint32_t>((end - begin) >> 4);
    const uint32_t off4 = static_cast<uint32_t>(local) * per4;
    const float4* a4 = reinterpret_cast<const float4*>(p.t.a + static_cast<size_t>(item) * n + begin);
    const float4* b4 = p.t.b != nullptr ? reinterpret_cast<const float4*>(p.t.b + static_cast<size_t>(item) * n + begin) : nullptr;
    uint32_t* ci = codes + static_cast<size_t>(item) * wpi + (begin / kRatio);
    for (uint32_t u = threadIdx.x; u < units; u += kPutThreads) {
      float4 v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        if (p.cache) {
          v[j] = cache4[swz(off4 + 4 * u + j)];
        } else {
          v[j] = a4[4 * u + j];
          if (b4 != nullptr) {
            const float4 w = b4[4 * u + j];
            v[j].x += w.x; v[j].y += w.y; v[j].z += w.z; v[j].w += w.w;
          }
        }
      }
      pack16<BIT>(v, alpha, sh, sc).store(ci + static_cast<size_t>(u) * kWords);
    }
  }
  put_end(p, seq);
}

// ------------------------------------------------------------------------------------------------ relay
// The data rank outside the stage pipeline owns no shard: its graph is this one kernel, which moves the next input
// micro-batch from the host-fed ring (filled by link_feed on the copy stream) into the first stage's ring, with a raw
// header the first stage's receive checks. Both rings' sequence counters advance together (one relay per payload).
struct RelayArgs {
  LinkRx rx;              // host-fed ring of this device
  LinkTx tx;              // the first stage's ring (peer mapping)
  size_t bytes;
  int items;
  unsigned long long timeout_ns;
};

__global__ void __launch_bounds__(kPutThreads) link_relay_kernel(const RelayArgs r) {
  __shared__ uint64_t s_in, s_out;
  if (threadIdx.x == 0) {
    const uint64_t in_seq = *reinterpret_cast<volatile uint64_t*>(r.rx.seq);
    const uint64_t out_seq = *reinterpret_cast<volatile uint64_t*>(r.tx.seq);
    const uint64_t n_in = static_cast<uint64_t>(r.rx.n_slots), n_out = static_cast<uint64_t>(r.tx.n_slots);
    spin_until_ge<32, 512>(r.rx.full + in_seq % n_in, in_seq / n_in + 1, r.timeout_ns, r.rx.status, kLinkErrWaitFull);
    spin_until_ge<32, 512>(r.tx.free_ + out_seq % n_out, out_seq / n_out, r.timeout_ns, r.tx.status, kLinkErrWaitFree);
    s_in = in_seq;
    s_out = out_seq;
  }
  __syncthreads();
  const uint64_t in_seq = s_in, out_seq = s_out;
  const uint64_t in_slot = in_seq % static_cast<uint64_t>(r.rx.n_slots);
  const uint64_t out_slot = out_seq % static_cast<uint64_t>(r.tx.n_slots);
  const uint8_t* src = r.rx.ring + in_slot * r.rx.slot_bytes + kLinkHeaderBytes;
  uint8_t* base = r.tx.ring + out_slot * r.tx.slot_bytes;
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    LinkHeader* h = reinterpret_cast<LinkHeader*>(base);
    h->magic = kLinkMagic;
    h->n_tensors = kLinkRawKind;
    h->items = static_cast<uint32_t>(r.items);
    h->pad = 0;
    LinkTensorHdr th;
    th.bit = 0;
    th.dtype = kLinkDtypeBytes;
    th.n = r.bytes;
    th.data_off = kLinkHeaderBytes;
    th.alpha = INFINITY;
    th.pad = 0;
    h->t[0] = th;
  }
  uint8_t* dst = base + kLinkHeaderBytes;
  const size_t tid = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x;
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t n16 = r.bytes >> 4;
  const uint4* s4 = reinterpret_cast<const uint4*>(src);
  uint4* d4 = reinterpret_cast<uint4*>(dst);
  stream4(n16, tid, stride, [&](size_t i) { return __ldcg(s4 + i); }, [&](size_t i, uint4 v) { d4[i] = v; });
  for (size_t i = (n16 << 4) + tid; i < r.bytes; i += stride) dst[i] = __ldcg(src + i);
  // as put_end: one GPU-scope fence per CTA after its barrier; the last CTA to arrive publishes the peer slot and then
  // hands the host-fed slot back (its free flag is link_feed's back-pressure)
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const unsigned prev = atomicAdd(r.tx.done_ctr, 1u);
    if (prev == gridDim.x - 1) {
      *r.tx.done_ctr = 0;
      *reinterpret_cast<volatile uint64_t*>(r.tx.seq) = out_seq + 1;
      *reinterpret_cast<volatile uint64_t*>(r.rx.seq) = in_seq + 1;
      __threadfence_system();
      st_release_sys(r.tx.full + out_slot, out_seq / static_cast<uint64_t>(r.tx.n_slots) + 1);
      st_release_sys(r.rx.free_ + in_slot, in_seq / static_cast<uint64_t>(r.rx.n_slots) + 1);
    }
  }
}

// ------------------------------------------------------------------------------------------------ shared-memory input
// A first stage fed by a data rank without a GPU copies each input out of the shared-memory ring on its copy stream
// (pe_pipe_submit); this kernel, enqueued behind that copy, hands the slot back: the copy engine has finished reading it
// when the kernel starts.
__global__ void __launch_bounds__(1) link_shm_release_kernel(uint64_t* free_flag, uint64_t value) {
  st_release_sys(free_flag, value);
}

// ------------------------------------------------------------------------------------------------ host helpers
static int sm_count() {
  static int cached = 0;
  if (cached == 0) {
    int dev = 0, n = 0;
    if (cudaGetDevice(&dev) == cudaSuccess && cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) == cudaSuccess && n > 0)
      cached = n;
    else
      cached = kNumSMs;
  }
  return cached;
}

// private per-end counters: seq @0, done_ctr @64, bar_count @128, bar_gen @192, partials @256
constexpr size_t kCtlBytes = 256 + (kLinkMaxItems + 160) * kQPartialDoubles * sizeof(double);

static void preload_kernels();

static int alloc_common(pe_link* l) {
  PE_CUDA(cudaMalloc(&l->ctl_block, kCtlBytes));
  PE_CUDA(cudaMemset(l->ctl_block, 0, kCtlBytes));
  PE_CUDA(cudaHostAlloc(reinterpret_cast<void**>(&l->status_host), 64, cudaHostAllocMapped));
  memset(l->status_host, 0, 64);
  unsigned* status_dev = nullptr;
  PE_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(&status_dev), l->status_host, 0));
  uint8_t* c = static_cast<uint8_t*>(l->ctl_block);
  l->rx.seq = l->tx.seq = reinterpret_cast<uint64_t*>(c);   // each object's rx and tx ends get their own below if both exist
  l->rx.done_ctr = l->tx.done_ctr = reinterpret_cast<unsigned*>(c + 64);
  l->tx.bar_count = reinterpret_cast<unsigned*>(c + 128);
  l->tx.bar_gen = reinterpret_cast<unsigned*>(c + 192);
  l->tx.partials = reinterpret_cast<double*>(c + 256);
  l->rx.status = l->tx.status = status_dev;
  l->timeout_ns = link_timeout_ns();
  preload_kernels();
  const char* w = getenv("PIPEEDGE_WIRE_F16");
  l->wire_f16 = (w != nullptr && w[0] == '1') ? 1 : 0;
  return PE_OK;
}

// Force the kernels' module to load now: inside a stream capture a first-use load could be refused.
static void preload_kernels() {
  static bool done = false;
  if (done) return;
  cudaFuncAttributes attr;
  cudaFuncGetAttributes(&attr, link_get_kernel);
  cudaFuncGetAttributes(&attr, link_wait_kernel);
  cudaFuncGetAttributes(&attr, link_put_copy_kernel);
  cudaFuncGetAttributes(&attr, link_put_staged_kernel);
  cudaFuncGetAttributes(&attr, link_relay_kernel);
  cudaFuncGetAttributes(&attr, link_shm_release_kernel);
  cudaFuncGetAttributes(&attr, link_put_quant_kernel<2>);
  cudaFuncGetAttributes(&attr, link_put_quant_kernel<4>);
  cudaFuncGetAttributes(&attr, link_put_quant_kernel<8>);
  cudaFuncGetAttributes(&attr, link_put_quant_kernel<16>);
  cudaFuncSetAttribute(link_put_quant_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kQuantCacheBytes));
  cudaFuncSetAttribute(link_put_quant_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kQuantCacheBytes));
  cudaFuncSetAttribute(link_put_quant_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kQuantCacheBytes));
  cudaFuncSetAttribute(link_put_quant_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(kQuantCacheBytes));
  cudaGetLastError();
  done = true;
}

int link_check(pe_link* l) {
  if (l == nullptr || l->status_host == nullptr) return PE_OK;
  const unsigned code = *reinterpret_cast<volatile unsigned*>(l->status_host);
  if (code == kLinkErrNone) return PE_OK;
  static const char* names[] = {"", "the producer never delivered (full flag wait timed out)",
                                "the consumer never released the slot (free flag wait timed out)",
                                "payload description does not match the stage's expectation",
                                "grid barrier of the fused quantise-and-send kernel timed out"};
  set_error("link protocol error %u: %s", code, code < 5 ? names[code] : "unknown");
  return PE_ERR_CUDA;
}

int link_ticket_send(pe_link* l, long long a, long long b) {
  const long long msg[2] = {a, b};
  const int fd = (l->kind == 1) ? l->fd_peer : l->fd;
  PE_REQUIRE(fd >= 0, "link ticket: no channel");
  PE_REQUIRE(write_all(fd, msg, sizeof(msg)) == 0, "link ticket: socket write failed: %s", strerror(errno));
  return PE_OK;
}

int link_ticket_recv(pe_link* l, long long* out2) {
  PE_REQUIRE(l->fd >= 0, "link ticket: no channel");
  const int r = read_all(l->fd, out2, 2 * sizeof(long long));
  if (r == 1) return 1;
  PE_REQUIRE(r == 0, "link ticket: socket read failed: %s", strerror(errno));
  return PE_OK;
}

// ------------------------------------------------------------------------------------------------ launches
static size_t roundup(size_t x, size_t a) { return (x + a - 1) / a * a; }

static size_t wire_bytes(const pe_link* l, int items, size_t n, int bit) {
  if (bit == 0) return static_cast<size_t>(items) * n * (l->wire_f16 ? 2 : 4);
  return static_cast<size_t>(items) * quant_words(n, bit) * 4;
}

// How link_put ships one tensor of `items` x `n` values at `bit` bits on a GPU with `sms` SMs. `aligned`: a (and b)
// are 16-byte aligned. The one place that decides it: link_put launches what this returns, and
// pe_debug_link_put_plan reports it.
struct PutPlan {
  int path;        // PE_LINK_PATH_*
  int grid;        // CTAs of the send kernel
  int chunks;      // fused: segments per item
  size_t per;      // fused: elements per segment (multiple of 16)
  int cache;       // fused: the CTA's fp32 slice stays in shared memory between the passes (else pass 2 re-reads HBM)
  size_t smem;     // fused: dynamic shared memory
};

static PutPlan plan_put(int items, size_t n, int bit, bool aligned, int sms) {
  PutPlan pl = {};
  const size_t total = static_cast<size_t>(items) * n;
  if (bit == 0) {
    pl.path = PE_LINK_PATH_COPY;
    const size_t want = (total / 4 + kPutThreads - 1) / kPutThreads;
    // half the SMs move a few MB as fast as all of them and pay half the per-CTA arrival / fence cost
    const size_t cap = static_cast<size_t>((sms + 1) / 2);
    pl.grid = static_cast<int>(want < 1 ? 1 : (want > cap ? cap : want));
  } else if (quant_pack16_applies(bit, n, aligned)) {
    pl.path = PE_LINK_PATH_FUSED;
    // segments: `chunks` per item so that items * chunks ~ the grid; boundaries on multiples of 16 elements
    const int max_ctas = sms > 16 ? sms - 8 : sms;
    int chunks = items >= max_ctas ? 1 : max_ctas / items;
    const size_t by_size = (n + 4095) / 4096;
    if (static_cast<size_t>(chunks) > by_size) chunks = static_cast<int>(by_size);
    if (chunks > kQMaxChunks) chunks = kQMaxChunks;
    if (chunks < 1) chunks = 1;
    pl.chunks = chunks;
    pl.per = roundup((n + chunks - 1) / chunks, 16);
    const int segs = items * chunks;
    pl.grid = segs < max_ctas ? segs : max_ctas;
    const int segs_per_cta = (segs + pl.grid - 1) / pl.grid;
    const size_t cache_bytes = roundup(static_cast<size_t>(segs_per_cta) * pl.per * sizeof(float), 128);
    pl.cache = cache_bytes <= kQuantCacheBytes ? 1 : 0;
    pl.smem = pl.cache ? cache_bytes : 0;   // whole swizzle groups of 8 float4
  } else {
    // generic bit-widths / shapes: the stand-alone kernels quantise into local staging, one kernel ships it
    pl.path = PE_LINK_PATH_STAGED;
    const size_t bytes = static_cast<size_t>(items) * quant_words(n, bit) * 4;
    const size_t want = (bytes / 4 + kPutThreads - 1) / kPutThreads;
    pl.grid = static_cast<int>(want < 1 ? 1 : (want > static_cast<size_t>(2 * sms) ? 2 * sms : want));
  }
  return pl;
}

size_t link_payload_bytes(int items, size_t n, int bit, int wire_f16) {
  if (bit == 0) return static_cast<size_t>(items) * n * (wire_f16 ? 2 : 4);
  return static_cast<size_t>(items) * (quant_words(n, bit) * 4 + 2 * sizeof(float));
}

static bool put_aligned(const PutTensor& t) {
  return (reinterpret_cast<uintptr_t>(t.a) & 15) == 0 && (t.b == nullptr || (reinterpret_cast<uintptr_t>(t.b) & 15) == 0);
}

int link_put(pe_link* l, const PutTensor* t, int n_tensors, int items, int bit, int clamp, cudaStream_t stream,
             PutStamp* stamp) {
  PE_REQUIRE(l != nullptr && l->is_tx, "pe_link_put: not the producer end of a link");
  PE_REQUIRE(n_tensors >= 1 && n_tensors <= 2 && items > 0 && items <= kLinkMaxItems,
             "pe_link_put: %d tensors x %d items outside [1,2] x [1,%d]", n_tensors, items, kLinkMaxItems);
  PE_REQUIRE(bit >= 0 && bit <= 16, "pe_link_put: bit=%d outside [0,16]", bit);
  int last_staged = -1;   // the tensor after whose encode kernels stamp->encoded is launched
  if (stamp != nullptr) {
    stamp->bytes = 0;
    stamp->paths = 0;
    for (int ti = 0; ti < n_tensors; ++ti) {
      const int path = plan_put(items, t[ti].n, bit, put_aligned(t[ti]), sm_count()).path;
      if (path == PE_LINK_PATH_STAGED) last_staged = ti;
      stamp->paths |= 1 << path;
      stamp->bytes += link_payload_bytes(items, t[ti].n, bit, l->wire_f16);
    }
  }
  size_t off = kLinkHeaderBytes;
  for (int ti = 0; ti < n_tensors; ++ti) {
    PE_REQUIRE(t[ti].a != nullptr && t[ti].n > 0, "pe_link_put: null / empty tensor %d", ti);
    const size_t bytes = wire_bytes(l, items, t[ti].n, bit);
    PE_REQUIRE(off + bytes <= l->slot_bytes, "pe_link_put: payload (%zu bytes at %zu) exceeds the link's %zu-byte slots",
               bytes, off, l->slot_bytes);
    PutArgs p = {};
    p.tx = l->tx;
    p.t = t[ti];
    p.ti = ti;
    p.n_tensors = n_tensors;
    p.items = items;
    p.bit = bit;
    p.clamp = clamp;
    p.wire_f16 = l->wire_f16;
    p.is_last = ti == n_tensors - 1 ? 1 : 0;
    p.data_off = off;
    p.timeout_ns = l->timeout_ns;
    const size_t total = static_cast<size_t>(items) * t[ti].n;
    const bool aligned = put_aligned(t[ti]);
    const PutPlan pl = plan_put(items, t[ti].n, bit, aligned, sm_count());
    if (pl.path == PE_LINK_PATH_COPY) {
      PE_REQUIRE(aligned, "pe_link_put: payload tensors must be 16-byte aligned");
      link_put_copy_kernel<<<pl.grid, kPutThreads, 0, stream>>>(p);
      PE_CUDA(cudaGetLastError());
      count_launches(1);
    } else if (pl.path == PE_LINK_PATH_FUSED) {
      p.chunks = pl.chunks;
      p.per = pl.per;
      p.cache = pl.cache;
      p.factor_laplace = clamp_factor(bit, 0);
      p.factor_gelu = clamp_factor(bit, 1);
      switch (bit) {
        case 2: link_put_quant_kernel<2><<<pl.grid, kPutThreads, pl.smem, stream>>>(p); break;
        case 4: link_put_quant_kernel<4><<<pl.grid, kPutThreads, pl.smem, stream>>>(p); break;
        case 8: link_put_quant_kernel<8><<<pl.grid, kPutThreads, pl.smem, stream>>>(p); break;
        default: link_put_quant_kernel<16><<<pl.grid, kPutThreads, pl.smem, stream>>>(p); break;
      }
      PE_CUDA(cudaGetLastError());
      count_launches(1);
    } else {
      const float* x = t[ti].a;
      const size_t codes_bytes = roundup(bytes, 256);
      const size_t need = codes_bytes + 2 * roundup(items * sizeof(float), 256) + 256 + roundup(quant_workspace_bytes(items, t[ti].n), 256);
      PE_REQUIRE(l->quant_work != nullptr && need <= l->quant_work_bytes / 2 && total * sizeof(float) <= l->add_scratch_bytes,
                 "pe_link_put: staging buffers of this link are too small for %d items of %zu elements", items, t[ti].n);
      if (t[ti].b != nullptr) {
        PE_REQUIRE((total & 3) == 0, "pe_link_put: a + b payloads need a multiple of 4 elements");
        const int rc = add_impl(t[ti].a, t[ti].b, l->add_scratch, total, stream);
        if (rc != PE_OK) return rc;
        x = l->add_scratch;
      }
      uint8_t* w = static_cast<uint8_t*>(l->quant_work) + static_cast<size_t>(ti) * (l->quant_work_bytes / 2);
      uint8_t* codes = w;
      float* scale = reinterpret_cast<float*>(w + codes_bytes);
      float* shift = reinterpret_cast<float*>(w + codes_bytes + roundup(items * sizeof(float), 256));
      float* alpha = reinterpret_cast<float*>(w + codes_bytes + 2 * roundup(items * sizeof(float), 256));
      void* work = w + codes_bytes + 2 * roundup(items * sizeof(float), 256) + 256;
      int rc = quant_encode_impl(x, items, t[ti].n, bit, clamp, codes, scale, shift, alpha, work, stream);
      if (rc == PE_OK && ti == last_staged) rc = stamp->encoded(stamp->ctx, stream);
      if (rc != PE_OK) return rc;
      p.staged_codes = codes;
      p.staged_scale = scale;
      p.staged_shift = shift;
      p.staged_alpha = alpha;
      p.staged_bytes = bytes;
      link_put_staged_kernel<<<pl.grid, kPutThreads, 0, stream>>>(p);
      PE_CUDA(cudaGetLastError());
      count_launches(1);
    }
    off += roundup(bytes, 256);
  }
  return PE_OK;
}

static int launch_get(pe_link* l, const GetArgs& g, size_t work_units, bool may_decode, bool prewait,
                      cudaStream_t stream) {
  if (prewait) {
    // A consumer that may wait long while OTHER streams of this GPU compute (the data rank draining results) parks in
    // the one-warp kernel; the get kernel below then finds its flag raised. A stage's own compute stream has nothing
    // else to run while its input is missing, so there the get kernel waits by itself (one launch less per micro-batch).
    link_wait_kernel<<<1, 32, 0, stream>>>(g.rx, g.timeout_ns);
    PE_CUDA(cudaGetLastError());
    count_launches(1);
  }
  size_t want = (work_units + kGetThreads - 1) / kGetThreads;
  // copies: half the SMs (see link_put); dequantising payloads (the producer announced them at open) want every SM
  const size_t cap = static_cast<size_t>(l->quant_hint > 0 ? 2 * sm_count() : (sm_count() + 1) / 2);
  const int grid = static_cast<int>(want < 1 ? 1 : (want > cap ? cap : want));
  const size_t smem = may_decode ? 4096 * sizeof(float) : 0;   // LUT of 2^bit values for bit <= 12
  link_get_kernel<<<grid, kGetThreads, smem, stream>>>(g);
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  return PE_OK;
}

int link_get(pe_link* l, void* dst0, void* dst1, int items, size_t n0, size_t n1, int n_tensors, cudaStream_t stream,
             bool prewait) {
  PE_REQUIRE(l != nullptr && l->is_rx && l->kind != 2, "pe_link_get: not the consumer end of a peer link");
  PE_REQUIRE(dst0 != nullptr && items > 0 && items <= kLinkMaxItems && n0 > 0 && n_tensors >= 1 && n_tensors <= 2 &&
                 (n_tensors == 1 || (dst1 != nullptr && n1 > 0)),
             "pe_link_get: bad arguments");
  PE_REQUIRE((reinterpret_cast<uintptr_t>(dst0) & 15) == 0 && (dst1 == nullptr || (reinterpret_cast<uintptr_t>(dst1) & 15) == 0),
             "pe_link_get: destinations must be 16-byte aligned");
  GetArgs g = {};
  g.rx = l->rx;
  g.dst0 = dst0;
  g.dst1 = dst1;
  g.n0 = n0;
  g.n1 = n_tensors > 1 ? n1 : 0;
  g.items = items;
  g.n_tensors = n_tensors;
  g.raw = 0;
  g.timeout_ns = l->timeout_ns;
  return launch_get(l, g, static_cast<size_t>(items) * (n0 + g.n1) / 16, true, prewait, stream);
}

int link_get_raw(pe_link* l, void* dst, size_t bytes, int items, cudaStream_t stream, bool prewait) {
  PE_REQUIRE(l != nullptr && l->is_rx && dst != nullptr && bytes > 0, "pe_link_get_raw: bad arguments");
  PE_REQUIRE(kLinkHeaderBytes + bytes <= l->slot_bytes, "pe_link_get_raw: %zu bytes exceed the link's slots", bytes);
  PE_REQUIRE((reinterpret_cast<uintptr_t>(dst) & 15) == 0, "pe_link_get_raw: destination must be 16-byte aligned");
  PE_REQUIRE(items >= 0 && items <= kLinkMaxItems && (items == 0 || l->kind != 2),
             "pe_link_get_raw: a relayed raw payload (%d items) comes from a peer, not a host-fed link", items);
  GetArgs g = {};
  g.rx = l->rx;
  g.dst0 = dst;
  g.n0 = bytes;
  g.items = items > 0 ? items : 1;
  g.n_tensors = 1;
  g.raw = items > 0 ? 2 : 1;
  g.timeout_ns = l->timeout_ns;
  return launch_get(l, g, bytes / 64, false, prewait, stream);
}

int link_relay(pe_link* in, pe_link* out, int items, size_t bytes, cudaStream_t stream) {
  PE_REQUIRE(in != nullptr && in->kind == 2 && out != nullptr && out->is_tx,
             "link_relay: needs a host-fed input and the producer end of a link");
  PE_REQUIRE(items > 0 && items <= kLinkMaxItems && bytes > 0, "link_relay: %d items / %zu bytes outside [1,%d] / > 0",
             items, bytes, kLinkMaxItems);
  PE_REQUIRE(kLinkHeaderBytes + bytes <= in->slot_bytes && kLinkHeaderBytes + bytes <= out->slot_bytes,
             "link_relay: %zu bytes exceed the input ring's %zu-byte or the link's %zu-byte slots", bytes,
             in->slot_bytes - kLinkHeaderBytes, out->slot_bytes - kLinkHeaderBytes);
  RelayArgs r = {};
  r.rx = in->rx;
  r.tx = out->tx;
  r.bytes = bytes;
  r.items = items;
  r.timeout_ns = out->timeout_ns;
  // the copy path's rule (plan_put): one 16-byte vector per thread, at most half the SMs
  const size_t want = (bytes / 16 + kPutThreads - 1) / kPutThreads;
  const size_t cap = static_cast<size_t>((sm_count() + 1) / 2);
  const int grid = static_cast<int>(want < 1 ? 1 : (want > cap ? cap : want));
  link_relay_kernel<<<grid, kPutThreads, 0, stream>>>(r);
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  return PE_OK;
}

// Host-fed link: copy the next payload into the ring (waiting for its slot to be released) and raise its flag, both on
// `copy_stream`, so the transfer overlaps whatever the compute stream is doing.
int link_feed(pe_link* l, const void* src, size_t bytes, int src_is_host, cudaStream_t copy_stream) {
  PE_REQUIRE(l != nullptr && l->kind == 2 && src != nullptr && bytes > 0, "pe_link_feed: bad arguments");
  PE_REQUIRE(kLinkHeaderBytes + bytes <= l->slot_bytes, "pe_link_feed: %zu bytes exceed the link's %zu-byte slots", bytes,
             l->slot_bytes);
  const uint64_t slot = l->fed % static_cast<uint64_t>(l->n_slots), k = l->fed / static_cast<uint64_t>(l->n_slots);
  volatile uint64_t* free_flags = l->host_flags;
  uint64_t* vals = l->host_flags + kLinkMaxSlots;
  if (free_flags[slot] < k) {   // back-pressure: the stage has not consumed this slot's previous payload yet
    struct timespec t0, t1;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    unsigned spins = 0;
    while (__atomic_load_n(&l->host_flags[slot], __ATOMIC_ACQUIRE) < k) {
      if (++spins > 2000) {
        sched_yield();
        clock_gettime(CLOCK_MONOTONIC, &t1);
        const double waited = (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
        if (waited * 1e9 > static_cast<double>(l->timeout_ns)) {
          const int rc = link_check(l);
          if (rc != PE_OK) return rc;
          set_error("pe_link_feed: slot %llu was not released within the link timeout", static_cast<unsigned long long>(slot));
          return PE_ERR_CUDA;
        }
      }
    }
  }
  uint8_t* dst = l->rx.ring + slot * l->slot_bytes + kLinkHeaderBytes;
  PE_CUDA(cudaMemcpyAsync(dst, src, bytes, src_is_host ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToDevice, copy_stream));
  vals[slot] = k + 1;
  PE_CUDA(cudaMemcpyAsync(const_cast<uint64_t*>(l->rx.full) + slot, &vals[slot], sizeof(uint64_t), cudaMemcpyHostToDevice,
                          copy_stream));
  ++l->fed;
  return PE_OK;
}

// Producer-side staging for the generic bit-widths (stand-alone quant kernels quantise into local memory first): sized
// once for the link's slots, so that nothing is allocated while a stage's graph is being captured.
static int alloc_staging(pe_link* l) {
  const size_t payload = l->slot_bytes - kLinkHeaderBytes;
  l->add_scratch_bytes = roundup(payload, 256);
  PE_CUDA(cudaMalloc(reinterpret_cast<void**>(&l->add_scratch), l->add_scratch_bytes));
  // per tensor: codes (at most half of the fp32 payload at 16 bits) + scale / shift / alpha + the statistics workspace
  const size_t slice = roundup(payload / 2 + 4096 + quant_workspace_bytes(kLinkMaxItems, 1), 256);
  l->quant_work_bytes = 2 * slice;
  PE_CUDA(cudaMalloc(&l->quant_work, l->quant_work_bytes));
  return PE_OK;
}

static void free_link(pe_link* l) {
  if (l == nullptr) return;
  if (l->peer_block != nullptr) cudaIpcCloseMemHandle(l->peer_block);
  if (l->local_block != nullptr) cudaFree(l->local_block);
  if (l->ctl_block != nullptr) cudaFree(l->ctl_block);
  if (l->add_scratch != nullptr) cudaFree(l->add_scratch);
  if (l->quant_work != nullptr) cudaFree(l->quant_work);
  if (l->status_host != nullptr) cudaFreeHost(l->status_host);
  if (l->host_flags != nullptr) cudaFreeHost(l->host_flags);
  if (l->shm_registered) cudaHostUnregister(l->shm.base);
  hostring_unmap(&l->shm);
  if (l->kind == 1) {
    if (l->fd >= 0) close(l->fd);
    if (l->fd_peer >= 0) close(l->fd_peer);
  }
  delete l;
}

// A stage's end of a hop to or from a data rank without a GPU: map the segment named in `handle` and register it with
// CUDA, so that kernels reach its flags and slots and copy engines read it as pinned memory. *dev = the device alias of
// the mapping.
static int map_shm_end(pe_link* l, cudaIpcMemHandle_t handle, int n_slots, size_t slot_bytes, uint8_t** dev) {
  handle.reserved[sizeof(handle.reserved) - 1] = 0;
  int rc = hostring_map(handle.reserved, false, n_slots, slot_bytes, &l->shm);
  if (rc != PE_OK) return rc;
  PE_CUDA(cudaHostRegister(l->shm.base, l->shm.map_bytes, cudaHostRegisterMapped | cudaHostRegisterPortable));
  l->shm_registered = true;
  PE_CUDA(cudaHostGetDevicePointer(reinterpret_cast<void**>(dev), l->shm.base, 0));
  l->kind = 3;
  l->n_slots = n_slots;
  l->slot_bytes = slot_bytes;
  return PE_OK;
}

}  // namespace pe

// ==================================================================================================== C-ABI
extern "C" {

// Both ends call this once over the hop's connected socket `fd` (it stays owned by the caller and later carries the
// tickets); blocks until the peer has answered. The PRODUCER chooses the geometry: `slot_bytes` of payload room per slot
// (the 16 KiB header is added here) and `n_slots`; the consumer passes 0 for both.
int pe_link_open(int fd, int is_producer, size_t slot_payload_bytes, int n_slots, int quant_hint, pe_link** out) {
  using namespace pe;
  PE_REQUIRE(out != nullptr && fd >= 0, "pe_link_open: bad arguments");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;
  pe_link* l = new pe_link();
  l->fd = fd;
  l->kind = 0;
  rc = alloc_common(l);
  if (rc != PE_OK) { free_link(l); return rc; }
  if (is_producer) {
    if (n_slots < 2 || n_slots > kLinkMaxSlots || slot_payload_bytes == 0) {
      set_error("pe_link_open: n_slots=%d outside [2,%d] or empty slots", n_slots, kLinkMaxSlots);
      free_link(l);
      return PE_ERR_INVALID;
    }
    l->is_tx = true;
    l->n_slots = n_slots;
    l->slot_bytes = roundup(kLinkHeaderBytes + slot_payload_bytes, 4096);
    cudaError_t e = cudaMalloc(&l->local_block, kFlagsBytes);
    if (e == cudaSuccess) e = cudaMemset(l->local_block, 0, kFlagsBytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    HelloMsg hello = {};
    hello.magic = kLinkMagic;
    hello.n_slots = static_cast<uint32_t>(n_slots);
    hello.quant_hint = static_cast<uint32_t>(quant_hint > 0 ? quant_hint : 0);
    hello.slot_bytes = l->slot_bytes;
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&hello.handle, l->local_block);
    if (e != cudaSuccess) {
      check_cuda(e, "pe_link_open (producer set-up)");
      hello.magic = 0;   // tell the peer we failed, so that it does not block
      write_all(fd, &hello, sizeof(hello));
      free_link(l);
      return PE_ERR_CUDA;
    }
    ReplyMsg reply = {};
    if (write_all(fd, &hello, sizeof(hello)) != 0 || read_all(fd, &reply, sizeof(reply)) != 0 ||
        (reply.magic != kLinkMagic && reply.magic != kShmMagic) || reply.status != 0) {
      set_error("pe_link_open: handshake with the consumer failed");
      free_link(l);
      return PE_ERR_CUDA;
    }
    if (reply.magic == kShmMagic) {
      // the consumer is a data rank without a GPU: the send kernels store straight into its shared-memory ring, raw
      // f32 (the host reads the results as they are), and poll its free flags in mapped host memory
      uint8_t* dev = nullptr;
      rc = map_shm_end(l, reply.handle, n_slots, l->slot_bytes, &dev);
      const ReplyMsg ack = {kShmMagic, rc == PE_OK ? 0u : 1u, {}};
      if (write_all(fd, &ack, sizeof(ack)) != 0 && rc == PE_OK) {
        set_error("pe_link_open: socket write failed");
        rc = PE_ERR_CUDA;
      }
      if (rc == PE_OK) {
        l->tx.ring = dev + kShmCtlBytes;
        l->tx.full = reinterpret_cast<uint64_t*>(dev);
        l->tx.free_ = reinterpret_cast<const uint64_t*>(dev + kShmFreeOff);
        l->tx.slot_bytes = l->slot_bytes;
        l->tx.n_slots = n_slots;
        l->wire_f16 = 0;
        rc = alloc_staging(l);
      }
      if (rc != PE_OK) { free_link(l); return rc; }
      *out = l;
      return PE_OK;
    }
    e = cudaIpcOpenMemHandle(&l->peer_block, reply.handle, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) {
      check_cuda(e, "cudaIpcOpenMemHandle (consumer's ring)");
      free_link(l);
      return PE_ERR_CUDA;
    }
    l->tx.ring = static_cast<uint8_t*>(l->peer_block) + kFlagsBytes;
    l->tx.full = static_cast<uint64_t*>(l->peer_block);
    l->tx.free_ = static_cast<const uint64_t*>(l->local_block);
    l->tx.slot_bytes = l->slot_bytes;
    l->tx.n_slots = n_slots;
    rc = alloc_staging(l);
    if (rc != PE_OK) { free_link(l); return rc; }
  } else {
    l->is_rx = true;
    HelloMsg hello = {};
    ReplyMsg reply = {};
    reply.magic = kLinkMagic;
    if (read_all(fd, &hello, sizeof(hello)) != 0 || (hello.magic != kLinkMagic && hello.magic != kShmMagic) ||
        hello.n_slots < 2 || hello.n_slots > static_cast<uint32_t>(kLinkMaxSlots)) {
      set_error("pe_link_open: handshake with the producer failed");
      free_link(l);
      return PE_ERR_CUDA;
    }
    if (hello.magic == kShmMagic) {
      // the producer is a data rank without a GPU: its inputs are read out of the shared-memory ring by the host
      // (pe_link_shm_wait) and the copy engine (pe_pipe_submit), and handed back by pe_link_shm_release
      uint8_t* dev = nullptr;
      rc = map_shm_end(l, hello.handle, static_cast<int>(hello.n_slots), hello.slot_bytes, &dev);
      reply.magic = kShmMagic;
      reply.status = rc == PE_OK ? 0u : 1u;
      if (write_all(fd, &reply, sizeof(reply)) != 0 && rc == PE_OK) {
        set_error("pe_link_open: socket write failed");
        rc = PE_ERR_CUDA;
      }
      if (rc != PE_OK) { free_link(l); return rc; }
      l->shm_free_dev = reinterpret_cast<uint64_t*>(dev + kShmFreeOff);
      *out = l;
      return PE_OK;
    }
    l->n_slots = static_cast<int>(hello.n_slots);
    l->quant_hint = static_cast<int>(hello.quant_hint);
    l->slot_bytes = hello.slot_bytes;
    const size_t block = kFlagsBytes + l->slot_bytes * l->n_slots;
    cudaError_t e = cudaMalloc(&l->local_block, block);
    if (e == cudaSuccess) e = cudaMemset(l->local_block, 0, kFlagsBytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaIpcGetMemHandle(&reply.handle, l->local_block);
    if (e == cudaSuccess) e = cudaIpcOpenMemHandle(&l->peer_block, hello.handle, cudaIpcMemLazyEnablePeerAccess);
    reply.status = e == cudaSuccess ? 0u : 1u;
    const int w = write_all(fd, &reply, sizeof(reply));
    if (e != cudaSuccess || w != 0) {
      if (e != cudaSuccess) check_cuda(e, "pe_link_open (consumer set-up)");
      else set_error("pe_link_open: socket write failed");
      free_link(l);
      return PE_ERR_CUDA;
    }
    l->rx.ring = static_cast<uint8_t*>(l->local_block) + kFlagsBytes;
    l->rx.full = static_cast<const uint64_t*>(l->local_block);
    l->rx.free_ = static_cast<uint64_t*>(l->peer_block);
    l->rx.slot_bytes = l->slot_bytes;
    l->rx.n_slots = l->n_slots;
  }
  *out = l;
  return PE_OK;
}

// Both ends in this process (a one-rank pipeline's results path; tests): same kernels, same flags, no cudaIpc.
int pe_link_open_local(size_t slot_payload_bytes, int n_slots, int quant_hint, pe_link** out) {
  using namespace pe;
  PE_REQUIRE(out != nullptr && n_slots >= 2 && n_slots <= kLinkMaxSlots && slot_payload_bytes > 0,
             "pe_link_open_local: bad arguments");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;
  pe_link* l = new pe_link();
  l->kind = 1;
  l->is_tx = l->is_rx = true;
  l->quant_hint = quant_hint;
  rc = alloc_common(l);
  if (rc != PE_OK) { free_link(l); return rc; }
  int sv[2];
  if (socketpair(AF_UNIX, SOCK_STREAM, 0, sv) != 0) {
    set_error("pe_link_open_local: socketpair failed: %s", strerror(errno));
    free_link(l);
    return PE_ERR_CUDA;
  }
  l->fd = sv[0];        // consumer reads tickets here
  l->fd_peer = sv[1];   // producer writes them here
  l->n_slots = n_slots;
  l->slot_bytes = roundup(kLinkHeaderBytes + slot_payload_bytes, 4096);
  const size_t block = 2 * kFlagsBytes + l->slot_bytes * n_slots;
  cudaError_t e = cudaMalloc(&l->local_block, block);
  if (e == cudaSuccess) e = cudaMemset(l->local_block, 0, 2 * kFlagsBytes);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    check_cuda(e, "pe_link_open_local");
    free_link(l);
    return PE_ERR_NOMEM;
  }
  uint8_t* b = static_cast<uint8_t*>(l->local_block);
  l->rx.full = l->tx.full = reinterpret_cast<uint64_t*>(b);
  l->rx.free_ = reinterpret_cast<uint64_t*>(b + kFlagsBytes);
  l->tx.free_ = reinterpret_cast<const uint64_t*>(b + kFlagsBytes);
  l->rx.ring = l->tx.ring = b + 2 * kFlagsBytes;
  l->rx.slot_bytes = l->tx.slot_bytes = l->slot_bytes;
  l->rx.n_slots = l->tx.n_slots = n_slots;
  rc = alloc_staging(l);
  if (rc != PE_OK) { free_link(l); return rc; }
  // the two ends need their own sequence / arrival counters
  uint8_t* c = static_cast<uint8_t*>(l->ctl_block);
  l->rx.seq = reinterpret_cast<uint64_t*>(c + 8);
  l->rx.done_ctr = reinterpret_cast<unsigned*>(c + 72);
  *out = l;
  return PE_OK;
}

// Consumer end fed by the host (the data rank's inputs): pe_link_feed copies into the ring, a raw get drains it.
int pe_link_open_host(size_t slot_payload_bytes, int n_slots, pe_link** out) {
  using namespace pe;
  PE_REQUIRE(out != nullptr && n_slots >= 2 && n_slots <= kLinkMaxSlots && slot_payload_bytes > 0,
             "pe_link_open_host: bad arguments");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;
  pe_link* l = new pe_link();
  l->kind = 2;
  l->is_rx = true;
  rc = alloc_common(l);
  if (rc != PE_OK) { free_link(l); return rc; }
  l->n_slots = n_slots;
  l->slot_bytes = roundup(kLinkHeaderBytes + slot_payload_bytes, 4096);
  const size_t block = kFlagsBytes + l->slot_bytes * n_slots;
  cudaError_t e = cudaMalloc(&l->local_block, block);
  if (e == cudaSuccess) e = cudaMemset(l->local_block, 0, kFlagsBytes);
  if (e == cudaSuccess) e = cudaHostAlloc(reinterpret_cast<void**>(&l->host_flags), 2 * kLinkMaxSlots * sizeof(uint64_t), cudaHostAllocMapped);
  if (e == cudaSuccess) e = cudaDeviceSynchronize();
  if (e != cudaSuccess) {
    check_cuda(e, "pe_link_open_host");
    free_link(l);
    return PE_ERR_NOMEM;
  }
  memset(l->host_flags, 0, 2 * kLinkMaxSlots * sizeof(uint64_t));
  uint64_t* free_dev = nullptr;
  e = cudaHostGetDevicePointer(reinterpret_cast<void**>(&free_dev), l->host_flags, 0);
  if (e != cudaSuccess) {
    check_cuda(e, "cudaHostGetDevicePointer");
    free_link(l);
    return PE_ERR_CUDA;
  }
  uint8_t* b = static_cast<uint8_t*>(l->local_block);
  l->rx.full = reinterpret_cast<const uint64_t*>(b);
  l->rx.free_ = free_dev;
  l->rx.ring = b + kFlagsBytes;
  l->rx.slot_bytes = l->slot_bytes;
  l->rx.n_slots = n_slots;
  *out = l;
  return PE_OK;
}

int pe_link_close(pe_link* link) {
  pe::free_link(link);
  return PE_OK;
}

size_t pe_link_slot_bytes(const pe_link* link) { return link == nullptr ? 0 : link->slot_bytes - pe::kLinkHeaderBytes; }

// Producer: enqueue the kernels that ship a payload of one or two tensors (x_i = a_i + b_i when b_i != NULL), quantised to
// `bit` bits when bit > 0 (`clamp` = PE_CLAMP_*), on `stream`.
int pe_link_put(pe_link* link, const void* a0, const void* b0, size_t n0, const void* a1, const void* b1, size_t n1,
                int items, int bit, int clamp, void* stream) {
  pe::PutTensor t[2] = {{static_cast<const float*>(a0), static_cast<const float*>(b0), n0},
                        {static_cast<const float*>(a1), static_cast<const float*>(b1), n1}};
  return pe::link_put(link, t, a1 != nullptr ? 2 : 1, items, bit, clamp, static_cast<cudaStream_t>(stream));
}

// The fused QuantPipe encode-and-send of one tensor (SURVEY.md 8b): forward_hook_quant_encode (runtime.py:73-91) +
// TensorSendThread's send (p2p/__init__.py:170-204) as ONE kernel for bit in {2,4,8,16}, n % 16 == 0.
int pe_quant_encode_send(pe_link* link, const void* x, const void* skip, int items, size_t n, int bit, int clamp,
                         void* stream) {
  PE_REQUIRE(bit >= 1 && bit <= 16, "pe_quant_encode_send: bit=%d outside [1,16]", bit);
  pe::PutTensor t[1] = {{static_cast<const float*>(x), static_cast<const float*>(skip), n}};
  return pe::link_put(link, t, 1, items, bit, clamp, static_cast<cudaStream_t>(stream));
}

int pe_link_get(pe_link* link, void* dst0, void* dst1, int items, size_t n0, size_t n1, void* stream) {
  return pe::link_get(link, dst0, dst1, items, n0, n1, dst1 != nullptr ? 2 : 1, static_cast<cudaStream_t>(stream), true);
}

int pe_link_get_raw(pe_link* link, void* dst, size_t bytes, void* stream) {
  return pe::link_get_raw(link, dst, bytes, 0, static_cast<cudaStream_t>(stream), true);
}

int pe_link_feed(pe_link* link, const void* src, size_t bytes, int src_is_host, void* copy_stream) {
  return pe::link_feed(link, src, bytes, src_is_host, static_cast<cudaStream_t>(copy_stream));
}

int pe_link_ticket_send(pe_link* link, long long a, long long b) {
  PE_REQUIRE(link != nullptr, "pe_link_ticket_send: null link");
  return pe::link_ticket_send(link, a, b);
}

int pe_link_ticket_recv(pe_link* link, long long* out2) {
  PE_REQUIRE(link != nullptr && out2 != nullptr, "pe_link_ticket_recv: null pointer");
  return pe::link_ticket_recv(link, out2);
}

int pe_link_check(pe_link* link) { return pe::link_check(link); }

int pe_link_is_shm(const pe_link* link) { return link != nullptr && link->kind == 3 ? 1 : 0; }

// Consumer end of a shared-memory ring (a first stage fed by a data rank without a GPU): wait on the host (bounded) for
// the payload the last ticket announced, check its header, *src = the payload in registered host memory.
int pe_link_shm_wait(pe_link* link, int items, size_t bytes, const void** src) {
  PE_REQUIRE(link != nullptr && link->kind == 3 && link->is_rx && src != nullptr,
             "pe_link_shm_wait: not the consumer end of a shared-memory ring");
  return pe::hostring_read(&link->shm, items, bytes, src);
}

// ... and hand that slot back to the data rank behind everything enqueued on `stream` so far (the copy out of it): a
// one-thread kernel raises free[s] with st.release.sys in mapped host memory. No host synchronisation.
int pe_link_shm_release(pe_link* link, void* stream) {
  using namespace pe;
  PE_REQUIRE(link != nullptr && link->kind == 3 && link->is_rx, "pe_link_shm_release: not the consumer end of a shared-memory ring");
  HostRing& g = link->shm;
  const uint64_t n = static_cast<uint64_t>(g.n_slots);
  link_shm_release_kernel<<<1, 1, 0, static_cast<cudaStream_t>(stream)>>>(link->shm_free_dev + g.seq % n, g.seq / n + 1);
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  ++g.seq;
  return PE_OK;
}

// Tests: copy `bytes` at `offset` of the slot that holds payload number `seq` to host memory (consumer end; synchronises).
int pe_link_debug_read(pe_link* link, unsigned long long seq, size_t offset, void* host_dst, size_t bytes) {
  using namespace pe;
  PE_REQUIRE(link != nullptr && link->is_rx && host_dst != nullptr, "pe_link_debug_read: bad arguments");
  PE_REQUIRE(offset + bytes <= link->slot_bytes, "pe_link_debug_read: outside the slot");
  PE_CUDA(cudaDeviceSynchronize());
  const uint8_t* src = link->rx.ring + (seq % static_cast<unsigned long long>(link->n_slots)) * link->slot_bytes + offset;
  PE_CUDA(cudaMemcpy(host_dst, src, bytes, cudaMemcpyDeviceToHost));
  return PE_OK;
}

// Host-only: how pe_link_put would ship one tensor on this device (kNumSMs SMs when there is none).
int pe_debug_link_put_plan(int items, size_t n, int bit, int aligned, int* out5) {
  using namespace pe;
  PE_REQUIRE(out5 != nullptr && items > 0 && items <= kLinkMaxItems && n > 0 && bit >= 0 && bit <= 16,
             "pe_debug_link_put_plan: bad arguments");
  const PutPlan pl = plan_put(items, n, bit, aligned != 0, sm_count());
  out5[0] = pl.path;
  out5[1] = pl.grid;
  out5[2] = pl.chunks;
  out5[3] = static_cast<int>(pl.per);
  out5[4] = pl.cache;
  return PE_OK;
}

// Host-only: the payload bytes a put of one [items, n] tensor at `bit` bits writes (what a timestamped pipeline reports).
size_t pe_link_payload_bytes(int items, size_t n, int bit, int wire_f16) {
  if (items <= 0 || bit < 0 || bit > 16) return 0;
  return pe::link_payload_bytes(items, n, bit, wire_f16);
}

}  // extern "C"
