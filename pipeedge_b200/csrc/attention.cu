// Unmasked multi-head self-attention, softmax(Q K^T * d^-0.5) V, for S <= 512 tokens and head_dim d = 64 or 80
// (80: ViT-Huge; the kernel is a template on d, any multiple of 16 would do).
// One CTA per (query split, head, item): K and V of the head are staged once in shared memory with cp.async
// (16-byte chunks, padded rows -> conflict-free ldmatrix, one commit group per 64-key chunk so that the first
// chunk's maths overlaps the rest of the load); each warp owns 16 query rows and walks the keys in chunks of
// 64 - the last chunk trimmed to whole 16-key groups - with an online softmax (fp32 max/sum, exp2 with the
// scale folded in); P is rounded to fp16 for the P.V product, accumulators stay fp32 in registers. The number
// of warps per CTA and of query splits is picked so that S = 197 wastes < 6 % of the rows (13 row groups ->
// 2 CTAs of 7 warps) instead of padding to 256.
// Tensor cores through the warp-level mma.sync m16n8k16 path: the fall-back for the shapes the wgmma kernel
// (attention_wgmma.cu) does not take - head_dim 80, S > 256 - and the kernel PE_ATTN_WGMMA=0 selects. Attention is
// ~4% of the block's FLOPs (SURVEY.md 8d). Replaces HF eager_attention_forward (see pe_attention in the header).
#include <cstdlib>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"

namespace pe {

void count_launches(int n);
int attention_wgmma_impl(const void* qkv, void* ctx, int batch, int tokens, int heads, int head_dim,
                         cudaStream_t stream);

constexpr int kAttnKc = 64;
constexpr int kAttnMaxWarps = 8;

__device__ __forceinline__ void cp_async_16(void* smem, const void* gmem) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
// wait until at most `pending` of this thread's commit groups are still in flight
__device__ __forceinline__ void cp_async_wait_pending(int pending) {
  switch (pending) {
    case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
    case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
    case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
    case 3: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
    case 4: asm volatile("cp.async.wait_group 4;" ::: "memory"); break;
    case 5: asm volatile("cp.async.wait_group 5;" ::: "memory"); break;
    case 6: asm volatile("cp.async.wait_group 6;" ::: "memory"); break;
    default: asm volatile("cp.async.wait_group 7;" ::: "memory"); break;
  }
}
__device__ __forceinline__ void ldmatrix_x4(uint32_t (&r)[4], const void* smem) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(smem)));
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t (&r)[4], const void* smem) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(smem_u32(smem)));
}
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, "
      "{%0, %1, %2, %3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

// grid = (query splits, heads, items); block = warps * 32; each warp: 16 query rows.
template <int kAttnD>
__global__ void __launch_bounds__(kAttnMaxWarps * 32)
attention_kernel(const __half* __restrict__ qkv, __half* __restrict__ ctx, int tokens, int heads, float scale_log2e) {
  extern __shared__ __align__(16) uint8_t attn_smem[];
  constexpr int kAttnLd = kAttnD + 8;   // halves per smem row: 144 / 176 bytes, conflict-free for ldmatrix
  pdl_launch_dependents();
  pdl_wait();
  const int nwarps = blockDim.x >> 5;
  const int qrows = nwarps * 16;                          // query rows of this CTA
  const int kpad = (tokens + 15) & ~15;                   // keys rounded up to whole 16-key groups
  __half* sq = reinterpret_cast<__half*>(attn_smem);
  __half* sk = sq + qrows * kAttnLd;
  __half* sv = sk + static_cast<size_t>(kpad) * kAttnLd;

  const int q0 = blockIdx.x * qrows;
  const int head = blockIdx.y;
  const int item = blockIdx.z;
  const int hidden = heads * kAttnD;
  const size_t row_pitch = static_cast<size_t>(3) * hidden;
  const __half* base = qkv + static_cast<size_t>(item) * tokens * row_pitch + static_cast<size_t>(head) * kAttnD;
  const int tid = threadIdx.x;
  const int nchunks = (kpad + kAttnKc - 1) / kAttnKc;

  // ---- stage Q (group 0 together with the first key chunk), then K/V chunk by chunk
  {
    constexpr int kCpr = kAttnD / 8;   // 16-byte chunks per head row
    const int nthreads = blockDim.x;
    const uint4 zero = make_uint4(0, 0, 0, 0);
    for (int idx = tid; idx < qrows * kCpr; idx += nthreads) {
      const int r = idx / kCpr, chunk16 = idx - r * kCpr;
      __half* dst = sq + r * kAttnLd + chunk16 * 8;
      if (q0 + r < tokens) cp_async_16(dst, base + static_cast<size_t>(q0 + r) * row_pitch + chunk16 * 8);
      else *reinterpret_cast<uint4*>(dst) = zero;
    }
    for (int c = 0; c < nchunks; ++c) {
      const int kbeg = c * kAttnKc, kend = min(kpad, (c + 1) * kAttnKc);
      for (int idx = tid; idx < (kend - kbeg) * kCpr; idx += nthreads) {
        const int rr = idx / kCpr, chunk16 = idx - rr * kCpr;
        const int r = kbeg + rr;
        __half* dk = sk + static_cast<size_t>(r) * kAttnLd + chunk16 * 8;
        __half* dv = sv + static_cast<size_t>(r) * kAttnLd + chunk16 * 8;
        if (r < tokens) {
          const __half* src = base + static_cast<size_t>(r) * row_pitch + chunk16 * 8;
          cp_async_16(dk, src + hidden);
          cp_async_16(dv, src + 2 * hidden);
        } else {
          *reinterpret_cast<uint4*>(dk) = zero;
          *reinterpret_cast<uint4*>(dv) = zero;
        }
      }
      cp_async_commit();
    }
  }

  const int warp = tid >> 5, lane = tid & 31;
  const int wrow = warp * 16;  // this warp's first query row within the CTA
  const bool warp_active = q0 + wrow < tokens;   // warp-uniform; idle warps still take part in the barriers

  uint32_t qf[kAttnD / 16][4];
  float o[kAttnD / 8][4];
#pragma unroll
  for (int i = 0; i < kAttnD / 8; ++i) { o[i][0] = o[i][1] = o[i][2] = o[i][3] = 0.f; }
  float m_run[2] = {-INFINITY, -INFINITY};  // running max (of raw scores) for rows lane/4 and lane/4+8
  float l_run[2] = {0.f, 0.f};

  for (int kc = 0; kc < nchunks; ++kc) {
    cp_async_wait_pending(nchunks - 1 - kc);
    __syncthreads();
    if (!warp_active) continue;
    if (kc == 0) {
#pragma unroll
      for (int ks = 0; ks < kAttnD / 16; ++ks) {
        const int r = wrow + (lane & 7) + ((lane >> 3) & 1) * 8;
        const int c = ks * 16 + (lane >> 4) * 8;
        ldmatrix_x4(qf[ks], sq + r * kAttnLd + c);
      }
    }
    const int key0 = kc * kAttnKc;
    const int ngrp = min(kAttnKc, kpad - key0) >> 4;   // 16-key groups in this chunk (1..4), warp-uniform
    float s[kAttnKc / 8][4];
#pragma unroll
    for (int i = 0; i < kAttnKc / 8; ++i) { s[i][0] = s[i][1] = s[i][2] = s[i][3] = 0.f; }
    // S = Q K^T
#pragma unroll
    for (int ks = 0; ks < kAttnD / 16; ++ks) {
#pragma unroll
      for (int np = 0; np < kAttnKc / 16; ++np) {
        if (np < ngrp) {
          uint32_t kf[4];
          const int key = key0 + np * 16 + (lane & 7) + (lane >> 4) * 8;
          const int c = ks * 16 + ((lane >> 3) & 1) * 8;
          ldmatrix_x4(kf, sk + static_cast<size_t>(key) * kAttnLd + c);
          mma_16816(s[2 * np], qf[ks], kf[0], kf[1]);
          mma_16816(s[2 * np + 1], qf[ks], kf[2], kf[3]);
        }
      }
    }
    // mask keys past the sequence end (also the groups this chunk does not have)
    if (key0 + kAttnKc > tokens) {
#pragma unroll
      for (int nt = 0; nt < kAttnKc / 8; ++nt) {
        const int key = key0 + nt * 8 + (lane & 3) * 2;
        if (key >= tokens) { s[nt][0] = -INFINITY; s[nt][2] = -INFINITY; }
        if (key + 1 >= tokens) { s[nt][1] = -INFINITY; s[nt][3] = -INFINITY; }
      }
    }
    // online softmax
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < kAttnKc / 8; ++nt) {
      mx[0] = fmaxf(mx[0], fmaxf(s[nt][0], s[nt][1]));
      mx[1] = fmaxf(mx[1], fmaxf(s[nt][2], s[nt][3]));
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    }
    float corr[2], msc[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const float m_new = fmaxf(m_run[h], mx[h]);   // every chunk holds at least one real key -> finite
      corr[h] = exp2f((m_run[h] - m_new) * scale_log2e);
      m_run[h] = m_new;
      msc[h] = m_new * scale_log2e;
    }
    float psum[2] = {0.f, 0.f};
    uint32_t pf[kAttnKc / 16][4];
#pragma unroll
    for (int nt = 0; nt < kAttnKc / 8; ++nt) {
      const float p0 = exp2f(s[nt][0] * scale_log2e - msc[0]);
      const float p1 = exp2f(s[nt][1] * scale_log2e - msc[0]);
      const float p2 = exp2f(s[nt][2] * scale_log2e - msc[1]);
      const float p3 = exp2f(s[nt][3] * scale_log2e - msc[1]);
      psum[0] += p0 + p1;
      psum[1] += p2 + p3;
      // C fragments of two adjacent key tiles form one A fragment (16 keys) for P.V
      pf[nt >> 1][(nt & 1) * 2 + 0] = pack_half2(p0, p1);
      pf[nt >> 1][(nt & 1) * 2 + 1] = pack_half2(p2, p3);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      psum[h] += __shfl_xor_sync(0xffffffffu, psum[h], 1);
      psum[h] += __shfl_xor_sync(0xffffffffu, psum[h], 2);
      l_run[h] = l_run[h] * corr[h] + psum[h];
    }
#pragma unroll
    for (int i = 0; i < kAttnD / 8; ++i) {
      o[i][0] *= corr[0]; o[i][1] *= corr[0];
      o[i][2] *= corr[1]; o[i][3] *= corr[1];
    }
    // O += P V
#pragma unroll
    for (int ks = 0; ks < kAttnKc / 16; ++ks) {
      if (ks < ngrp) {
#pragma unroll
        for (int dp = 0; dp < kAttnD / 16; ++dp) {
          uint32_t vf[4];
          const int key = key0 + ks * 16 + (lane & 7) + ((lane >> 3) & 1) * 8;
          const int c = dp * 16 + (lane >> 4) * 8;
          ldmatrix_x4_trans(vf, sv + static_cast<size_t>(key) * kAttnLd + c);
          mma_16816(o[2 * dp], pf[ks], vf[0], vf[1]);
          mma_16816(o[2 * dp + 1], pf[ks], vf[2], vf[3]);
        }
      }
    }
  }
  if (!warp_active) return;

  // ---- normalise and store the merged-head context
  const float inv0 = 1.0f / l_run[0], inv1 = 1.0f / l_run[1];
  const int r_lo = q0 + wrow + (lane >> 2), r_hi = r_lo + 8;
  __half* out = ctx + static_cast<size_t>(item) * tokens * hidden + static_cast<size_t>(head) * kAttnD;
#pragma unroll
  for (int i = 0; i < kAttnD / 8; ++i) {
    const int c = i * 8 + (lane & 3) * 2;
    if (r_lo < tokens)
      *reinterpret_cast<__half2*>(out + static_cast<size_t>(r_lo) * hidden + c) = __floats2half2_rn(o[i][0] * inv0, o[i][1] * inv0);
    if (r_hi < tokens)
      *reinterpret_cast<__half2*>(out + static_cast<size_t>(r_hi) * hidden + c) = __floats2half2_rn(o[i][2] * inv1, o[i][3] * inv1);
  }
}

template <int kAttnD>
static int launch_attention(const void* qkv, void* ctx, int batch, int tokens, int heads, cudaStream_t stream) {
  // 16-row groups -> query splits of at most 8 warps; prefer the fewest splits (K/V are staged once per CTA)
  // that still give the SMs a full wave of CTAs
  const int groups = (tokens + 15) / 16;
  int splits = (groups + kAttnMaxWarps - 1) / kAttnMaxWarps;
  while (static_cast<long>(splits) * heads * batch < kNumSMs && splits < groups) ++splits;
  const int warps = (groups + splits - 1) / splits;
  splits = (groups + warps - 1) / warps;
  const int kpad = (tokens + 15) & ~15;
  PE_REQUIRE((kpad + kAttnKc - 1) / kAttnKc <= 8, "pe_attention: tokens=%d exceeds 512", tokens);
  const size_t smem = static_cast<size_t>(warps * 16 + 2 * kpad) * (kAttnD + 8) * sizeof(__half);
  PE_REQUIRE(smem <= 227 * 1024, "pe_attention: tokens=%d exceeds the shared-memory resident K/V limit", tokens);
  static size_t configured = 0;
  if (configured == 0)
    cudaFuncSetAttribute(attention_kernel<kAttnD>, cudaFuncAttributePreferredSharedMemoryCarveout,
                         cudaSharedmemCarveoutMaxShared);
  if (smem > configured) {
    PE_CUDA(cudaFuncSetAttribute(attention_kernel<kAttnD>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem)));
    configured = smem;
  }
  const dim3 grid(splits, heads, batch);
  const float scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(kAttnD));
  PE_CUDA(launch_pdl(attention_kernel<kAttnD>, grid, dim3(warps * 32), smem, stream, static_cast<const __half*>(qkv),
                     static_cast<__half*>(ctx), tokens, heads, scale_log2e));
  count_launches(1);
  return PE_OK;
}

int attention_impl(const void* qkv, void* ctx, int batch, int tokens, int heads, int head_dim, cudaStream_t stream) {
  PE_REQUIRE(qkv && ctx, "pe_attention: null pointer");
  PE_REQUIRE(batch > 0 && tokens > 0 && heads > 0, "pe_attention: bad shape");
  static const int use_wgmma = [] {
    const char* e = getenv("PE_ATTN_WGMMA");
    return (e != nullptr && e[0] == '0') ? 0 : 1;     // PE_ATTN_WGMMA=0 selects the mma.sync kernel below
  }();
  if (use_wgmma) {   // shapes the wgmma kernel does not take (head_dim != 64, S > 256) fall through
    const int rc = attention_wgmma_impl(qkv, ctx, batch, tokens, heads, head_dim, stream);
    if (rc != PE_ERR_INVALID) return rc;
  }
  if (head_dim == 64) return launch_attention<64>(qkv, ctx, batch, tokens, heads, stream);
  if (head_dim == 80) return launch_attention<80>(qkv, ctx, batch, tokens, heads, stream);
  set_error("pe_attention: head_dim=%d unsupported (64 and 80 are built)", head_dim);
  return PE_ERR_INVALID;
}

}  // namespace pe
