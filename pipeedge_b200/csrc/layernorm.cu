// LayerNorm over the last dim (fp32 in, fp32 and/or fp16 out) and dtype casts. HBM/L2-bound:
// one warp per row, 128-bit loads, the row lives in registers between the two statistics passes.
// Replaces nn.LayerNorm at vit.py:59,66,168 and inside BertSelfOutput/BertOutput/BertEmbeddings.
#include "../../include/pipeedge_b200.h"
#include <cstdlib>

#include "common.cuh"
#include "ln_dev.cuh"

namespace pe {

void count_launches(int n);
int linear_ln_cluster(int n);

// Every kernel of the stage asks for the same (maximum-shared) L1/shared split as the GEMM and attention kernels:
// switching the carve-out between consecutive kernels makes the SMs drain and reconfigure.
template <typename K>
static void prefer_max_shared(K kernel) {
  cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared);
}

constexpr int kLnMaxVec = 12;  // float4 per lane: hidden <= 12 * 4 * 32 = 1536
constexpr int kLnWarpsPerBlock = 4;

// t = x (+ resid); optionally sum_out = t (the updated fp32 residual stream); then LayerNorm(t).
// Folding the residual add in here keeps it out of the GEMM epilogues, where each lane owns a different ROW
// and a residual read costs 32 cache lines per instruction; here a warp reads whole rows.
// kVec = float4s per lane (hidden <= kVec * 128): sized per model width so that the row AND its gamma / beta slices stay
// in registers. gamma / beta are model weights, so they are fetched BEFORE the programmatic dependency on the
// producing kernel resolves: their L2 latency overlaps the predecessor's tail instead of following the statistics.
template <int kVec>
__global__ void __launch_bounds__(kLnWarpsPerBlock * 32)
layernorm_kernel(const float* __restrict__ x, const float* resid, const float* __restrict__ gamma,
                 const float* __restrict__ beta, float eps, float* sum_out, float* out_f32, __half* out_f16, int rows,
                 int hidden) {
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int nvec = hidden >> 2;  // hidden % 4 == 0 enforced by the host
  float4 gv[kVec], bv[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      gv[i] = __ldg(reinterpret_cast<const float4*>(gamma) + idx);
      bv[i] = __ldg(reinterpret_cast<const float4*>(beta) + idx);
    }
  }
  pdl_wait();
  const int row = blockIdx.x * kLnWarpsPerBlock + (threadIdx.x >> 5);
  if (row >= rows) return;
  const float4* xr = reinterpret_cast<const float4*>(x + static_cast<size_t>(row) * hidden);
  const float4* rr = resid != nullptr ? reinterpret_cast<const float4*>(resid + static_cast<size_t>(row) * hidden) : nullptr;
  // Every load of the row (and of its residual) is issued before the first use: sum_out may alias resid, so the
  // compiler cannot hoist a later row load above an earlier sum_out store by itself, and a warp that stalls on its
  // first add with two loads in flight leaves the kernel latency-bound (ncu r02b: 1.0 TB/s).
  float4 v[kVec], rv[kVec];
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) v[i] = xr[idx];
  }
  if (rr != nullptr) {
#pragma unroll
    for (int i = 0; i < kVec; ++i) {
      const int idx = lane + i * 32;
      if (idx < nvec) rv[i] = rr[idx];
    }
  }
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      if (rr != nullptr) {
        v[i].x += rv[i].x; v[i].y += rv[i].y; v[i].z += rv[i].z; v[i].w += rv[i].w;
        if (sum_out != nullptr) reinterpret_cast<float4*>(sum_out + static_cast<size_t>(row) * hidden)[idx] = v[i];
      }
      sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mean = warp_sum(sum) / static_cast<float>(hidden);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float var = warp_sum(sq) / static_cast<float>(hidden);
  const float rstd = 1.0f / sqrtf(var + eps);
#pragma unroll
  for (int i = 0; i < kVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      const float4 g = gv[i], b = bv[i];
      float4 o;
      o.x = (v[i].x - mean) * rstd * g.x + b.x;
      o.y = (v[i].y - mean) * rstd * g.y + b.y;
      o.z = (v[i].z - mean) * rstd * g.z + b.z;
      o.w = (v[i].w - mean) * rstd * g.w + b.w;
      if (out_f32 != nullptr) reinterpret_cast<float4*>(out_f32 + static_cast<size_t>(row) * hidden)[idx] = o;
      if (out_f16 != nullptr) {
        uint2 pk;
        *reinterpret_cast<__half2*>(&pk.x) = __floats2half2_rn(o.x, o.y);
        *reinterpret_cast<__half2*>(&pk.y) = __floats2half2_rn(o.z, o.w);
        reinterpret_cast<uint2*>(out_f16 + static_cast<size_t>(row) * hidden)[idx] = pk;
      }
    }
  }
}

// The stand-alone mirror of the fused projection + residual + LayerNorm epilogue (ln_dev.cuh): one warp per row, one LANE
// per 32-column chunk (the fused kernel's thread), chunk statistics merged through shuffles in exactly the fused
// kernel's order (chunks inside a slice, then slices). Used wherever a LayerNorm has no projection of its own stage in
// front of it - a stage's first sub-layer, the final LayerNorm - when the fused kernel is enabled, so that the result of
// a pipeline does not depend on where it is cut.
template <int kCpl>   // chunks per lane: hidden <= kCpl * 1024
__global__ void __launch_bounds__(kLnWarpsPerBlock * 32)
layernorm_chunked_kernel(const float* __restrict__ x, const float* resid, const float* __restrict__ gamma,
                         const float* __restrict__ beta, float eps, float* sum_out, float* out_f32, __half* out_f16,
                         int rows, int hidden, int slice) {
  pdl_launch_dependents();
  const int lane = threadIdx.x & 31;
  const int nchunks = hidden >> 5;
  pdl_wait();
  const int row = blockIdx.x * kLnWarpsPerBlock + (threadIdx.x >> 5);
  if (row >= rows) return;
  const size_t base = static_cast<size_t>(row) * hidden;
  float v[kCpl][32];
  float mean_c[kCpl], m2_c[kCpl];
#pragma unroll
  for (int q = 0; q < kCpl; ++q) {
    const int c = lane + 32 * q;
    mean_c[q] = 0.f; m2_c[q] = 0.f;
    if (c < nchunks) {
      const float4* x4 = reinterpret_cast<const float4*>(x + base + c * 32);
      float4 xv[8], rv[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) xv[i] = x4[i];
      if (resid != nullptr) {
        const float4* r4 = reinterpret_cast<const float4*>(resid + base + c * 32);
#pragma unroll
        for (int i = 0; i < 8; ++i) rv[i] = r4[i];
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (resid != nullptr) {
          xv[i].x = __fadd_rn(xv[i].x, rv[i].x); xv[i].y = __fadd_rn(xv[i].y, rv[i].y);
          xv[i].z = __fadd_rn(xv[i].z, rv[i].z); xv[i].w = __fadd_rn(xv[i].w, rv[i].w);
          if (sum_out != nullptr) reinterpret_cast<float4*>(sum_out + base + c * 32)[i] = xv[i];
        }
        v[q][4 * i] = xv[i].x; v[q][4 * i + 1] = xv[i].y; v[q][4 * i + 2] = xv[i].z; v[q][4 * i + 3] = xv[i].w;
      }
      ln_chunk32(v[q], mean_c[q], m2_c[q]);
    }
  }
  // merge in the fused kernel's order; every lane computes the same totals
  const int cps = slice >> 5, nslices = hidden / slice;
  float cnt = 0.f, mean = 0.f, m2 = 0.f;
  for (int sidx = 0; sidx < nslices; ++sidx) {
    float scnt = 0.f, smean = 0.f, sm2 = 0.f;
    for (int k = 0; k < cps; ++k) {
      const int c = sidx * cps + k;
      float mc = 0.f, qc = 0.f;
#pragma unroll
      for (int q = 0; q < kCpl; ++q) {
        const float a = __shfl_sync(0xffffffffu, mean_c[q], c & 31);
        const float b = __shfl_sync(0xffffffffu, m2_c[q], c & 31);
        if ((c >> 5) == q) { mc = a; qc = b; }
      }
      if (k == 0) { scnt = 32.f; smean = mc; sm2 = qc; }
      else ln_merge(scnt, smean, sm2, 32.f, mc, qc);
    }
    ln_merge(cnt, mean, m2, static_cast<float>(slice), smean, sm2);
  }
  const float rstd = ln_rstd(m2, 1.0f / static_cast<float>(hidden), eps);
#pragma unroll
  for (int q = 0; q < kCpl; ++q) {
    const int c = lane + 32 * q;
    if (c < nchunks) {
      const float4* g4 = reinterpret_cast<const float4*>(gamma + c * 32);
      const float4* b4 = reinterpret_cast<const float4*>(beta + c * 32);
#pragma unroll
      for (int i = 0; i < 4; ++i) {     // 8 columns per trip: two fp32 stores, one fp16 store
        const float4 ga = __ldg(g4 + 2 * i), gb = __ldg(g4 + 2 * i + 1), ba = __ldg(b4 + 2 * i), bb = __ldg(b4 + 2 * i + 1);
        const float4 lo = make_float4(ln_apply(v[q][8 * i], mean, rstd, ga.x, ba.x), ln_apply(v[q][8 * i + 1], mean, rstd, ga.y, ba.y),
                                      ln_apply(v[q][8 * i + 2], mean, rstd, ga.z, ba.z), ln_apply(v[q][8 * i + 3], mean, rstd, ga.w, ba.w));
        const float4 hi = make_float4(ln_apply(v[q][8 * i + 4], mean, rstd, gb.x, bb.x), ln_apply(v[q][8 * i + 5], mean, rstd, gb.y, bb.y),
                                      ln_apply(v[q][8 * i + 6], mean, rstd, gb.z, bb.z), ln_apply(v[q][8 * i + 7], mean, rstd, gb.w, bb.w));
        if (out_f32 != nullptr) {
          reinterpret_cast<float4*>(out_f32 + base + c * 32)[2 * i] = lo;
          reinterpret_cast<float4*>(out_f32 + base + c * 32)[2 * i + 1] = hi;
        }
        if (out_f16 != nullptr) {
          uint4 pk;
          __half2* h2 = reinterpret_cast<__half2*>(&pk);
          h2[0] = __floats2half2_rn(lo.x, lo.y); h2[1] = __floats2half2_rn(lo.z, lo.w);
          h2[2] = __floats2half2_rn(hi.x, hi.y); h2[3] = __floats2half2_rn(hi.z, hi.w);
          reinterpret_cast<uint4*>(out_f16 + base + c * 32)[i] = pk;
        }
      }
    }
  }
}

// PE_FUSE_LN=1: projections run with the fused residual + LayerNorm epilogue wherever the stage allows (stage.cu), and the
// remaining stand-alone LayerNorms use the kernel above so that both paths agree bit for bit.
bool fuse_ln_enabled() {
  static const bool on = [] {
    const char* e = getenv("PE_FUSE_LN");
    return e != nullptr && e[0] == '1';
  }();
  return on;
}

int layernorm_impl(const void* x, const void* resid, const void* gamma, const void* beta, float eps, void* sum_out,
                   void* out_f32, void* out_f16, int rows, int hidden, cudaStream_t stream) {
  PE_REQUIRE(x && gamma && beta && (out_f32 || out_f16), "pe_layernorm: null pointer");
  PE_REQUIRE(resid != nullptr || sum_out == nullptr, "pe_residual_layernorm: sum_out needs resid");
  PE_REQUIRE(rows > 0 && hidden > 0 && (hidden & 3) == 0 && hidden <= kLnMaxVec * 128,
             "pe_layernorm: hidden=%d must be a multiple of 4 and <= %d", hidden, kLnMaxVec * 128);
  const int grid = (rows + kLnWarpsPerBlock - 1) / kLnWarpsPerBlock;
  const int cn = linear_ln_cluster(hidden);
  if (fuse_ln_enabled() && cn > 0 && hidden <= 2048 && (hidden & 31) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0) {
    auto kernel = hidden <= 1024 ? layernorm_chunked_kernel<1> : layernorm_chunked_kernel<2>;
    PE_CUDA(launch_pdl(kernel, dim3(grid), dim3(kLnWarpsPerBlock * 32), 0, stream, static_cast<const float*>(x),
                       static_cast<const float*>(resid), static_cast<const float*>(gamma), static_cast<const float*>(beta),
                       eps, static_cast<float*>(sum_out), static_cast<float*>(out_f32), static_cast<__half*>(out_f16), rows,
                       hidden, hidden / cn));
    count_launches(1);
    return PE_OK;
  }
  static bool configured = false;
  if (!configured) {
    prefer_max_shared(layernorm_kernel<6>);
    prefer_max_shared(layernorm_kernel<8>);
    prefer_max_shared(layernorm_kernel<kLnMaxVec>);
    configured = true;
  }
  auto kernel = hidden <= 6 * 128 ? layernorm_kernel<6> : (hidden <= 8 * 128 ? layernorm_kernel<8> : layernorm_kernel<kLnMaxVec>);
  PE_CUDA(launch_pdl(kernel, dim3(grid), dim3(kLnWarpsPerBlock * 32), 0, stream,
                     static_cast<const float*>(x), static_cast<const float*>(resid), static_cast<const float*>(gamma),
                     static_cast<const float*>(beta), eps, static_cast<float*>(sum_out), static_cast<float*>(out_f32),
                     static_cast<__half*>(out_f16), rows, hidden));
  count_launches(1);
  return PE_OK;
}

__global__ void cast_f32_f16_kernel(const float* __restrict__ src, __half* __restrict__ dst, size_t n) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t n4 = n >> 2;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4; i += stride) {
    const float4 v = reinterpret_cast<const float4*>(src)[i];
    uint2 pk;
    *reinterpret_cast<__half2*>(&pk.x) = __floats2half2_rn(v.x, v.y);
    *reinterpret_cast<__half2*>(&pk.y) = __floats2half2_rn(v.z, v.w);
    reinterpret_cast<uint2*>(dst)[i] = pk;
  }
  for (size_t i = (n4 << 2) + blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += stride)
    dst[i] = __float2half_rn(src[i]);
}

__global__ void cast_f16_f32_kernel(const __half* __restrict__ src, float* __restrict__ dst, size_t n) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t n2 = n >> 1;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n2; i += stride) {
    const float2 v = __half22float2(reinterpret_cast<const __half2*>(src)[i]);
    reinterpret_cast<float2*>(dst)[i] = v;
  }
  if ((n & 1) && blockIdx.x == 0 && threadIdx.x == 0) dst[n - 1] = __half2float(src[n - 1]);
}

int cast_impl(const void* src, void* dst, size_t n, bool to_half, cudaStream_t stream) {
  PE_REQUIRE(src && dst, "pe_cast: null pointer");
  if (n == 0) return PE_OK;
  const int block = 256;
  size_t want = (n / 4 + block - 1) / block;
  const int grid = static_cast<int>(want < 1 ? 1 : (want > static_cast<size_t>(kNumSMs) * 8 ? kNumSMs * 8 : want));
  static bool configured = false;
  if (!configured) { prefer_max_shared(cast_f32_f16_kernel); prefer_max_shared(cast_f16_f32_kernel); configured = true; }
  if (to_half) {
    PE_REQUIRE((reinterpret_cast<uintptr_t>(src) & 15) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0,
               "pe_cast_f32_to_f16: misaligned");
    cast_f32_f16_kernel<<<grid, block, 0, stream>>>(static_cast<const float*>(src), static_cast<__half*>(dst), n);
  } else {
    PE_REQUIRE((reinterpret_cast<uintptr_t>(src) & 3) == 0 && (reinterpret_cast<uintptr_t>(dst) & 7) == 0,
               "pe_cast_f16_to_f32: misaligned");
    cast_f16_f32_kernel<<<grid, block, 0, stream>>>(static_cast<const __half*>(src), static_cast<float*>(dst), n);
  }
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  return PE_OK;
}

// out = a + b (fp32): materialises the residual stream when a stage ends right after an output projection / FC2.
__global__ void add_f32_kernel(const float* __restrict__ a, const float* b, float* out, size_t n4) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n4; i += stride) {
    const float4 x = reinterpret_cast<const float4*>(a)[i];
    const float4 y = reinterpret_cast<const float4*>(b)[i];
    reinterpret_cast<float4*>(out)[i] = make_float4(x.x + y.x, x.y + y.y, x.z + y.z, x.w + y.w);
  }
}

// The same, one float per thread, for operands that are not 16-byte aligned (a link payload's a / b may start anywhere).
__global__ void add_f32_scalar_kernel(const float* __restrict__ a, const float* b, float* out, size_t n) {
  const size_t stride = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; i < n; i += stride) out[i] = a[i] + b[i];
}

int add_impl(const void* a, const void* b, void* out, size_t n, cudaStream_t stream) {
  PE_REQUIRE(a && b && out && (n & 3) == 0, "pe_add: bad arguments");
  const bool vec = ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(out)) & 15) == 0;
  const size_t units = vec ? n >> 2 : n;
  size_t want = (units + 255) / 256;
  const int grid = static_cast<int>(want < 1 ? 1 : (want > static_cast<size_t>(kNumSMs) * 8 ? kNumSMs * 8 : want));
  static bool configured = false;
  if (!configured) { prefer_max_shared(add_f32_kernel); configured = true; }
  if (vec)
    add_f32_kernel<<<grid, 256, 0, stream>>>(static_cast<const float*>(a), static_cast<const float*>(b),
                                             static_cast<float*>(out), units);
  else
    add_f32_scalar_kernel<<<grid, 256, 0, stream>>>(static_cast<const float*>(a), static_cast<const float*>(b),
                                                    static_cast<float*>(out), n);
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  return PE_OK;
}

// Busy-wait kernel: keeps the stream occupied for ~ms so that work enqueued behind it is fully queued
// before it starts (used by pe_stage_profile to keep host launch latency out of per-kernel timings).
__global__ void spin_kernel(long long cycles) {
  const long long t0 = clock64();
  while (clock64() - t0 < cycles) {}
}

int spin_impl(float ms, cudaStream_t stream) {
  spin_kernel<<<1, 1, 0, stream>>>(static_cast<long long>(ms * 1.9e6f));
  PE_CUDA(cudaGetLastError());
  return PE_OK;
}

}  // namespace pe
