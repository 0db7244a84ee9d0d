// Unmasked multi-head self-attention on Hopper tensor cores (wgmma), head_dim 64, S <= 256 keys
// (PE_ATTN_WGMMA=0 selects the mma.sync kernel of attention.cu instead, which also serves every other shape).
//
// One CTA = one warpgroup per (64 query rows, head, item); warp w owns query rows [16w, 16w + 16).
//   1. Q [64 x 64], K [kp x 64], V [kp x 64] (kp = S rounded up to 32) arrive as three TMA boxes of 128-byte rows
//      (SWIZZLE_128B) through a 3-D tensor map [item][row][3H]: rows past the item's S are out of bounds inside the
//      item -> zero-filled. Q + K complete on one mbarrier, V on a second, so S = Q K^T and the softmax run while V
//      is still arriving.
//   2. S = Q K^T: 4 x wgmma m64n(kp)k16, A = Q and B = K both K-major from shared memory, fp32 in registers.
//   3. softmax on the accumulator fragments: each row lives in the four lanes of a quad (max / sum by two shuffles),
//      keys >= S masked, exp2 with the scale folded in; P is packed to fp16 pairs in registers.
//   4. O = P V: kp/16 x wgmma m64n64k16 with A = P straight from those registers (the accumulator fragment of two
//      adjacent 8-key column blocks is the A fragment of one 16-key step) and B = V read MN-major (imm-trans-b) from
//      the very image TMA wrote: 8-key groups 1024 B apart, +2048 B per K=16 step, no transpose of V anywhere.
//   5. epilogue: scale by 1 / row sum, fp16 pairs into Q's (dead) buffer in the 128-byte swizzle, one TMA store of
//      the 64 x 64 tile into ctx [item][row][H]; rows >= S are clipped by the tensor map.
#include "../../include/pipeedge_b200.h"
#include "common.cuh"
#include "wgmma.cuh"

namespace pe {

void count_launches(int n);

namespace {

constexpr int kD = 64;
constexpr int kRows = 64;        // query rows per CTA: one warpgroup's wgmma M
constexpr int kThreads = 128;

__device__ __forceinline__ void tma_load_3d_addr(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar_addr, int c0,
                                                 int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar_addr), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1, int c2) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_src), "r"(c0), "r"(c1), "r"(c2)
               : "memory");
}
__device__ __forceinline__ void st_shared_u32(uint32_t addr, uint32_t v) {
  asm volatile("st.shared.u32 [%0], %1;" ::"r"(addr), "r"(v) : "memory");
}

// O[64 x 64] (+)= P V with P from registers (A fragment of m64nNk16: {row g, k 2c..2c+1}, {row g+8, same},
// {row g, k 8+2c..}, {row g+8, k 8+2c..}) and V MN-major in shared memory.
__device__ __forceinline__ void wgmma_pv(float (&d)[32], const uint32_t (&a)[4], uint64_t desc_b, uint32_t scale_d) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {" PE_R32 "}, {%32, %33, %34, %35}, %36, p, 1, 1, 1;\n\t}"
      : PE_D16(0), PE_D16(16)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(desc_b), "r"(scale_d));
}

__device__ __forceinline__ uint32_t pack_half2(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}

template <int KP>
__global__ void __launch_bounds__(kThreads)
attention_wgmma_kernel(const __grid_constant__ CUtensorMap tm_q, const __grid_constant__ CUtensorMap tm_kv,
                       const __grid_constant__ CUtensorMap tm_o, int tokens, int heads, float scale_log2e) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t bar_qk, bar_v;
  // SWIZZLE_128B tiles start on 1024-byte boundaries (KP * 128 is a multiple of 4 KiB)
  const uint32_t sq = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t sk = sq + kRows * 128;
  const uint32_t sv = sk + KP * 128;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * kRows, head = blockIdx.y, item = blockIdx.z;
  const int hidden = heads * kD;
  const uint32_t qk_addr = smem_u32(&bar_qk), v_addr = smem_u32(&bar_v);
  pdl_launch_dependents();
  if (tid == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_kv);
    tma_prefetch_desc(&tm_o);
    mbar_init(&bar_qk, 1);
    mbar_init(&bar_v, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();   // qkv is the predecessor's output
  if (tid == 0) {
    mbar_arrive_expect_tx_addr(qk_addr, (kRows + KP) * 128);   // whole boxes, zero-filled rows included
    mbar_arrive_expect_tx_addr(v_addr, KP * 128);
    tma_load_3d_addr(sq, &tm_q, qk_addr, head * kD, q0, item);
    tma_load_3d_addr(sk, &tm_kv, qk_addr, hidden + head * kD, 0, item);
    tma_load_3d_addr(sv, &tm_kv, v_addr, 2 * hidden + head * kD, 0, item);
  }
  mbar_wait_addr(qk_addr, 0);

  // ---- S = Q K^T (K += 16 fp16 = 32 bytes inside the swizzled row: +2 in 16-byte units)
  float s[KP / 2];
#pragma unroll
  for (int i = 0; i < KP / 2; ++i) s[i] = 0.f;
  const uint64_t dq = wgmma_desc_kmajor_sw128(sq), dk = wgmma_desc_kmajor_sw128(sk);
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < kD / 16; ++k) Wgmma<KP>::mma(s, dq + 2 * k, dk + 2 * k, k != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();

  // ---- softmax: register 4j + {0,1} = row g, keys 8j + 2c + {0,1}; 4j + {2,3} = row g + 8
  const int g = lane >> 2, c = lane & 3;
  float mx0 = -INFINITY, mx1 = -INFINITY;
#pragma unroll
  for (int j = 0; j < KP / 8; ++j) {
    const int key = 8 * j + 2 * c;
    if (key >= tokens) { s[4 * j] = -INFINITY; s[4 * j + 2] = -INFINITY; }
    if (key + 1 >= tokens) { s[4 * j + 1] = -INFINITY; s[4 * j + 3] = -INFINITY; }
    mx0 = fmaxf(mx0, fmaxf(s[4 * j], s[4 * j + 1]));
    mx1 = fmaxf(mx1, fmaxf(s[4 * j + 2], s[4 * j + 3]));
  }
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
  mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
  mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
  const float b0 = mx0 * scale_log2e, b1 = mx1 * scale_log2e;   // key 0 is always real: finite
  float l0 = 0.f, l1 = 0.f;
  uint32_t pa[KP / 16][4];
#pragma unroll
  for (int j = 0; j < KP / 8; ++j) {
    const float p0 = exp2f(fmaf(s[4 * j], scale_log2e, -b0));
    const float p1 = exp2f(fmaf(s[4 * j + 1], scale_log2e, -b0));
    const float p2 = exp2f(fmaf(s[4 * j + 2], scale_log2e, -b1));
    const float p3 = exp2f(fmaf(s[4 * j + 3], scale_log2e, -b1));
    l0 += p0 + p1;
    l1 += p2 + p3;
    pa[j >> 1][(j & 1) * 2] = pack_half2(p0, p1);
    pa[j >> 1][(j & 1) * 2 + 1] = pack_half2(p2, p3);
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);

  // ---- O = P V
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  mbar_wait_addr(v_addr, 0);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < KP / 16; ++ks)
    wgmma_pv(o, pa[ks], wgmma_desc_kmajor_sw128(sv + static_cast<uint32_t>(ks) * 2048u), ks != 0 ? 1u : 0u);
  wgmma_commit();
  wgmma_wait<0>();

  // ---- normalise, stage the fp16 tile in Q's buffer as TMA's 128-byte swizzle lays it out (16-byte chunk j of row r
  // at chunk j ^ (r & 7): the 32 lanes of a warp hit 32 different banks), one TMA store of the merged-head context
  const float inv0 = 1.0f / l0, inv1 = 1.0f / l1;
  const int r0 = warp * 16 + g, r1 = r0 + 8;
  __syncthreads();   // every warp's Q K^T has finished reading Q
#pragma unroll
  for (int j = 0; j < kD / 8; ++j) {
    const uint32_t c4 = static_cast<uint32_t>(4 * c);
    st_shared_u32(sq + static_cast<uint32_t>(r0) * 128u + ((j ^ (r0 & 7)) << 4) + c4,
                  pack_half2(o[4 * j] * inv0, o[4 * j + 1] * inv0));
    st_shared_u32(sq + static_cast<uint32_t>(r1) * 128u + ((j ^ (r1 & 7)) << 4) + c4,
                  pack_half2(o[4 * j + 2] * inv1, o[4 * j + 3] * inv1));
  }
  fence_proxy_async_smem();   // the generic-proxy writes above, before the async-proxy store reads them
  __syncthreads();
  if (tid == 0) {
    tma_store_3d(&tm_o, sq, head * kD, q0, item);
    tma_store_commit();
    tma_store_wait_all();
  }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// A [batch][tokens][width] fp16 tensor (qkv: width 3H, ctx: width H); box = 64 columns x `box_rows` rows of one item.
int encode_rows_3d(CUtensorMap* map, const void* base, int batch, int tokens, int width, int box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (fn == nullptr) {
    set_error("cuTensorMapEncodeTiled is unavailable");
    return PE_ERR_CUDA;
  }
  const cuuint64_t dims[3] = {static_cast<cuuint64_t>(width), static_cast<cuuint64_t>(tokens),
                              static_cast<cuuint64_t>(batch)};
  const cuuint64_t strides[2] = {static_cast<cuuint64_t>(width) * 2,
                                 static_cast<cuuint64_t>(width) * 2 * static_cast<cuuint64_t>(tokens)};
  const cuuint32_t box[3] = {64u, static_cast<cuuint32_t>(box_rows), 1u};
  const cuuint32_t estr[3] = {1, 1, 1};
  const CUresult rc = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 3, const_cast<void*>(base), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled (attention) failed (CUresult %d)", static_cast<int>(rc));
    return PE_ERR_CUDA;
  }
  return PE_OK;
}

template <int KP>
int launch(const CUtensorMap& tm_q, const CUtensorMap& tm_kv, const CUtensorMap& tm_o, int batch, int tokens,
           int heads, cudaStream_t stream) {
  const size_t smem = static_cast<size_t>(kRows + 2 * KP) * 128 + 1024;
  static bool configured = false;
  if (!configured) {
    PE_CUDA(cudaFuncSetAttribute(attention_wgmma_kernel<KP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 static_cast<int>(smem)));
    configured = true;
  }
  const dim3 grid((tokens + kRows - 1) / kRows, heads, batch);
  const float scale_log2e = 1.4426950408889634f / sqrtf(static_cast<float>(kD));
  PE_CUDA(launch_pdl(attention_wgmma_kernel<KP>, grid, dim3(kThreads), smem, stream, tm_q, tm_kv, tm_o, tokens, heads,
                     scale_log2e));
  count_launches(1);
  return PE_OK;
}

}  // namespace

// Returns PE_ERR_INVALID (without an error message change) when the shape is outside what this kernel handles, so the
// caller can fall back to the mma.sync kernel.
int attention_wgmma_impl(const void* qkv, void* ctx, int batch, int tokens, int heads, int head_dim,
                         cudaStream_t stream) {
  if (head_dim != kD || tokens > 256 || tokens < 1 || (reinterpret_cast<uintptr_t>(qkv) & 15) != 0 ||
      (reinterpret_cast<uintptr_t>(ctx) & 15) != 0)
    return PE_ERR_INVALID;
  const int kp = (tokens + 31) & ~31;
  CUtensorMap tm_q, tm_kv, tm_o;
  int rc = encode_rows_3d(&tm_q, qkv, batch, tokens, 3 * heads * kD, kRows);
  if (rc != PE_OK) return rc;
  rc = encode_rows_3d(&tm_kv, qkv, batch, tokens, 3 * heads * kD, kp);
  if (rc != PE_OK) return rc;
  rc = encode_rows_3d(&tm_o, ctx, batch, tokens, heads * kD, kRows);
  if (rc != PE_OK) return rc;
  switch (kp) {
    case 32: return launch<32>(tm_q, tm_kv, tm_o, batch, tokens, heads, stream);
    case 64: return launch<64>(tm_q, tm_kv, tm_o, batch, tokens, heads, stream);
    case 96: return launch<96>(tm_q, tm_kv, tm_o, batch, tokens, heads, stream);
    case 128: return launch<128>(tm_q, tm_kv, tm_o, batch, tokens, heads, stream);
    case 160: return launch<160>(tm_q, tm_kv, tm_o, batch, tokens, heads, stream);
    case 192: return launch<192>(tm_q, tm_kv, tm_o, batch, tokens, heads, stream);
    case 224: return launch<224>(tm_q, tm_kv, tm_o, batch, tokens, heads, stream);
    default: return launch<256>(tm_q, tm_kv, tm_o, batch, tokens, heads, stream);
  }
}

}  // namespace pe
