// LayerNorm row statistics shared by the fused projection + residual + LayerNorm epilogue (gemm_wgmma.cu) and the
// stand-alone kernel that mirrors it (layernorm.cu). A row is cut into 32-column chunks; each chunk is reduced to
// (mean, M2 = sum of squared deviations) by ONE thread in index order, chunks are merged in column order inside a slice of
// `slice` columns, slices in column order across the row (Chan's parallel update). Every step is an explicit IEEE
// operation (no contraction, no reassociation), so the fused kernel - where slices live in different CTAs of a cluster -
// and the stand-alone kernel produce bit-identical statistics and outputs: a pipeline's result does not depend on where
// the partition cuts fall.
#pragma once
#include "common.cuh"

namespace pe {

__device__ __forceinline__ void ln_chunk32(const float (&v)[32], float& mean_c, float& m2_c) {
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) sum = __fadd_rn(sum, v[i]);
  mean_c = __fmul_rn(sum, 1.0f / 32.0f);
  float m2 = 0.f;
#pragma unroll
  for (int i = 0; i < 32; ++i) {
    const float d = __fsub_rn(v[i], mean_c);
    m2 = __fmaf_rn(d, d, m2);
  }
  m2_c = m2;
}

// (cnt, mean, m2) <- merge with a block of n_b values of statistics (mean_b, m2_b)
__device__ __forceinline__ void ln_merge(float& cnt, float& mean, float& m2, float n_b, float mean_b, float m2_b) {
  const float tot = __fadd_rn(cnt, n_b);
  const float delta = __fsub_rn(mean_b, mean);
  mean = __fmaf_rn(delta, __fdiv_rn(n_b, tot), mean);
  m2 = __fadd_rn(__fadd_rn(m2, m2_b), __fmul_rn(__fmul_rn(delta, delta), __fdiv_rn(__fmul_rn(cnt, n_b), tot)));
  cnt = tot;
}

__device__ __forceinline__ float ln_rstd(float m2, float inv_n, float eps) {
  return __fdiv_rn(1.0f, __fsqrt_rn(__fmaf_rn(m2, inv_n, eps)));
}

__device__ __forceinline__ float ln_apply(float v, float mean, float rstd, float g, float b) {
  return __fmaf_rn(__fmul_rn(__fsub_rn(v, mean), rstd), g, b);
}

}  // namespace pe
