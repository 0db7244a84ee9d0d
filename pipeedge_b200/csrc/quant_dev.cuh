// QuantPipe pieces shared by quant.cu (stand-alone encode / decode) and link.cu (quantisation fused into the inter-stage
// send / receive kernels): every step whose bits both must agree on is written here once, and the host entry points of
// quant.cu are declared here for its callers.
#pragma once
#include <math.h>
#include <stdint.h>

#include "common.cuh"

namespace pe {

constexpr int kQMaxChunks = 64;      // partial-reduction chunks per item
constexpr int kQPartialDoubles = 5;  // min, max, sum, sumsq, sumsq of fp32-rounded squares

// ------------------------------------------------------------------ host entry points (quant.cu)
float clamp_factor(int bit, int gelu);
size_t quant_words(size_t n, int bit);
size_t quant_workspace_bytes(int items, size_t n);
int quant_stats_impl(const void* x, int items, size_t n, int bit, int clamp, void* scale, void* shift, void* alpha,
                     void* work, cudaStream_t stream);
int quant_encode_impl(const void* x, int items, size_t n, int bit, int clamp, void* codes, void* scale, void* shift,
                      void* alpha, void* work, cudaStream_t stream);
int quant_decode_impl(const void* codes, int items, size_t n, int bit, const void* scale, const void* shift, void* out,
                      cudaStream_t stream);

// The 16-value path (quant_pack16_kernel, link_put_quant_kernel) applies: 16 codes fill whole words, and the input is
// read as float4s.
inline bool quant_pack16_applies(int bit, size_t n, bool aligned16) {
  return (bit == 2 || bit == 4 || bit == 8 || bit == 16) && n % 16 == 0 && aligned16;
}

// ------------------------------------------------------------------ statistics
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
  return v;
}

// min / max and the fp64 sums clamp_alpha needs. A thread adds its elements in order; `ss += d * d` contracts to a DFMA.
struct QStats {
  float mn, mx;
  double s, ss, ss32;

  __device__ __forceinline__ static QStats empty() { return {INFINITY, -INFINITY, 0.0, 0.0, 0.0}; }
  __device__ __forceinline__ void add(float e) {
    mn = fminf(mn, e);
    mx = fmaxf(mx, e);
    const double d = static_cast<double>(e);
    s += d;
    ss += d * d;
    ss32 += static_cast<double>(__fmul_rn(e, e));
  }
  __device__ __forceinline__ void add(float4 v) { add(v.x); add(v.y); add(v.z); add(v.w); }
};

// The block's statistics -> one partial of kQPartialDoubles doubles at `out`: warps reduce, then thread 0 folds the
// warps in order. May be called in a loop: the first barrier keeps red[] until thread 0 has read the previous call's.
template <int kWarps>
__device__ __forceinline__ void stats_to_partial(QStats st, double (&red)[kWarps][kQPartialDoubles], double* out) {
  st.mn = warp_reduce(st.mn, [](float a, float b) { return fminf(a, b); });
  st.mx = warp_max(st.mx);
  st.s = warp_sum_d(st.s); st.ss = warp_sum_d(st.ss); st.ss32 = warp_sum_d(st.ss32);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  __syncthreads();
  if (lane == 0) {
    red[warp][0] = st.mn; red[warp][1] = st.mx; red[warp][2] = st.s; red[warp][3] = st.ss; red[warp][4] = st.ss32;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    double o0 = red[0][0], o1 = red[0][1], o2 = red[0][2], o3 = red[0][3], o4 = red[0][4];
    for (int w = 1; w < kWarps; ++w) {
      o0 = fmin(o0, red[w][0]); o1 = fmax(o1, red[w][1]);
      o2 += red[w][2]; o3 += red[w][3]; o4 += red[w][4];
    }
    out[0] = o0; out[1] = o1; out[2] = o2; out[3] = o3; out[4] = o4;
  }
}

// One item's partials [item][chunks][kQPartialDoubles], folded in chunk order. kFromGrid: other CTAs of the running grid
// wrote them, so they are read from L2 (__ldcg; L1 is not coherent). Partials an earlier kernel wrote are read with
// plain loads, which keep the fold shorter when there are many chunks.
template <bool kFromGrid>
__device__ __forceinline__ QStats fold_item(const double* partials, int item, int chunks) {
  const auto ld = [](const double* p) { return kFromGrid ? __ldcg(p) : *p; };
  double mn = INFINITY, mx = -INFINITY, s = 0.0, ss = 0.0, ss32 = 0.0;
  for (int c = 0; c < chunks; ++c) {
    const double* q = partials + (static_cast<size_t>(item) * chunks + c) * kQPartialDoubles;
    mn = fmin(mn, ld(q)); mx = fmax(mx, ld(q + 1));
    s += ld(q + 2); ss += ld(q + 3); ss32 += ld(q + 4);
  }
  return {static_cast<float>(mn), static_cast<float>(mx), s, ss, ss32};
}

// clamp_op.py:11-33: the Banner-2019 threshold from whole-tensor statistics accumulated in fp64.
//   Laplace (min < 0.2): torch.var(x, unbiased=False) -> fp32; GeLU: 2 * sum(x^2) / numel with fp32 squares.
__device__ __forceinline__ float clamp_alpha(int clamp, double gmin, double gs, double gss, double gss32, double cnt,
                                             float factor_laplace, float factor_gelu) {
  if (clamp == 0) return INFINITY;   // PE_CLAMP_NONE
  float variance, factor;
  const bool laplace = clamp == 2 || (clamp == 1 && gmin < 0.2);   // PE_CLAMP_LAPLACE / PE_CLAMP_AUTO
  if (laplace) {
    const double mean = gs / cnt;
    double var_d = gss / cnt - mean * mean;
    if (var_d < 0.0) var_d = 0.0;
    variance = static_cast<float>(var_d);
    factor = factor_laplace;
  } else {
    variance = __fdiv_rn(__fmul_rn(2.0f, static_cast<float>(gss32)), static_cast<float>(cnt));
    factor = factor_gelu;
  }
  return __fmul_rn(factor, __fsqrt_rn(__fmul_rn(0.5f, variance)));
}

// The threshold of `items` items of n values; item_total(i) is item i's QStats (fold_item), folded in item order.
template <typename ItemTotal>
__device__ __forceinline__ float fold_items_alpha(int items, ItemTotal item_total, size_t n, int clamp,
                                                  float factor_laplace, float factor_gelu) {
  double gmin = INFINITY, gs = 0.0, gss = 0.0, gss32 = 0.0;
  for (int i = 0; i < items; ++i) {
    const QStats t = item_total(i);
    gmin = fmin(gmin, static_cast<double>(t.mn));
    gs += t.s; gss += t.ss; gss32 += t.ss32;
  }
  return clamp_alpha(clamp, gmin, gs, gss, gss32, static_cast<double>(items) * static_cast<double>(n), factor_laplace,
                     factor_gelu);
}

// Clamp is monotonic: min / max of the clamped item = clamped min / max (basic_op.py:127-129).
__device__ __forceinline__ void item_scale_shift(float mn, float mx, float alpha, float& scale, float& shift) {
  shift = fminf(fmaxf(mn, -alpha), alpha);
  scale = __fsub_rn(fminf(fmaxf(mx, -alpha), alpha), shift);
}

// ------------------------------------------------------------------ encode
// basic_op.py:127-130 (`_quant_op`): clamp, (x - shift) / scale, * (2^bit - 1), np.around, astype(uint32).
// IEEE round-to-nearest sub / div / mul (no FMA contraction), rintf = round-half-to-even.
__device__ __forceinline__ uint32_t quant_code(float x, float alpha, float shift, float scale, float levels) {
  const float xc = fminf(fmaxf(x, -alpha), alpha);
  const float r = __fdiv_rn(__fsub_rn(xc, shift), scale);
  return static_cast<uint32_t>(rintf(__fmul_rn(levels, r)));
}

// 16 consecutive values -> 16 * BIT / 32 words, LSB-first (BIT in {2, 4, 8, 16}); store() writes them as one vector.
template <int BIT>
struct Packed16 {
  static constexpr int kWords = 16 * BIT / 32;
  uint32_t w[kWords];

  __device__ __forceinline__ void store(uint32_t* dst) const {
    if (kWords == 1) dst[0] = w[0];
    else if (kWords == 2) *reinterpret_cast<uint2*>(dst) = make_uint2(w[0], w[1]);
    else {
#pragma unroll
      for (int k = 0; k < kWords; k += 4) *reinterpret_cast<uint4*>(dst + k) = make_uint4(w[k], w[k + 1], w[k + 2], w[k + 3]);
    }
  }
};

template <int BIT>
__device__ __forceinline__ Packed16<BIT> pack16(const float4 (&v)[4], float alpha, float shift, float scale) {
  constexpr int kRatio = 32 / BIT;
  const float levels = static_cast<float>((1u << BIT) - 1u);
  uint32_t q[16];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    q[4 * j + 0] = quant_code(v[j].x, alpha, shift, scale, levels);
    q[4 * j + 1] = quant_code(v[j].y, alpha, shift, scale, levels);
    q[4 * j + 2] = quant_code(v[j].z, alpha, shift, scale, levels);
    q[4 * j + 3] = quant_code(v[j].w, alpha, shift, scale, levels);
  }
  Packed16<BIT> out;
#pragma unroll
  for (int k = 0; k < Packed16<BIT>::kWords; ++k) {
    uint32_t acc = 0;
#pragma unroll
    for (int j = 0; j < kRatio; ++j) acc |= q[k * kRatio + j] << (j * BIT);
    out.w[k] = acc;
  }
  return out;
}

// ------------------------------------------------------------------ decode
// `_intmap2float` + `tensor_decode` (basic_op.py:146-163): float32(code / (2^bit - 1)) with a float64 divide, then
// * scale + shift as two fp32 roundings.
__device__ __forceinline__ float dequant_unit(uint32_t code, double levels) {
  return static_cast<float>(static_cast<double>(code) / levels);
}
__device__ __forceinline__ float dequant_value(float unit, float scale, float shift) {
  return __fadd_rn(__fmul_rn(unit, scale), shift);
}

struct QDecoder {
  int bit, ratio;   // ratio = codes per word
  uint32_t mask;
  double levels;
  const float* lut;
  bool use_lut;     // false: divide per code

  // code j (LSB-first) of `word`, decoded
  __device__ __forceinline__ float value(uint32_t word, int j, float scale, float shift) const {
    const uint32_t c = (word >> (j * bit)) & mask;
    return dequant_value(use_lut ? lut[c] : dequant_unit(c, levels), scale, shift);
  }
  // the word holding values e0 .. e0 + ratio - 1 of an item of n values -> out[0 ..) (stops at the item's end)
  __device__ __forceinline__ void word(uint32_t w, size_t e0, size_t n, float scale, float shift, float* out) const {
    for (int j = 0; j < ratio; ++j) {
      if (e0 + j >= n) break;
      out[j] = value(w, j, scale, shift);
    }
  }
};

// Every thread of the block calls this. For bit <= 12 the 2^bit possible units are tabulated in `lut` (shared memory)
// instead of divided per code.
__device__ __forceinline__ QDecoder fill_dequant_lut(float* lut, int bit) {
  const uint32_t mask = (1u << bit) - 1u;
  const QDecoder d = {bit, 32 / bit, mask, static_cast<double>(mask), lut, bit <= 12};
  if (d.use_lut) {
    for (uint32_t c = threadIdx.x; c <= mask; c += blockDim.x) lut[c] = dequant_unit(c, d.levels);
    __syncthreads();
  }
  return d;
}

}  // namespace pe
