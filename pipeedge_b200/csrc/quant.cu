// QuantPipe on the device: Banner-2019 clamp + per-item affine quantise + LSB-first bit-pack, and the
// inverse. HBM-bound byte/integer work: two streaming passes over the fp32 activation (statistics,
// then quantise+pack) and one over the codes. Bit-exactness against the NumPy reference comes from
// using IEEE round-to-nearest sub/div/mul intrinsics (no FMA contraction), rintf (half-to-even) and
// fp64 accumulation for the variance that sets the clamp threshold.
// Replaces runtime.py:73-119 + quantization/basic_op.py + clamp_op.py (see the header for the mapping).
#include <math.h>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"
#include "quant_dev.cuh"

namespace pe {

void count_launches(int n);

constexpr int kQStatThreads = 256;

// ------------------------------------------------------------------ Lambert W (host, fp64)
static double lambert_w0(double z) {
  // principal branch for z >= 0: Halley iterations from the asymptotic guess
  if (z == 0.0) return 0.0;
  double w = z < 3.0 ? 0.5 * z / (1.0 + 0.5 * z) + 0.3 : log(z) - log(log(z));
  for (int it = 0; it < 100; ++it) {
    const double ew = exp(w);
    const double f = w * ew - z;
    const double step = f / (ew * (w + 1.0) - (w + 2.0) * f / (2.0 * w + 2.0));
    w -= step;
    if (fabs(step) <= 1e-16 * fabs(w)) break;
  }
  return w;
}

float clamp_factor(int bit, int gelu) {
  // clamp_op.py:6-8,22-24: lambertw(3 * 4^bit) (Laplace) or lambertw(3 * 4^(bit+1)) (GeLU), cast to f32
  return static_cast<float>(lambert_w0(3.0 * pow(4.0, static_cast<double>(bit + (gelu ? 1 : 0)))));
}

// ------------------------------------------------------------------ pass 1: statistics
__global__ void __launch_bounds__(kQStatThreads)
quant_stats_kernel(const float* __restrict__ x, size_t n, int chunks, double* __restrict__ partials) {
  const int item = blockIdx.y, chunk = blockIdx.x;
  const float* xi = x + static_cast<size_t>(item) * n;
  // chunk boundaries on multiples of 4 elements so the body can use float4 when xi is 16-byte aligned
  const size_t per = ((n + chunks - 1) / chunks + 3) & ~static_cast<size_t>(3);
  const size_t begin = static_cast<size_t>(chunk) * per;
  const size_t end = begin + per < n ? begin + per : n;
  // float4 body when xi is 16-byte aligned, then the scalar rest
  const bool vec = ((reinterpret_cast<uintptr_t>(xi) & 15) == 0);
  const size_t nv = vec && begin < end ? (end - begin) >> 2 : 0;
  const float4* x4 = reinterpret_cast<const float4*>(xi + begin);
  QStats st = QStats::empty();
  for (size_t i = threadIdx.x; i < nv; i += kQStatThreads) st.add(x4[i]);
  for (size_t i = begin + (nv << 2) + threadIdx.x; i < end; i += kQStatThreads) st.add(xi[i]);
  __shared__ double red[kQStatThreads / 32][kQPartialDoubles];
  stats_to_partial(st, red, partials + (static_cast<size_t>(item) * chunks + chunk) * kQPartialDoubles);
}

// ------------------------------------------------------------------ pass 1b: thresholds (one block)
struct QuantHeader {  // lives at the start of the workspace; read by the pack kernel
  float alpha;
  float pad[3];
};

__global__ void quant_finalize_kernel(double* partials, int items, int chunks, size_t n, int clamp,
                                      float factor_laplace, float factor_gelu, QuantHeader* hdr, float* item_min,
                                      float* item_max, float* scale, float* shift, float* alpha_out) {
  // fixed-order reductions -> run-to-run deterministic: one thread per item over its chunks, then
  // thread 0 over the items (the per-item sums are parked in the partials' first chunk slot)
  __shared__ float s_alpha;
  for (int i = threadIdx.x; i < items; i += blockDim.x) {
    const QStats t = fold_item<false>(partials, i, chunks);
    item_min[i] = t.mn;
    item_max[i] = t.mx;
    double* p0 = partials + static_cast<size_t>(i) * chunks * kQPartialDoubles;
    p0[2] = t.s; p0[3] = t.ss; p0[4] = t.ss32;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    const float alpha = fold_items_alpha(items, [&](int i) {
      const double* p0 = partials + static_cast<size_t>(i) * chunks * kQPartialDoubles;
      return QStats{item_min[i], item_max[i], p0[2], p0[3], p0[4]};
    }, n, clamp, factor_laplace, factor_gelu);
    s_alpha = alpha;
    hdr->alpha = alpha;
    if (alpha_out != nullptr) *alpha_out = alpha;
  }
  __syncthreads();
  const float alpha = s_alpha;
  for (int i = threadIdx.x; i < items; i += blockDim.x) item_scale_shift(item_min[i], item_max[i], alpha, scale[i], shift[i]);
}

// ------------------------------------------------------------------ pass 2: quantise + pack
// Fast path: bit in {2,4,8,16} and n % 16 == 0. One thread = 16 consecutive elements (4 x float4 in,
// 16*bit/32 words out as one vector store).
template <int BIT>
__global__ void __launch_bounds__(256)
quant_pack16_kernel(const float* __restrict__ x, size_t n, const QuantHeader* __restrict__ hdr,
                    const float* __restrict__ scale, const float* __restrict__ shift, uint32_t* __restrict__ codes,
                    size_t words_per_item) {
  constexpr int kWords = 16 * BIT / 32;
  const int item = blockIdx.y;
  const size_t groups = n >> 4;
  const float alpha = hdr->alpha;
  const float sh = shift[item], sc = scale[item];
  const float4* xi = reinterpret_cast<const float4*>(x + static_cast<size_t>(item) * n);
  uint32_t* ci = codes + static_cast<size_t>(item) * words_per_item;
  for (size_t g = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; g < groups;
       g += static_cast<size_t>(gridDim.x) * blockDim.x) {
    float4 v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = xi[g * 4 + j];
    pack16<BIT>(v, alpha, sh, sc).store(ci + g * kWords);
  }
}

// Generic path: any bit in [1,16], any n. One thread = one output word (floor(32/bit) codes).
__global__ void __launch_bounds__(256)
quant_pack_generic_kernel(const float* __restrict__ x, size_t n, int bit, const QuantHeader* __restrict__ hdr,
                          const float* __restrict__ scale, const float* __restrict__ shift,
                          uint32_t* __restrict__ codes, size_t words_per_item) {
  const int item = blockIdx.y;
  const int ratio = 32 / bit;
  const float alpha = hdr->alpha;
  const float sh = shift[item], sc = scale[item];
  const float levels = static_cast<float>((1u << bit) - 1u);
  const float* xi = x + static_cast<size_t>(item) * n;
  uint32_t* ci = codes + static_cast<size_t>(item) * words_per_item;
  for (size_t w = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; w < words_per_item;
       w += static_cast<size_t>(gridDim.x) * blockDim.x) {
    uint32_t acc = 0;
    const size_t e0 = w * ratio;
    for (int j = 0; j < ratio; ++j) {
      const size_t e = e0 + j;
      if (e < n) acc |= quant_code(xi[e], alpha, sh, sc, levels) << (j * bit);  // zero-padded tail
    }
    ci[w] = acc;
  }
}

// ------------------------------------------------------------------ decode
__global__ void __launch_bounds__(256)
quant_decode_kernel(const uint32_t* __restrict__ codes, size_t n, int bit, size_t words_per_item,
                    const float* __restrict__ scale, const float* __restrict__ shift, float* __restrict__ out) {
  extern __shared__ float lut[];
  const int item = blockIdx.y;
  const QDecoder dec = fill_dequant_lut(lut, bit);
  const float sc = scale[item], sh = shift[item];
  const uint32_t* ci = codes + static_cast<size_t>(item) * words_per_item;
  float* oi = out + static_cast<size_t>(item) * n;
  for (size_t w = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; w < words_per_item;
       w += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const size_t e0 = w * dec.ratio;
    dec.word(ci[w], e0, n, sc, sh, oi + e0);
  }
}

// ------------------------------------------------------------------ host entry points
static int pick_chunks(int items, size_t n) {
  long want = (2L * kNumSMs + items - 1) / items;
  long by_size = static_cast<long>((n + 4095) / 4096);
  long c = want < by_size ? want : by_size;
  if (c < 1) c = 1;
  if (c > kQMaxChunks) c = kQMaxChunks;
  return static_cast<int>(c);
}

size_t quant_words(size_t n, int bit) {
  if (bit < 1 || bit > 32) return 0;
  const size_t ratio = static_cast<size_t>(32 / bit);
  return (n + ratio - 1) / ratio;
}

size_t quant_workspace_bytes(int items, size_t /*n*/) {
  // header + per-item min/max + partials
  return 256 + static_cast<size_t>(items) * 2 * sizeof(float) + 256 +
         static_cast<size_t>(items) * kQMaxChunks * kQPartialDoubles * sizeof(double);
}

// statistics + thresholds: fills scale/shift (and *alpha) and leaves the QuantHeader at the start of `work`
int quant_stats_impl(const void* x, int items, size_t n, int bit, int clamp, void* scale, void* shift, void* alpha,
                     void* work, cudaStream_t stream) {
  PE_REQUIRE(x && scale && shift && work, "pe_quant: null pointer");
  PE_REQUIRE(items > 0 && n > 0, "pe_quant: empty tensor");
  PE_REQUIRE(bit >= 1 && bit <= 16, "pe_quant: bit=%d outside [1,16]", bit);
  PE_REQUIRE(clamp >= PE_CLAMP_NONE && clamp <= PE_CLAMP_GELU, "pe_quant: bad clamp mode %d", clamp);
  PE_REQUIRE((reinterpret_cast<uintptr_t>(work) & 255) == 0, "pe_quant: workspace must be 256-byte aligned");
  uint8_t* wsp = static_cast<uint8_t*>(work);
  QuantHeader* hdr = reinterpret_cast<QuantHeader*>(wsp);
  float* item_min = reinterpret_cast<float*>(wsp + 256);
  float* item_max = item_min + items;
  const size_t off = (256 + static_cast<size_t>(items) * 2 * sizeof(float) + 255) & ~static_cast<size_t>(255);
  double* partials = reinterpret_cast<double*>(wsp + off);
  const int chunks = pick_chunks(items, n);
  const float* xf = static_cast<const float*>(x);

  quant_stats_kernel<<<dim3(chunks, items), kQStatThreads, 0, stream>>>(xf, n, chunks, partials);
  PE_CUDA(cudaGetLastError());
  quant_finalize_kernel<<<1, 128, 0, stream>>>(partials, items, chunks, n, clamp, clamp_factor(bit, 0),
                                               clamp_factor(bit, 1), hdr, item_min, item_max,
                                               static_cast<float*>(scale), static_cast<float*>(shift),
                                               static_cast<float*>(alpha));
  PE_CUDA(cudaGetLastError());
  count_launches(2);
  return PE_OK;
}

int quant_encode_impl(const void* x, int items, size_t n, int bit, int clamp, void* codes, void* scale, void* shift,
                      void* alpha, void* work, cudaStream_t stream) {
  PE_REQUIRE(codes != nullptr, "pe_quant_encode: null pointer");
  PE_REQUIRE((reinterpret_cast<uintptr_t>(codes) & 15) == 0, "pe_quant_encode: codes must be 16-byte aligned");
  const int rc = quant_stats_impl(x, items, n, bit, clamp, scale, shift, alpha, work, stream);
  if (rc != PE_OK) return rc;
  const QuantHeader* hdr = reinterpret_cast<const QuantHeader*>(work);
  const float* xf = static_cast<const float*>(x);
  const size_t words = quant_words(n, bit);
  uint32_t* cw = static_cast<uint32_t*>(codes);
  if (quant_pack16_applies(bit, n, (reinterpret_cast<uintptr_t>(x) & 15) == 0)) {
    const size_t groups = n / 16;
    size_t bx = (groups + 255) / 256;
    const size_t cap = static_cast<size_t>(kNumSMs) * 8 / static_cast<size_t>(items) + 1;
    if (bx > cap) bx = cap;
    const dim3 grid(static_cast<unsigned>(bx), items);
    const float* sc = static_cast<const float*>(scale);
    const float* sh = static_cast<const float*>(shift);
    switch (bit) {
      case 2: quant_pack16_kernel<2><<<grid, 256, 0, stream>>>(xf, n, hdr, sc, sh, cw, words); break;
      case 4: quant_pack16_kernel<4><<<grid, 256, 0, stream>>>(xf, n, hdr, sc, sh, cw, words); break;
      case 8: quant_pack16_kernel<8><<<grid, 256, 0, stream>>>(xf, n, hdr, sc, sh, cw, words); break;
      default: quant_pack16_kernel<16><<<grid, 256, 0, stream>>>(xf, n, hdr, sc, sh, cw, words); break;
    }
  } else {
    size_t bx = (words + 255) / 256;
    const size_t cap = static_cast<size_t>(kNumSMs) * 8 / static_cast<size_t>(items) + 1;
    if (bx > cap) bx = cap;
    quant_pack_generic_kernel<<<dim3(static_cast<unsigned>(bx), items), 256, 0, stream>>>(
        xf, n, bit, hdr, static_cast<const float*>(scale), static_cast<const float*>(shift), cw, words);
  }
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  return PE_OK;
}

int quant_decode_impl(const void* codes, int items, size_t n, int bit, const void* scale, const void* shift, void* out,
                      cudaStream_t stream) {
  PE_REQUIRE(codes && scale && shift && out, "pe_quant_decode: null pointer");
  PE_REQUIRE(items > 0 && n > 0, "pe_quant_decode: empty tensor");
  PE_REQUIRE(bit >= 1 && bit <= 16, "pe_quant_decode: bit=%d outside [1,16]", bit);
  const size_t words = quant_words(n, bit);
  size_t bx = (words + 255) / 256;
  const size_t cap = static_cast<size_t>(kNumSMs) * 8 / static_cast<size_t>(items) + 1;
  if (bx > cap) bx = cap;
  const size_t smem = bit <= 12 ? (static_cast<size_t>(1) << bit) * sizeof(float) : 0;
  quant_decode_kernel<<<dim3(static_cast<unsigned>(bx), items), 256, smem, stream>>>(
      static_cast<const uint32_t*>(codes), n, bit, words, static_cast<const float*>(scale),
      static_cast<const float*>(shift), static_cast<float*>(out));
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  return PE_OK;
}

}  // namespace pe
