// Stage-0 edges of the pipeline (SURVEY.md 8a-A13): patch embedding for ViT/DeiT and the BERT embedding
// gather + LayerNorm. Small, HBM-bound kernels around one wgmma GEMM.
//   ViT/DeiT: HF ViTEmbeddings/DeiTEmbeddings = Conv2d(C, H, P, stride P) -> flatten -> [CLS (, DIST)] ++ patches, + pos.
//             The strided conv is a GEMM over im2col'ed patches: [B*Np, C*P*P] x [H, C*P*P]^T; its epilogue adds
//             the conv bias and the position rows and scatters into token rows n_prefix.. of each item.
//   BERT:     HF BertEmbeddings = LN(word[id] + type[0] + pos[position_ids[s]]).
#include "../../include/pipeedge_b200.h"
#include "common.cuh"

namespace pe {

void count_launches(int n);
int require_sm90();
int linear_impl(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n, int k,
                int epilogue, int rows_per_item, int out_item_rows, int out_row_offset, int resid_per_item,
                int static_w, cudaStream_t stream);

// pixels f32 [B, C, img, img] -> patches f16 [B * np_side^2, kpad]; column = c*P*P + i*P + j (the flattened
// Conv2d weight order), zero-padded up to kpad.
__global__ void im2col_patches_kernel(const float* __restrict__ pix, __half* __restrict__ out, int channels, int img,
                                      int patch, int np_side, int kdim, int kpad, size_t total) {
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int col = static_cast<int>(idx % kpad);
    const size_t row = idx / kpad;
    float v = 0.f;
    if (col < kdim) {
      const int j = col % patch, i = (col / patch) % patch, c = col / (patch * patch);
      const int np = np_side * np_side;
      const int p = static_cast<int>(row % np);
      const size_t b = row / np;
      const int py = p / np_side, px = p % np_side;
      v = pix[((b * channels + c) * img + (py * patch + i)) * static_cast<size_t>(img) + (px * patch + j)];
    }
    out[idx] = __float2half_rn(v);
  }
}

// out[b, r, :] = prefix[r, :] for the n_prefix leading token rows (CLS / distillation token, position
// already added by the caller when it built `prefix`).
__global__ void prefix_rows_kernel(const float* __restrict__ prefix, float* __restrict__ out, int n_prefix, int tokens,
                                   int hidden, int batch) {
  const size_t total = static_cast<size_t>(batch) * n_prefix * hidden;
  for (size_t idx = blockIdx.x * static_cast<size_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<size_t>(gridDim.x) * blockDim.x) {
    const int h = static_cast<int>(idx % hidden);
    const int r = static_cast<int>((idx / hidden) % n_prefix);
    const size_t b = idx / (static_cast<size_t>(hidden) * n_prefix);
    out[(b * tokens + r) * hidden + h] = prefix[static_cast<size_t>(r) * hidden + h];
  }
}

// One warp per token: gather the three embedding rows, sum in the reference's order, LayerNorm (two-pass).
constexpr int kEmbMaxVec = 12;
__global__ void __launch_bounds__(128)
bert_embed_kernel(const long long* __restrict__ ids, const long long* __restrict__ pos_ids,
                  const float* __restrict__ word, const float* __restrict__ type0, const float* __restrict__ pos,
                  const float* __restrict__ gamma, const float* __restrict__ beta, float eps, float* __restrict__ out,
                  int rows, int seq, int hidden) {
  const int row = blockIdx.x * 4 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const int nvec = hidden >> 2;
  const long long id = ids[row];
  const long long pid = pos_ids[row % seq];
  const float4* w4 = reinterpret_cast<const float4*>(word + static_cast<size_t>(id) * hidden);
  const float4* t4 = reinterpret_cast<const float4*>(type0);
  const float4* p4 = reinterpret_cast<const float4*>(pos + static_cast<size_t>(pid) * hidden);
  float4 v[kEmbMaxVec];
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < kEmbMaxVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      const float4 a = w4[idx], b = __ldg(t4 + idx), c = p4[idx];
      // (inputs_embeds + token_type_embeddings) + position_embeddings (HF modeling_bert.py:104-108)
      v[i] = make_float4((a.x + b.x) + c.x, (a.y + b.y) + c.y, (a.z + b.z) + c.z, (a.w + b.w) + c.w);
      sum += (v[i].x + v[i].y) + (v[i].z + v[i].w);
    }
  }
  const float mean = warp_sum(sum) / static_cast<float>(hidden);
  float sq = 0.f;
#pragma unroll
  for (int i = 0; i < kEmbMaxVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      const float a = v[i].x - mean, b = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      sq += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = 1.0f / sqrtf(warp_sum(sq) / static_cast<float>(hidden) + eps);
#pragma unroll
  for (int i = 0; i < kEmbMaxVec; ++i) {
    const int idx = lane + i * 32;
    if (idx < nvec) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(gamma) + idx);
      const float4 b = __ldg(reinterpret_cast<const float4*>(beta) + idx);
      float4 o;
      o.x = (v[i].x - mean) * rstd * g.x + b.x;
      o.y = (v[i].y - mean) * rstd * g.y + b.y;
      o.z = (v[i].z - mean) * rstd * g.z + b.z;
      o.w = (v[i].w - mean) * rstd * g.w + b.w;
      reinterpret_cast<float4*>(out + static_cast<size_t>(row) * hidden)[idx] = o;
    }
  }
}

}  // namespace pe

extern "C" {

int pe_patch_embed(const void* pixels, const void* w, const void* bias, const void* pos, const void* prefix, void* out,
                   void* patches_work, int batch, int channels, int img, int patch, int hidden, int n_prefix,
                   void* stream_v) {
  using namespace pe;
  PE_REQUIRE(pixels && w && bias && pos && prefix && out && patches_work, "pe_patch_embed: null pointer");
  PE_REQUIRE(batch > 0 && channels > 0 && patch > 0 && img % patch == 0 && hidden % 8 == 0 && n_prefix >= 1,
             "pe_patch_embed: bad shape");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;
  cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
  const int np_side = img / patch, np = np_side * np_side;
  const int kdim = channels * patch * patch;
  const int kpad = (kdim + 7) & ~7;
  const int tokens = np + n_prefix;
  const size_t total = static_cast<size_t>(batch) * np * kpad;
  const int grid = static_cast<int>((total + 255) / 256 > static_cast<size_t>(kNumSMs) * 16
                                        ? static_cast<size_t>(kNumSMs) * 16 : (total + 255) / 256);
  im2col_patches_kernel<<<grid, 256, 0, stream>>>(static_cast<const float*>(pixels), static_cast<__half*>(patches_work),
                                                  channels, img, patch, np_side, kdim, kpad, total);
  PE_CUDA(cudaGetLastError());
  const size_t ptotal = static_cast<size_t>(batch) * n_prefix * hidden;
  prefix_rows_kernel<<<static_cast<int>((ptotal + 255) / 256), 256, 0, stream>>>(
      static_cast<const float*>(prefix), static_cast<float*>(out), n_prefix, tokens, hidden, batch);
  PE_CUDA(cudaGetLastError());
  count_launches(2);
  // out[b, n_prefix + p, :] = patches[b*np + p, :] @ w^T + bias + pos[n_prefix + p, :]
  return linear_impl(patches_work, w, bias, pos, out, batch * np, hidden, kpad, PE_EPI_RESID_F32, np, tokens, n_prefix, 1,
                     /*static_w=*/0, stream);
}

int pe_bert_embed(const void* ids, const void* pos_ids, const void* word, const void* type0, const void* pos,
                  const void* gamma, const void* beta, float eps, void* out, int batch, int seq, int hidden,
                  void* stream_v) {
  using namespace pe;
  PE_REQUIRE(ids && pos_ids && word && type0 && pos && gamma && beta && out, "pe_bert_embed: null pointer");
  PE_REQUIRE(batch > 0 && seq > 0 && hidden % 4 == 0 && hidden <= kEmbMaxVec * 128, "pe_bert_embed: bad shape");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;
  const int rows = batch * seq;
  bert_embed_kernel<<<(rows + 3) / 4, 128, 0, static_cast<cudaStream_t>(stream_v)>>>(
      static_cast<const long long*>(ids), static_cast<const long long*>(pos_ids), static_cast<const float*>(word),
      static_cast<const float*>(type0), static_cast<const float*>(pos), static_cast<const float*>(gamma),
      static_cast<const float*>(beta), eps, static_cast<float*>(out), rows, seq, hidden);
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  return PE_OK;
}

}  // extern "C"
