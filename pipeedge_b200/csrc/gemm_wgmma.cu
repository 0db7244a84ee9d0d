// out = epilogue(A @ W^T + bias) on sm_90a tensor cores (wgmma).
//
// One persistent CTA per SM, warp-specialised (Hopper GEMM anatomy):
//   warp 8      TMA producer for the activations: cp.async.bulk.tensor 2D boxes of A [128 x 64] fp16 into a ring of
//               128B-swizzled shared-memory stages, completion on `full` mbarriers (it also arms them with the bytes)
//   warp 9      TMA producer for the weights: boxes of W [BN x 64] into the same stages
//   warps 0..7  two consumer warpgroups: warpgroup g issues wgmma.mma_async (M=64, N=BN, K=16) x4 per stage on rows
//               [64g, 64g+64) of the tile, accumulating fp32 in registers; once a stage's wgmmas have retired
//               (wgmma.wait_group) it is released to its writers (`empty`). After the last K block every warp applies
//               the epilogue to its 16 x BN slice of the accumulator (bias / GELU / residual / LayerNorm) and stores it.
// While the consumers run an epilogue the producers already fill the ring with the next tile's operands.
//
// CTAs may be launched as thread-block CLUSTERS of CM x CN: the CM CTAs that share a W tile each load 1/CM of it and
// TMA-MULTICAST it to the others, likewise the CN CTAs sharing an A tile, cutting L2 reads by up to CM (W) and CN (A).
// Every CTA's `full` barrier sees the bytes of its whole stage whoever issued them; each consumer warpgroup releases a
// stage to all of its writers (remote mbarrier arrivals). The fused projection + residual + LayerNorm uses clusters
// to give one row's column slices to the CN CTAs of a cluster; pe_linear plans single CTAs (see plan_gemm).
//
// Replaces every nn.Linear on the reference path (see include/pipeedge_b200.h: pe_linear).
#include <math.h>
#include <stdio.h>
#include <stdlib.h>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"
#include "ln_dev.cuh"
#include "wgmma.cuh"

namespace pe {

void count_launches(int n);
int require_sm90();

constexpr int kBlockM = 128;
constexpr int kBlockK = 64;  // 64 fp16 = 128 bytes = one SWIZZLE_128B row
constexpr int kMmaK = 16;
constexpr int kNumConsumerWarps = 8;                   // two warpgroups of 64 accumulator rows each
constexpr int kConsumerThreads = kNumConsumerWarps * 32;
constexpr int kProducerWarp = kNumConsumerWarps;       // warp 8: activations (A) + arms the full barriers
constexpr int kWeightWarp = kNumConsumerWarps + 1;     // warp 9: weights (W); never needs the predecessor's data
constexpr int kGemmThreads = (kNumConsumerWarps + 2) * 32;
constexpr int kMaxStages = 8;
constexpr int kTraceSlots = 32;   // pe_debug_gemm_trace: clock64 stamps per CTA
constexpr int kPipeSmemBudget = 144 * 1024;   // operand ring; the epilogue staging follows it
constexpr int kABytes = kBlockM * kBlockK * 2;  // 16 KiB

struct GemmParams {
  const float* bias;
  const float* resid;
  void* out;
  int m, n, k;
  int block_n;
  int stages;
  int num_m_blocks, num_n_blocks, num_k_blocks;
  long long* trace;                // debug: per-CTA clock64 timeline or nullptr
  int cm, cn;                      // cluster shape: CM CTAs along M share a W tile, CN along N share an A tile
  int num_super_m, num_super_n;    // cluster-level tiles (CM*128 x CN*BN)
  // Optional output-row remap (patch embedding writes token rows 1.. of each item and adds a
  // position table that repeats per item). rows_per_item == 0 disables it.
  int rows_per_item;   // GEMM rows per item
  int out_item_rows;   // output rows per item
  int out_row_offset;  // first output row of an item that GEMM row 0 maps to
  int resid_per_item;  // 1: resid is [out_item_rows, n] shared by all items
  int stg_offset;      // byte offset of the epilogue staging from the ring base: 0 = aliases the ring (one tile per CTA)
  int static_w;        // 1: W is not written by anything still pending on the stream -> may be read before pdl_wait()
  // PE_EPI_RESID_LN: v = A W^T + bias + resid, then LayerNorm(v) over the full row (the CN CTAs of a cluster own a row)
  const float* ln_gamma;
  const float* ln_beta;
  float ln_eps;
  int ln_off;          // byte offset (from the ring base) of the row-statistics exchange area
  int f32_is_ln;       // the fp32 output (out) carries LayerNorm(v) (post-LN models) instead of v (pre-LN models)
  __half* out16;       // PE_EPI_RESID_LN: LayerNorm(v) in fp16, or nullptr
};

// [128 rows][4 chunks] float2 chunk statistics + [2][128] float2 CTA statistics (double-buffered) + [128] float2 row
// (mean, rstd)
constexpr int kLnAreaBytes = 8192;

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
// Epilogue GELU (exact-erf form, as the reference's nn.GELU): |error| <= 7e-7 absolute, 4e-6 relative - far below the
// fp16 rounding of the value it feeds (tests/test_kernels_gpu.py compares with torch's erf GELU).
__device__ __forceinline__ float gelu_erf_fast(float x) {
  // gelu(x) = x Phi(x); with E(a) = Phi(-a) = erfc(a / sqrt2) / 2 (a = |x|):  gelu(x) = max(x, 0) - |x| E(|x|).
  // log2 E is smooth: a degree-7 fit on [0, 6] (Chebyshev nodes, scripts/fit_gelu.py) is within 5.7e-6, i.e. E is
  // relatively accurate to 4e-6 INCLUDING the tail that the negative half of GELU lives on. One MUFU (ex2) and 11
  // FMA-pipe instructions; the A&S 7.1.26 form used before needed rcp + ex2 and 13 (the epilogue is MUFU/issue bound).
  const float a = fminf(fabsf(x), 6.0f);
  float pl = fmaf(-1.889626233e-06f, a, 6.268140101e-05f);
  pl = fmaf(pl, a, -9.388679333e-04f);
  pl = fmaf(pl, a, 8.539461332e-03f);
  pl = fmaf(pl, a, -5.402068712e-02f);
  pl = fmaf(pl, a, -4.584097768e-01f);
  pl = fmaf(pl, a, -1.151269147e+00f);
  pl = fmaf(pl, a, -9.999943403e-01f);
  float e;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(pl));
  return fmaxf(x, 0.0f) - fabsf(x * e);
}

constexpr int kStgLd = 36;                        // floats per staged row: 144 B keeps 16-byte accesses conflict-free
constexpr int kLnLdPad = 4;           // PE_EPI_RESID_LN stages a warp's whole 16 x BN slice: BN + 4 floats per row
constexpr int kStgBytesPerWarp = 16 * (128 + kLnLdPad) * 4;
constexpr int kStgBytes = kNumConsumerWarps * kStgBytesPerWarp;

__device__ __forceinline__ void map_rows(const GemmParams& p, int row, int& out_row, int& resid_row) {
  out_row = row;
  resid_row = row;
  if (p.rows_per_item > 0) {
    const int item = row / p.rows_per_item;
    const int in_item = row - item * p.rows_per_item + p.out_row_offset;
    out_row = item * p.out_item_rows + in_item;
    resid_row = p.resid_per_item ? in_item : out_row;
  }
}

template <int EPI>
__device__ __forceinline__ float epi_act(float x) {
  if (EPI == PE_EPI_GELU_F16) return gelu_erf_fast(x);
  if (EPI == PE_EPI_TANH_F32) return tanhf(x);
  return x;
}

// One 16-row x 32-column chunk of the accumulator, already staged row-major in `stg` (this warp's private shared
// memory): re-read it so that consecutive lanes cover consecutive columns of a row, then apply the epilogue and store.
// The wgmma fragment gives each lane two columns of a row; after the transpose each instruction covers whole 64-128
// byte row segments and the residual loads of a chunk are all in flight at once.
template <int EPI>
__device__ __forceinline__ void epilogue_chunk16(const GemmParams& p, const float* stg, int row0, int col0, int lane) {
  constexpr bool kHalfOut = (EPI == PE_EPI_F16 || EPI == PE_EPI_GELU_F16);
  const bool vec_ok = (p.n & 7) == 0;
  if (kHalfOut) {
    // lane -> (row = it*8 + lane/4, 8 columns starting at (lane%4)*8): 16-byte fp16 stores, 64 B per row
    const int cc = (lane & 3) * 8;
    const int col = col0 + cc;
    const bool fast = vec_ok && col + 8 <= p.n;
    float4 b0 = make_float4(0.f, 0.f, 0.f, 0.f), b1 = b0;
    if (p.bias != nullptr && fast) {   // this lane's 8 columns are the same for all of its rows
      b0 = __ldg(reinterpret_cast<const float4*>(p.bias + col));
      b1 = __ldg(reinterpret_cast<const float4*>(p.bias + col + 4));
    }
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      const int rr = it * 8 + (lane >> 2);
      const int row = row0 + rr;
      if (row >= p.m || col >= p.n) continue;
      int out_row, resid_row;
      map_rows(p, row, out_row, resid_row);
      const float4 a = *reinterpret_cast<const float4*>(stg + rr * kStgLd + cc);
      const float4 b = *reinterpret_cast<const float4*>(stg + rr * kStgLd + cc + 4);
      float v[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
      __half* o = reinterpret_cast<__half*>(p.out) + static_cast<size_t>(out_row) * p.n + col;
      if (fast) {
        v[0] += b0.x; v[1] += b0.y; v[2] += b0.z; v[3] += b0.w;
        v[4] += b1.x; v[5] += b1.y; v[6] += b1.z; v[7] += b1.w;
        uint4 pk;
        __half2* h2 = reinterpret_cast<__half2*>(&pk);
#pragma unroll
        for (int i = 0; i < 4; ++i) h2[i] = __floats2half2_rn(epi_act<EPI>(v[2 * i]), epi_act<EPI>(v[2 * i + 1]));
        *reinterpret_cast<uint4*>(o) = pk;
      } else {
        for (int i = 0; i < 8 && col + i < p.n; ++i) {
          float x = v[i];
          if (p.bias != nullptr) x += __ldg(p.bias + col + i);
          o[i] = __float2half_rn(epi_act<EPI>(x));
        }
      }
    }
  } else {
    // lane -> (row = it*4 + lane/8, 4 columns starting at (lane%8)*4): 16-byte fp32 accesses, 128 B per row
    const int cc = (lane & 7) * 4;
    const int col = col0 + cc;
    const bool col_ok = col < p.n;
    const bool fast = vec_ok && col + 4 <= p.n;
    float4 res[4];
#pragma unroll
    for (int it = 0; it < 4; ++it) res[it] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (EPI == PE_EPI_RESID_F32) {
#pragma unroll
      for (int it = 0; it < 4; ++it) {   // all residual loads of the chunk are issued before any is used
        const int row = row0 + it * 4 + (lane >> 3);
        if (row < p.m && fast) {
          int out_row, resid_row;
          map_rows(p, row, out_row, resid_row);
          res[it] = *reinterpret_cast<const float4*>(p.resid + static_cast<size_t>(resid_row) * p.n + col);
        }
      }
    }
    float4 bias4 = make_float4(0.f, 0.f, 0.f, 0.f);
    if (p.bias != nullptr && fast) bias4 = __ldg(reinterpret_cast<const float4*>(p.bias + col));
#pragma unroll
    for (int it = 0; it < 4; ++it) {
      const int rr = it * 4 + (lane >> 3);
      const int row = row0 + rr;
      if (row >= p.m || !col_ok) continue;
      int out_row, resid_row;
      map_rows(p, row, out_row, resid_row);
      const float4 a = *reinterpret_cast<const float4*>(stg + rr * kStgLd + cc);
      float* o = reinterpret_cast<float*>(p.out) + static_cast<size_t>(out_row) * p.n + col;
      if (fast) {
        float4 r4;
        r4.x = epi_act<EPI>(a.x + bias4.x) + res[it].x;
        r4.y = epi_act<EPI>(a.y + bias4.y) + res[it].y;
        r4.z = epi_act<EPI>(a.z + bias4.z) + res[it].z;
        r4.w = epi_act<EPI>(a.w + bias4.w) + res[it].w;
        *reinterpret_cast<float4*>(o) = r4;
      } else {
        const float v[4] = {a.x, a.y, a.z, a.w};
        for (int i = 0; i < 4 && col + i < p.n; ++i) {
          float x = v[i];
          if (p.bias != nullptr) x += __ldg(p.bias + col + i);
          x = epi_act<EPI>(x);
          if (EPI == PE_EPI_RESID_F32) x += p.resid[static_cast<size_t>(resid_row) * p.n + col + i];
          o[i] = x;
        }
      }
    }
  }
}

// Columns [c0, c0 + 8 * J) of this warp's 16 accumulator rows (wgmma fragment: register 4j + {0,1} holds row lane/4,
// columns 8j + 2 (lane % 4) + {0,1}; 4j + {2,3} the same columns of row lane/4 + 8) -> row-major floats with leading
// dimension `ld`.
template <int J, int NACC>
__device__ __forceinline__ void stage_fragment(const float (&acc)[NACC], int j0, float* dst, int ld, int lane) {
  const int r = lane >> 2, c = (lane & 3) * 2;
#pragma unroll
  for (int j = 0; j < J; ++j) {
    *reinterpret_cast<float2*>(dst + r * ld + 8 * j + c) = make_float2(acc[4 * (j0 + j)], acc[4 * (j0 + j) + 1]);
    *reinterpret_cast<float2*>(dst + (r + 8) * ld + 8 * j + c) = make_float2(acc[4 * (j0 + j) + 2], acc[4 * (j0 + j) + 3]);
  }
}

template <int EPI, int BN>
__global__ void __launch_bounds__(kGemmThreads, 1)
gemm_wgmma_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_b, const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];
  __shared__ __align__(8) uint64_t ln_bar[2];     // PE_EPI_RESID_LN: "every CTA of the row has published its statistics"

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  long long* trace = p.trace != nullptr ? p.trace + static_cast<size_t>(blockIdx.x) * kTraceSlots : nullptr;
  if (trace != nullptr && threadIdx.x == 0) trace[0] = clock64();
  pdl_launch_dependents();   // the next kernel may become resident as SMs free up; it blocks in its own pdl_wait()
  // SWIZZLE_128B tiles must start on 1024-byte boundaries
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
  constexpr uint32_t stage_bytes = kABytes + static_cast<uint32_t>(BN) * (kBlockK * 2);

  // position inside the cluster: rank = m_rank + CM * n_rank
  const int csize = p.cm * p.cn;
  const uint32_t crank = csize > 1 ? cluster_ctarank() : 0u;
  const int m_rank = static_cast<int>(crank) % p.cm;
  const int n_rank = static_cast<int>(crank) / p.cm;
  uint16_t row_mask = 0, col_mask = 0;   // CTAs sharing my A tile (same m_rank) / my W tile (same n_rank)
  for (int c = 0; c < p.cn; ++c) row_mask |= static_cast<uint16_t>(1u << (m_rank + p.cm * c));
  for (int m = 0; m < p.cm; ++m) col_mask |= static_cast<uint16_t>(1u << (m + p.cm * n_rank));
  const uint16_t peers_mask = row_mask | col_mask;   // everyone who writes into my stages == everyone I write into

  if (warp == kProducerWarp && lane == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_b);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1);
      // one release per consumer warpgroup of every CTA that reads what this CTA writes into the stage
      mbar_init(&empty_bar[s], static_cast<uint32_t>(2 * (p.cm + p.cn - 1)));
    }
    for (int s = 0; s < 2; ++s) mbar_init(&ln_bar[s], static_cast<uint32_t>(p.cn));
    fence_barrier_init();
  }
  __syncthreads();
  if (csize > 1) cluster_sync_all();   // peers must not multicast into barriers that are not initialised yet
  // Everything above touched only this CTA's shared memory and kernel parameters. The predecessor's output (A via
  // TMA, resid) may be read, and buffers it may still be reading overwritten, only after pdl_wait(): the weight warp
  // first pulls in what does NOT depend on the predecessor (the weights), everyone else waits here.
  if (warp != kWeightWarp || p.static_w == 0) pdl_wait();
  if (trace != nullptr && threadIdx.x == 0) trace[1] = clock64();
  const int num_supers = p.num_super_m * p.num_super_n;
  const int cluster_id = static_cast<int>(blockIdx.x) / csize;
  const int num_clusters = static_cast<int>(gridDim.x) / csize;
  const int a_slice_rows = kBlockM / p.cn;       // my share of the A tile
  const int b_slice_rows = p.block_n / p.cm;     // my share of the W tile

  const uint32_t full_addr0 = keep_in_register(smem_u32(&full_bar[0]));
  const uint32_t empty_addr0 = keep_in_register(smem_u32(&empty_bar[0]));
  const int num_k_blocks = p.num_k_blocks, num_stages = p.stages;
  if (warp == kProducerWarp) {
    // ---------------------------------------------------------------- A producer (warp converged, one lane issues)
    const int cm = p.cm, cn = p.cn, nsm = p.num_super_m;
    const uint32_t a_off = static_cast<uint32_t>(n_rank * a_slice_rows) * (kBlockK * 2);
    int stage = 0;
    uint32_t phase = 0;
    for (int sup = cluster_id; sup < num_supers; sup += num_clusters) {
      const int a_row = ((sup % nsm) * cm + m_rank) * kBlockM + n_rank * a_slice_rows;
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait_addr(empty_addr0 + static_cast<uint32_t>(stage) * 8u, phase ^ 1u);   // all readers drained the stage
        if (elect_one()) {
          const uint32_t f = full_addr0 + static_cast<uint32_t>(stage) * 8u;
          const uint32_t sa = smem_base + static_cast<uint32_t>(stage) * stage_bytes + a_off;
          mbar_arrive_expect_tx_addr(f, stage_bytes);           // A and W bytes; W's complete_tx may already be in
          if (cn > 1) tma_load_2d_multicast_addr(sa, &tm_a, f, kb * kBlockK, a_row, row_mask);
          else tma_load_2d_addr(sa, &tm_a, f, kb * kBlockK, a_row);
        }
        __syncwarp();
        if (++stage == num_stages) { stage = 0; phase ^= 1u; }
      }
    }
  } else if (warp == kWeightWarp) {
    // ---------------------------------------------------------------- W producer (warp converged, one lane issues)
    const int cm = p.cm, cn = p.cn, nsm = p.num_super_m, bn = p.block_n;
    const uint32_t b_off = kABytes + static_cast<uint32_t>(m_rank * b_slice_rows) * (kBlockK * 2);
    // Static weights do not depend on the predecessor kernel: this warp skipped pdl_wait(), so while the predecessor
    // drains it already streams the first stages' weights into shared memory and pulls the rest of its weight panel
    // into L2 (shared out among the CTAs that read the same panel).
    if (p.static_w != 0 && cluster_id < num_supers && elect_one()) {
      const int b_row = ((cluster_id / nsm) * cn + n_rank) * bn + m_rank * b_slice_rows;
      const int sharers = nsm * cm;
      const int me = (cluster_id % nsm) * cm + m_rank;
      for (int kb = num_stages + me; kb < num_k_blocks; kb += sharers) tma_prefetch_l2_2d(&tm_b, kb * kBlockK, b_row);
    }
    __syncwarp();
    int stage = 0;
    uint32_t phase = 0;
    for (int sup = cluster_id; sup < num_supers; sup += num_clusters) {
      const int b_row = ((sup / nsm) * cn + n_rank) * bn + m_rank * b_slice_rows;
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait_addr(empty_addr0 + static_cast<uint32_t>(stage) * 8u, phase ^ 1u);
        if (elect_one()) {
          const uint32_t f = full_addr0 + static_cast<uint32_t>(stage) * 8u;
          const uint32_t sb = smem_base + static_cast<uint32_t>(stage) * stage_bytes + b_off;
          if (cm > 1) tma_load_2d_multicast_addr(sb, &tm_b, f, kb * kBlockK, b_row, col_mask);
          else tma_load_2d_addr(sb, &tm_b, f, kb * kBlockK, b_row);
        }
        __syncwarp();
        if (++stage == num_stages) { stage = 0; phase ^= 1u; }
      }
    }
  } else {
    // -------------------------------------------------------------- consumer warpgroups: main loop + epilogue
    const int wg = warp >> 2;
    const uint32_t a_wg_off = static_cast<uint32_t>(wg * 64) * (kBlockK * 2);   // this warpgroup's 64 rows of A
    // Releasing a stage: one lane of the warpgroup's first warp per CTA that wrote into it (this one included).
    const bool releaser = (warp & 3) == 0 && lane < csize && ((peers_mask >> lane) & 1u) != 0;
    const uint32_t empty_remote0 =
        csize > 1 ? mapa_shared(empty_addr0, static_cast<uint32_t>(lane < csize ? lane : 0)) : empty_addr0;
    float* stg = reinterpret_cast<float*>(smem_gen + p.stg_offset + warp * kStgBytesPerWarp);
    int stage = 0;
    uint32_t phase = 0;
    int par = 0;
    uint32_t ln_phases = 0u;   // bit b: phase of ln_bar[b]
    for (int sup = cluster_id; sup < num_supers; sup += num_clusters) {
      const int m_blk = (sup % p.num_super_m) * p.cm + m_rank;
      const int n_blk = (sup / p.num_super_m) * p.cn + n_rank;
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      int prev_stage = -1;
      for (int kb = 0; kb < num_k_blocks; ++kb) {
        mbar_wait_addr(full_addr0 + static_cast<uint32_t>(stage) * 8u, phase);
        if (trace != nullptr && sup == cluster_id && kb == 0 && threadIdx.x == 0) trace[2] = clock64();
        const uint32_t sa = smem_base + static_cast<uint32_t>(stage) * stage_bytes;
        const uint64_t da = wgmma_desc_kmajor_sw128(sa + a_wg_off);
        const uint64_t db = wgmma_desc_kmajor_sw128(sa + kABytes);
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < kBlockK / kMmaK; ++k)   // K += 16 fp16 = 32 bytes inside the swizzled row: +2 in 16-byte units
          Wgmma<BN>::mma(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
        wgmma_commit();
        wgmma_wait<1>();   // the previous stage's wgmmas have retired: it may be refilled
        if (prev_stage >= 0 && releaser) {
          const uint32_t e = empty_remote0 + static_cast<uint32_t>(prev_stage) * 8u;
          if (csize > 1) mbar_arrive_cluster(e);
          else mbar_arrive_addr(e);
        }
        prev_stage = stage;
        if (++stage == num_stages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      if (releaser) {
        const uint32_t e = empty_remote0 + static_cast<uint32_t>(prev_stage) * 8u;
        if (csize > 1) mbar_arrive_cluster(e);
        else mbar_arrive_addr(e);
      }
      if (trace != nullptr && sup == cluster_id && threadIdx.x == 0) trace[3] = clock64();
      // the staging aliases the ring when each CTA has one tile: the other warpgroup may still be reading it
      if (p.stg_offset == 0) named_barrier<1>(kConsumerThreads);
      const int row0 = m_blk * kBlockM + warp * 16;   // this warp's 16 accumulator rows
      if (EPI == PE_EPI_RESID_LN) {
        // ---- projection + residual add + LayerNorm in one epilogue. The CN CTAs of a cluster hold the CN column
        // slices (BN <= 128) of the same 128 rows. Per row: each 32-column chunk is reduced to (mean, M2) by one thread
        // in index order, chunks are merged per CTA, CTAs exchange (mean, M2) through distributed shared memory (one
        // remote mbarrier arrival per peer), merged in rank order with Chan's update - every CTA derives bit-identical
        // row statistics. Then v (or LayerNorm(v)) goes out as fp32 and LayerNorm(v) as fp16.
        constexpr int kLd = BN + kLnLdPad;
        constexpr int kChunks = BN / 32;
        float2* ln_part = reinterpret_cast<float2*>(smem_gen + p.ln_off);   // [128 rows][4 chunks]
        float2* ln_cta = ln_part + 4 * kBlockM;                             // [2][128], double-buffered by tile parity
        float2* ln_row = ln_cta + 2 * kBlockM;                              // [128] (mean, rstd)
        const int r_cta = warp * 16;                                        // first CTA-local row of this warp
        const int gcol0 = n_blk * BN;
        stage_fragment<BN / 8>(acc, 0, stg, kLd, lane);
        __syncwarp();
        for (int idx = lane; idx < 16 * kChunks; idx += 32) {
          const int r = idx & 15, c = idx >> 4;
          const int row = row0 + r, gcol = gcol0 + c * 32;
          float* vr = stg + r * kLd + c * 32;
          float v[32];
          if (row < p.m) {
            const float4* r4 = reinterpret_cast<const float4*>(p.resid + static_cast<size_t>(row) * p.n + gcol);
            const float4* b4 = reinterpret_cast<const float4*>(p.bias + gcol);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              const float4 a4 = *reinterpret_cast<const float4*>(vr + 4 * i);
              const float4 rv = r4[i], bv = __ldg(b4 + i);
              v[4 * i] = __fadd_rn(__fadd_rn(a4.x, bv.x), rv.x);
              v[4 * i + 1] = __fadd_rn(__fadd_rn(a4.y, bv.y), rv.y);
              v[4 * i + 2] = __fadd_rn(__fadd_rn(a4.z, bv.z), rv.z);
              v[4 * i + 3] = __fadd_rn(__fadd_rn(a4.w, bv.w), rv.w);
            }
          } else {
#pragma unroll
            for (int i = 0; i < 32; ++i) v[i] = 0.f;
          }
#pragma unroll
          for (int i = 0; i < 8; ++i)
            *reinterpret_cast<float4*>(vr + 4 * i) = make_float4(v[4 * i], v[4 * i + 1], v[4 * i + 2], v[4 * i + 3]);
          float mean_c, m2_c;
          ln_chunk32(v, mean_c, m2_c);
          ln_part[(r_cta + r) * 4 + c] = make_float2(mean_c, m2_c);
        }
        __syncwarp();
        if (lane < 16) {   // this CTA's slice of the row: merge its chunks in column order
          const float2 q0 = ln_part[(r_cta + lane) * 4];
          float cnt = 32.f, mean = q0.x, m2 = q0.y;
          for (int c = 1; c < kChunks; ++c) {
            const float2 q = ln_part[(r_cta + lane) * 4 + c];
            ln_merge(cnt, mean, m2, 32.f, q.x, q.y);
          }
          ln_cta[par * kBlockM + r_cta + lane] = make_float2(mean, m2);
        }
        named_barrier<2>(kConsumerThreads);
        if (warp == 0 && lane < p.cn)   // tell every CTA of the row (incl. this one) that my statistics are published
          mbar_arrive_cluster(mapa_shared(smem_u32(&ln_bar[par]), static_cast<uint32_t>(lane)));
        mbar_wait_cluster(&ln_bar[par], (ln_phases >> par) & 1u);
        ln_phases ^= 1u << par;
        if (lane < 16) {
          float cnt = 0.f, mean = 0.f, m2 = 0.f;
          const uint32_t mine = smem_u32(&ln_cta[par * kBlockM + r_cta + lane]);
          const float bn = static_cast<float>(p.block_n);
          for (int j = 0; j < p.cn; ++j) {     // slices in column order (cluster rank = slice index)
            const float2 q = ld_dsmem_f2(mapa_shared(mine, static_cast<uint32_t>(j)));
            ln_merge(cnt, mean, m2, bn, q.x, q.y);
          }
          ln_row[r_cta + lane] = make_float2(mean, ln_rstd(m2, 1.0f / static_cast<float>(p.n), p.ln_eps));
        }
        __syncwarp();
        if (lane < BN / 4) {   // lane -> 4 consecutive columns of every row: 16-byte fp32 / 8-byte fp16 stores
          const int gcol = gcol0 + lane * 4;
          const float4 g4 = __ldg(reinterpret_cast<const float4*>(p.ln_gamma + gcol));
          const float4 e4 = __ldg(reinterpret_cast<const float4*>(p.ln_beta + gcol));
          for (int r = 0; r < 16 && row0 + r < p.m; ++r) {
            const float4 v = *reinterpret_cast<const float4*>(stg + r * kLd + lane * 4);
            const float2 st = ln_row[r_cta + r];
            const float4 ln = make_float4(ln_apply(v.x, st.x, st.y, g4.x, e4.x), ln_apply(v.y, st.x, st.y, g4.y, e4.y),
                                          ln_apply(v.z, st.x, st.y, g4.z, e4.z), ln_apply(v.w, st.x, st.y, g4.w, e4.w));
            const size_t off = static_cast<size_t>(row0 + r) * p.n + gcol;
            if (p.out != nullptr) *reinterpret_cast<float4*>(static_cast<float*>(p.out) + off) = p.f32_is_ln ? ln : v;
            if (p.out16 != nullptr) {
              uint2 pk;
              __half2* h2 = reinterpret_cast<__half2*>(&pk);
              h2[0] = __floats2half2_rn(ln.x, ln.y);
              h2[1] = __floats2half2_rn(ln.z, ln.w);
              *reinterpret_cast<uint2*>(p.out16 + off) = pk;
            }
          }
        }
        par ^= 1;
      } else {
        // ---- registers -> staged 16 x 32 chunk -> (bias, activation, residual, convert) -> coalesced stores
#pragma unroll
        for (int c = 0; c < BN / 32; ++c) {
          const int col0 = n_blk * BN + c * 32;
          stage_fragment<4>(acc, 4 * c, stg, kStgLd, lane);
          __syncwarp();
          if (row0 < p.m && col0 < p.n) epilogue_chunk16<EPI>(p, stg, row0, col0, lane);
          __syncwarp();
        }
      }
      if (trace != nullptr && sup == cluster_id && threadIdx.x == 0) trace[5] = clock64();
    }
  }

  __syncthreads();
  // no CTA may leave while a peer can still multicast into its shared memory or arrive on its barriers
  if (csize > 1) cluster_sync_all();
  if (trace != nullptr && threadIdx.x == 0) trace[6] = clock64();
}

// ------------------------------------------------------------------------------------ host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn == nullptr) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &qres) != cudaSuccess ||
        qres != cudaDriverEntryPointSuccess || ptr == nullptr) {
      set_error("cuTensorMapEncodeTiled is not available from the driver");
      return nullptr;
    }
    fn = reinterpret_cast<EncodeTiledFn>(ptr);
  }
  return fn;
}

// Row-major fp16 [rows, cols] -> boxes of [box_rows, 64] with the 128-byte swizzle; OOB reads give 0.
static int encode_f16_2d(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn fn = get_encode_fn();
  if (fn == nullptr) return PE_ERR_CUDA;
  const cuuint64_t dims[2] = {cols, rows};
  const cuuint64_t strides[1] = {cols * 2};
  const cuuint32_t box[2] = {kBlockK, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult rc = fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr,
                         CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (rc != CUDA_SUCCESS) {
    set_error("cuTensorMapEncodeTiled failed (CUresult %d) for [%llu x %llu] box %u", static_cast<int>(rc),
              static_cast<unsigned long long>(rows), static_cast<unsigned long long>(cols), box_rows);
    return PE_ERR_CUDA;
  }
  return PE_OK;
}

static long long* g_gemm_trace = nullptr;   // set by pe_debug_gemm_trace
void set_gemm_trace(void* buf) { g_gemm_trace = static_cast<long long*>(buf); }

struct GemmPlan {
  int cm, cn, bn;
};

static int max_clusters(int csize) {
  // co-scheduled clusters of 1 CTA/SM kernels: 132 SMs in 66 TPCs, GPCs of 16-18 SMs (clusters never straddle a GPC)
  return csize == 1 ? kNumSMs : (csize == 2 ? kNumSMs / 2 : 128 / csize);
}

// Cost model in SM cycles, from the H100 SXM's dense fp16 tensor rate (~4096 FLOP per cycle per SM) rather than a fit:
//   main loop: K/64 blocks of 4*BN tensor cycles (a 128 x BN x 64 block is 2*128*64*BN FLOP) plus ~150 cycles of
//     barrier / issue latency per block that the two consumer warpgroups do not hide;
//   epilogue of a 128 x BN tile ~800 + c*BN, c growing with the per-element work (GELU and tanh are MUFU / issue bound);
//   tiles are dealt round-robin to <= 132 CTAs; the accumulators live in registers, so a CTA's epilogue is not hidden
//     under its next tile's MMAs (the producers only prefetch that tile's first stages).
// Clusters cut L2 reads but are not L2-bound at these shapes, so pe_linear plans single CTAs; PE_GEMM_FORCE="CM,CN,BN"
// selects any plan (tuning and tests).
GemmPlan plan_gemm(int m, int n, int k, int epilogue) {
  int forced[3] = {0, 0, 0};
  const char* env = getenv("PE_GEMM_FORCE");
  if (env != nullptr && sscanf(env, "%d,%d,%d", &forced[0], &forced[1], &forced[2]) == 3 && forced[0] > 0)
    return {forced[0], forced[1], forced[2]};
  GemmPlan best = {1, 1, 32};
  double best_cost = 1e30;
  const double kb = (k + kBlockK - 1) / kBlockK;
  const double epi_per_col = epilogue == PE_EPI_GELU_F16 ? 14.0 : (epilogue == PE_EPI_TANH_F32 ? 16.0
                             : (epilogue == PE_EPI_RESID_F32 ? 6.0 : 4.0));
  for (int bn = 256; bn >= 32; bn -= 32) {
    const long tiles = static_cast<long>((m + kBlockM - 1) / kBlockM) * ((n + bn - 1) / bn);
    const long rounds = (tiles + kNumSMs - 1) / kNumSMs;       // tiles of the busiest CTA
    const double cost = 3000.0 + rounds * (kb * (150.0 + 4.0 * bn) + 800.0 + epi_per_col * bn);
    if (cost < best_cost - 1e-9) {
      best_cost = cost;
      best = {1, 1, bn};
    }
  }
  return best;
}

template <int EPI, int BN>
static int launch_gemm(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  static bool configured = false;
  // the attribute bounds DYNAMIC shared memory; static barriers live outside it (227 KiB total per CTA)
  const int max_smem = kPipeSmemBudget + kStgBytes + kLnAreaBytes + 1024;
  if (!configured) {
    PE_CUDA(cudaFuncSetAttribute(gemm_wgmma_kernel<EPI, BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem));
    configured = true;
  }
  const uint32_t stage_bytes = kABytes + static_cast<uint32_t>(p.block_n) * (kBlockK * 2);
  const size_t ring = static_cast<size_t>(p.stages) * stage_bytes, stg_end = static_cast<size_t>(p.stg_offset) + kStgBytes;
  size_t smem = (ring > stg_end ? ring : stg_end) + 1024;
  if (EPI == PE_EPI_RESID_LN) smem = static_cast<size_t>(p.ln_off) + kLnAreaBytes + 1024;
  const int csize = p.cm * p.cn;
  const int supers = p.num_super_m * p.num_super_n;
  const int avail = max_clusters(csize);
  const int clusters = supers < avail ? supers : avail;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(static_cast<unsigned>(clusters * csize));
  cfg.blockDim = dim3(kGemmThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[2];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = static_cast<unsigned>(csize);
  attr[0].val.clusterDim.y = 1;
  attr[0].val.clusterDim.z = 1;
  attr[1].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[1].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 2 : 1;
  PE_CUDA(cudaLaunchKernelEx(&cfg, gemm_wgmma_kernel<EPI, BN>, ta, tb, p));
  count_launches(1);
  return PE_OK;
}

// The wgmma tile width is a compile-time operand: one kernel per BN (a multiple of 32 up to kMaxBN).
template <int EPI, int kMaxBN = 256>
static int launch_gemm_bn(const CUtensorMap& ta, const CUtensorMap& tb, const GemmParams& p, cudaStream_t stream) {
  switch (p.block_n) {
    case 32: return launch_gemm<EPI, 32>(ta, tb, p, stream);
    case 64: return launch_gemm<EPI, 64>(ta, tb, p, stream);
    case 96: return launch_gemm<EPI, 96>(ta, tb, p, stream);
    case 128: return launch_gemm<EPI, 128>(ta, tb, p, stream);
    default: break;
  }
  if constexpr (kMaxBN > 128) {
    switch (p.block_n) {
      case 160: return launch_gemm<EPI, 160>(ta, tb, p, stream);
      case 192: return launch_gemm<EPI, 192>(ta, tb, p, stream);
      case 224: return launch_gemm<EPI, 224>(ta, tb, p, stream);
      case 256: return launch_gemm<EPI, 256>(ta, tb, p, stream);
      default: break;
    }
  }
  set_error("pe_linear: no kernel for block_n=%d", p.block_n);
  return PE_ERR_INVALID;
}

// Tile grid, ring depth and staging placement that follow from a plan (shared by the launcher and pe_debug_gemm_plan).
static void fill_geometry(GemmParams& p, const GemmPlan& plan, int m, int n, int k, int reserve = 0) {
  p.m = m; p.n = n; p.k = k;
  p.block_n = plan.bn;
  p.cm = plan.cm;
  p.cn = plan.cn;
  const uint32_t stage_bytes = kABytes + static_cast<uint32_t>(p.block_n) * (kBlockK * 2);
  p.num_m_blocks = (m + kBlockM - 1) / kBlockM;
  p.num_n_blocks = (n + p.block_n - 1) / p.block_n;
  p.num_super_m = (p.num_m_blocks + p.cm - 1) / p.cm;
  p.num_super_n = (p.num_n_blocks + p.cn - 1) / p.cn;
  // One tile per CTA: the epilogue starts only after the last MMA has read the ring, so its staging may alias the
  // ring and the staging's space goes to pipeline depth too. With several tiles per CTA the
  // next tile's loads overlap the epilogue and the two need separate space.
  const bool one_round = p.num_super_m * p.num_super_n <= max_clusters(p.cm * p.cn);
  int stages = ((one_round ? kPipeSmemBudget + kStgBytes : kPipeSmemBudget) - reserve) / static_cast<int>(stage_bytes);
  p.stages = stages > kMaxStages ? kMaxStages : (stages < 2 ? 2 : stages);
  if (const char* cap = getenv("PE_GEMM_STAGES")) {   // tuning scripts only
    const int c = atoi(cap);
    if (c >= 2 && c < p.stages) p.stages = c;
  }
  p.stg_offset = one_round ? 0 : p.stages * static_cast<int>(stage_bytes);
  p.num_k_blocks = (k + kBlockK - 1) / kBlockK;
}

int linear_impl(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n, int k,
                int epilogue, int rows_per_item, int out_item_rows, int out_row_offset, int resid_per_item,
                int static_w, cudaStream_t stream) {
  PE_REQUIRE(a && w && out, "pe_linear: null pointer");
  PE_REQUIRE(m > 0 && n > 0 && k > 0, "pe_linear: bad shape m=%d n=%d k=%d", m, n, k);
  PE_REQUIRE((k & 7) == 0, "pe_linear: k=%d must be a multiple of 8 (16-byte TMA row pitch)", k);
  PE_REQUIRE((reinterpret_cast<uintptr_t>(a) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0,
             "pe_linear: operands must be 16-byte aligned");
  PE_REQUIRE(epilogue != PE_EPI_RESID_F32 || resid != nullptr, "pe_linear: PE_EPI_RESID_F32 needs resid");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;

  const GemmPlan plan = plan_gemm(m, n, k, epilogue);
  PE_REQUIRE(plan.bn >= 32 && plan.bn <= 256 && plan.bn % 32 == 0 && plan.cm >= 1 && plan.cn >= 1 &&
                 plan.cm * plan.cn <= 8 && kBlockM % plan.cn == 0 && (plan.bn / plan.cm) % 8 == 0,
             "pe_linear: bad tile plan cm=%d cn=%d bn=%d", plan.cm, plan.cn, plan.bn);
  GemmParams p = {};
  p.bias = static_cast<const float*>(bias);
  p.resid = static_cast<const float*>(resid);
  p.out = out;
  fill_geometry(p, plan, m, n, k);
  p.trace = g_gemm_trace;
  p.rows_per_item = rows_per_item;
  p.out_item_rows = out_item_rows;
  p.out_row_offset = out_row_offset;
  p.resid_per_item = resid_per_item;
  p.static_w = static_w != 0 ? 1 : 0;

  CUtensorMap ta, tb;   // each CTA loads its SLICE of a tile: 128/CN rows of A, BN/CM rows of W
  rc = encode_f16_2d(&ta, a, static_cast<uint64_t>(m), static_cast<uint64_t>(k), static_cast<uint32_t>(kBlockM / p.cn));
  if (rc != PE_OK) return rc;
  rc = encode_f16_2d(&tb, w, static_cast<uint64_t>(n), static_cast<uint64_t>(k), static_cast<uint32_t>(p.block_n / p.cm));
  if (rc != PE_OK) return rc;
  switch (epilogue) {
    case PE_EPI_F16: return launch_gemm_bn<PE_EPI_F16>(ta, tb, p, stream);
    case PE_EPI_GELU_F16: return launch_gemm_bn<PE_EPI_GELU_F16>(ta, tb, p, stream);
    case PE_EPI_RESID_F32: return launch_gemm_bn<PE_EPI_RESID_F32>(ta, tb, p, stream);
    case PE_EPI_F32: return launch_gemm_bn<PE_EPI_F32>(ta, tb, p, stream);
    case PE_EPI_TANH_F32: return launch_gemm_bn<PE_EPI_TANH_F32>(ta, tb, p, stream);
    default: set_error("pe_linear: unknown epilogue %d", epilogue); return PE_ERR_INVALID;
  }
}

// Cluster width for the fused projection + residual + LayerNorm: the CN CTAs of a cluster own the CN column slices of a
// row, each at most 128 columns wide (a multiple of 32). 0 = this width is not supported.
int linear_ln_cluster(int n) {
  for (int cn = 8; cn >= 1; cn >>= 1)
    if (n % cn == 0 && (n / cn) % 32 == 0 && n / cn <= 128 && kBlockM % cn == 0) return cn;
  return 0;
}

// out_f32 (nullable) = v or LayerNorm(v) (`f32_is_ln`), out_f16 (nullable) = LayerNorm(v), v = a @ w^T + bias + resid.
int linear_ln_impl(const void* a, const void* w, const void* bias, const void* resid, const void* gamma, const void* beta,
                   float eps, void* out_f32, int f32_is_ln, void* out_f16, int m, int n, int k, int static_w,
                   cudaStream_t stream) {
  PE_REQUIRE(a && w && bias && resid && gamma && beta && (out_f32 || out_f16), "pe_linear_residual_layernorm: null pointer");
  PE_REQUIRE(m > 0 && n > 0 && k > 0 && (k & 7) == 0, "pe_linear_residual_layernorm: bad shape m=%d n=%d k=%d", m, n, k);
  const int cn = linear_ln_cluster(n);
  PE_REQUIRE(cn > 0, "pe_linear_residual_layernorm: n=%d is not supported (needs n = cn * bn, cn in {1,2,4,8}, bn %% 32 == 0, bn <= 128)", n);
  PE_REQUIRE((reinterpret_cast<uintptr_t>(a) & 15) == 0 && (reinterpret_cast<uintptr_t>(w) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(resid) & 15) == 0 && (reinterpret_cast<uintptr_t>(bias) & 15) == 0 &&
                 (reinterpret_cast<uintptr_t>(gamma) & 15) == 0 && (reinterpret_cast<uintptr_t>(beta) & 15) == 0 &&
                 (out_f32 == nullptr || (reinterpret_cast<uintptr_t>(out_f32) & 15) == 0) &&
                 (out_f16 == nullptr || (reinterpret_cast<uintptr_t>(out_f16) & 15) == 0),
             "pe_linear_residual_layernorm: operands must be 16-byte aligned");
  int rc = require_sm90();
  if (rc != PE_OK) return rc;
  const GemmPlan plan = {1, cn, n / cn};
  GemmParams p = {};
  p.bias = static_cast<const float*>(bias);
  p.resid = static_cast<const float*>(resid);
  p.out = out_f32;
  p.out16 = static_cast<__half*>(out_f16);
  fill_geometry(p, plan, m, n, k, kLnAreaBytes);
  p.trace = nullptr;
  p.static_w = static_w != 0 ? 1 : 0;
  p.ln_gamma = static_cast<const float*>(gamma);
  p.ln_beta = static_cast<const float*>(beta);
  p.ln_eps = eps;
  p.f32_is_ln = f32_is_ln;
  {
    const uint32_t stage_bytes = kABytes + static_cast<uint32_t>(p.block_n) * (kBlockK * 2);
    const size_t ring = static_cast<size_t>(p.stages) * stage_bytes, stg_end = static_cast<size_t>(p.stg_offset) + kStgBytes;
    p.ln_off = static_cast<int>(((ring > stg_end ? ring : stg_end) + 1023) / 1024 * 1024);
  }
  CUtensorMap ta, tb;
  rc = encode_f16_2d(&ta, a, static_cast<uint64_t>(m), static_cast<uint64_t>(k), static_cast<uint32_t>(kBlockM / p.cn));
  if (rc != PE_OK) return rc;
  rc = encode_f16_2d(&tb, w, static_cast<uint64_t>(n), static_cast<uint64_t>(k), static_cast<uint32_t>(p.block_n));
  if (rc != PE_OK) return rc;
  return launch_gemm_bn<PE_EPI_RESID_LN, 128>(ta, tb, p, stream);
}

// Host-only: the plan and launch geometry pe_linear would use for this shape (no device needed).
// out6 = {cm, cn, block_n, stages, tiles, ctas}.
int gemm_plan_query(int m, int n, int k, int epilogue, int* out6) {
  PE_REQUIRE(out6 != nullptr && m > 0 && n > 0 && k > 0, "pe_debug_gemm_plan: bad arguments");
  PE_REQUIRE(epilogue >= PE_EPI_F16 && epilogue <= PE_EPI_TANH_F32, "pe_debug_gemm_plan: unknown epilogue %d", epilogue);
  const GemmPlan plan = plan_gemm(m, n, k, epilogue);
  GemmParams p = {};
  fill_geometry(p, plan, m, n, k);
  const int supers = p.num_super_m * p.num_super_n, avail = max_clusters(p.cm * p.cn);
  out6[0] = p.cm; out6[1] = p.cn; out6[2] = p.block_n; out6[3] = p.stages;
  out6[4] = p.num_m_blocks * p.num_n_blocks;
  out6[5] = (supers < avail ? supers : avail) * p.cm * p.cn;
  return PE_OK;
}

// ------------------------------------------------------------------- debug reference (CUDA cores)
template <int EPI>
__global__ void gemm_simt_kernel(const __half* __restrict__ a, const __half* __restrict__ w,
                                 const float* __restrict__ bias, const float* resid, void* out, int m, int n, int k) {
  __shared__ float sa[16][17];
  __shared__ float sw[16][17];
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int row = blockIdx.y * 16 + ty, col = blockIdx.x * 16 + tx;
  float acc = 0.f;
  for (int k0 = 0; k0 < k; k0 += 16) {
    const int ar = blockIdx.y * 16 + ty, ac = k0 + tx;
    sa[ty][tx] = (ar < m && ac < k) ? __half2float(a[static_cast<size_t>(ar) * k + ac]) : 0.f;
    const int wr = blockIdx.x * 16 + ty, wc = k0 + tx;
    sw[ty][tx] = (wr < n && wc < k) ? __half2float(w[static_cast<size_t>(wr) * k + wc]) : 0.f;
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk) acc += sa[ty][kk] * sw[tx][kk];
    __syncthreads();
  }
  if (row >= m || col >= n) return;
  if (bias != nullptr) acc += bias[col];
  if (EPI == PE_EPI_GELU_F16) acc = gelu_erf(acc);
  if (EPI == PE_EPI_TANH_F32) acc = tanhf(acc);
  if (EPI == PE_EPI_RESID_F32) acc += resid[static_cast<size_t>(row) * n + col];
  if (EPI == PE_EPI_F16 || EPI == PE_EPI_GELU_F16) {
    reinterpret_cast<__half*>(out)[static_cast<size_t>(row) * n + col] = __float2half_rn(acc);
  } else {
    reinterpret_cast<float*>(out)[static_cast<size_t>(row) * n + col] = acc;
  }
}

int linear_simt_impl(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n, int k,
                     int epilogue, cudaStream_t stream) {
  PE_REQUIRE(a && w && out && m > 0 && n > 0 && k > 0, "pe_debug_linear_simt: bad arguments");
  const dim3 grid((n + 15) / 16, (m + 15) / 16), block(16, 16);
  const __half* ha = static_cast<const __half*>(a);
  const __half* hw = static_cast<const __half*>(w);
  const float* fb = static_cast<const float*>(bias);
  const float* fr = static_cast<const float*>(resid);
  switch (epilogue) {
    case PE_EPI_F16: gemm_simt_kernel<PE_EPI_F16><<<grid, block, 0, stream>>>(ha, hw, fb, fr, out, m, n, k); break;
    case PE_EPI_GELU_F16: gemm_simt_kernel<PE_EPI_GELU_F16><<<grid, block, 0, stream>>>(ha, hw, fb, fr, out, m, n, k); break;
    case PE_EPI_RESID_F32: gemm_simt_kernel<PE_EPI_RESID_F32><<<grid, block, 0, stream>>>(ha, hw, fb, fr, out, m, n, k); break;
    case PE_EPI_F32: gemm_simt_kernel<PE_EPI_F32><<<grid, block, 0, stream>>>(ha, hw, fb, fr, out, m, n, k); break;
    case PE_EPI_TANH_F32: gemm_simt_kernel<PE_EPI_TANH_F32><<<grid, block, 0, stream>>>(ha, hw, fb, fr, out, m, n, k); break;
    default: set_error("pe_debug_linear_simt: unknown epilogue %d", epilogue); return PE_ERR_INVALID;
  }
  PE_CUDA(cudaGetLastError());
  count_launches(1);
  return PE_OK;
}

}  // namespace pe
