// Shared device helpers for the sm_90a kernels: mbarrier, TMA, clusters, wgmma synchronisation and descriptors,
// warp reductions and the status/error plumbing of the C-ABI.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace pe {

// ---------------------------------------------------------------- status / errors (api.cu)
void set_error(const char* fmt, ...);
int check_cuda(cudaError_t err, const char* what);
#define PE_CUDA(call)                                  \
  do {                                                 \
    int _rc = ::pe::check_cuda((call), #call);         \
    if (_rc != 0) return _rc;                          \
  } while (0)
#define PE_REQUIRE(cond, ...)                          \
  do {                                                 \
    if (!(cond)) {                                     \
      ::pe::set_error(__VA_ARGS__);                    \
      return PE_ERR_INVALID;                           \
    }                                                  \
  } while (0)

// ---------------------------------------------------------------- stream sockets (hop.cu)
// Send / receive all n bytes, retrying on EINTR: 0 ok, -1 error (errno says why); read_all returns 1 at EOF.
int write_all(int fd, const void* buf, size_t n);
int read_all(int fd, void* buf, size_t n);

constexpr int kNumSMs = 132;  // H100 SXM

// ---------------------------------------------------------------- small utilities
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ int lane_id() { return threadIdx.x & 31; }

template <typename T, typename Op>
__device__ __forceinline__ T warp_reduce(T v, Op op) {
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, off));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
  return warp_reduce(v, [](float a, float b) { return a + b; });
}
__device__ __forceinline__ float warp_max(float v) {
  return warp_reduce(v, [](float a, float b) { return fmaxf(a, b); });
}

// ---------------------------------------------------------------- programmatic dependent launch (PDL)
// Every kernel of the stage path is launched with programmatic stream serialisation: it may become resident while
// its predecessor is still draining, runs its private prologue (barrier init, descriptor prefetch) and then
// blocks in pdl_wait() until the predecessor has completed and its writes are visible. Rules (stage.cu relies on them):
// no global read of produced data and no global write before pdl_wait(); every PDL-launched kernel calls pdl_wait()
// on every thread that touches global memory, so completion stays transitive along the stream.
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

bool pdl_enabled();   // api.cu: on unless PE_NO_PDL=1

// Launch `kernel` with the PDL attribute (when enabled) on `stream`.
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                              Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
// ---- lean variants for the single-issuer hot loops: 32-bit shared addresses computed once, the spin lives in
// PTX (a handful of instructions per retry). A lone warp issues roughly one dependent instruction every 6-8
// cycles, so every instruction in those loops costs as much as ~1/64 of a 128x256x64 MMA block.
__device__ __forceinline__ bool elect_one() {
  uint32_t pred;
  asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
  return pred != 0;
}
// Bounded (2^24 retries of a hardware-suspending try_wait ~ seconds) so that a protocol bug traps instead of hanging.
__device__ __forceinline__ void mbar_wait_addr(uint32_t bar_addr, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\tmov.u32 n, 0;\n"
      "PE_WAIT:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra PE_DONE;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.lt.u32 p, n, 16777216;\n\t"
      "@p bra PE_WAIT;\n\t"
      "trap;\n"
      "PE_DONE:\n\t}"
      ::"r"(bar_addr), "r"(parity)
      : "memory");
}
// Both phases complete? The two try_waits are issued back to back, so their ~100-cycle result latencies overlap; a
// miss (returns 0) falls back to mbar_wait_addr on each.
__device__ __forceinline__ uint32_t mbar_try2_addr(uint32_t bar0, uint32_t parity0, uint32_t bar1, uint32_t parity1) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred q0, q1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 q0, [%1], %2;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 q1, [%3], %4;\n\t"
      "and.pred q0, q0, q1;\n\t"
      "selp.u32 %0, 1, 0, q0;\n\t}"
      : "=r"(ok)
      : "r"(bar0), "r"(parity0), "r"(bar1), "r"(parity1)
      : "memory");
  return ok;
}
// Keeps a loop-invariant shared-memory address in a register: without it the compiler re-derives the address inside
// the loop (S2UR SR_CgaCtaId + shifts for every use of a __shared__ symbol's shared-window address).
__device__ __forceinline__ uint32_t keep_in_register(uint32_t x) {
  asm volatile("mov.u32 %0, %0;" : "+r"(x));
  return x;
}
__device__ __forceinline__ void mbar_arrive_addr(uint32_t bar_addr) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar_addr) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx_addr(uint32_t bar_addr, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_addr), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d_addr(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar_addr, int c0,
                                                 int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar_addr), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d_multicast_addr(uint32_t smem_dst, const CUtensorMap* map, uint32_t bar_addr,
                                                           int c0, int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar_addr), "r"(c0), "r"(c1), "h"(cta_mask)
      : "memory");
}
// ---------------------------------------------------------------- TMA
// Pull one box of a tensor into L2 without a shared-memory destination (weights ahead of their first use).
__device__ __forceinline__ void tma_prefetch_l2_2d(const CUtensorMap* map, int c0, int c1) {
  asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}
// 2D tiled load, global -> shared, completion signalled on `bar` (complete_tx::bytes).
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                            int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
      : "memory");
}

// 2D tiled load multicast to every CTA of the cluster named in `cta_mask`: the box lands at the same
// CTA-relative shared-memory offset in each destination and completes on each destination's own mbarrier.
__device__ __forceinline__ void tma_load_2d_multicast(void* smem_dst, const CUtensorMap* map, uint64_t* bar, int c0,
                                                      int c1, uint16_t cta_mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster"
      " [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(smem_u32(smem_dst)), "l"(reinterpret_cast<uint64_t>(map)), "r"(smem_u32(bar)), "r"(c0), "r"(c1),
        "h"(cta_mask)
      : "memory");
}

// 2D tiled store, shared -> global (bulk async group of the issuing thread); out-of-bounds parts are clipped.
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t smem_src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(map)), "r"(smem_src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// the issuing thread's stores have finished READING shared memory (it may be overwritten)
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// ... have completed entirely
__device__ __forceinline__ void tma_store_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// ---------------------------------------------------------------- clusters
__device__ __forceinline__ uint32_t cluster_ctarank() {
  uint32_t r;
  asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
  return r;
}
__device__ __forceinline__ void cluster_sync_all() {
  asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
  asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// distributed shared memory: the address of the same shared-memory location in CTA `rank` of this cluster
__device__ __forceinline__ uint32_t mapa_shared(uint32_t addr, uint32_t rank) {
  uint32_t r;
  asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(addr), "r"(rank));
  return r;
}
__device__ __forceinline__ float2 ld_dsmem_f2(uint32_t cluster_addr) {
  float2 v;
  asm volatile("ld.shared::cluster.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "r"(cluster_addr) : "memory");
  return v;
}
// arrive on an mbarrier of another CTA of the cluster; orders this CTA's earlier shared-memory writes before it
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t cluster_bar_addr) {
  asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar_addr) : "memory");
}
// arrive on an mbarrier of another CTA of the cluster with the default CTA-scope release: for a consumer handing a ring
// stage back to the CTA that refills it, where the only order needed (its reads of the stage are done) comes from the
// wgmma.wait_group before it. The cluster-scope release above makes every arrival wait for this CTA's outstanding
// memory operations to become visible cluster-wide, which stalls the releasing warp once per stage.
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_bar_addr) {
  asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_bar_addr) : "memory");
}
// wait on this CTA's mbarrier with cluster-scope acquire (pairs with mbar_arrive_cluster); bounded like mbar_wait_addr
// and without a printf, which would be a function call that serialises the caller's wgmma pipeline
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .u32 n;\n\tmov.u32 n, 0;\n"
      "PE_WAITC:\n\t"
      "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra PE_DONEC;\n\t"
      "add.u32 n, n, 1;\n\t"
      "setp.lt.u32 p, n, 16777216;\n\t"
      "@p bra PE_WAITC;\n\t"
      "trap;\n"
      "PE_DONEC:\n\t}"
      ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
// named barrier among `threads` threads of the CTA (ids 1..15; 0 is __syncthreads)
template <int kId>
__device__ __forceinline__ void named_barrier(int threads) {
  asm volatile("bar.sync %0, %1;" ::"n"(kId), "r"(threads) : "memory");
}
// the same with a barrier id known only at run time (e.g. one per warpgroup)
__device__ __forceinline__ void named_barrier_id(int id, int threads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(threads) : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA)
// Order this thread's earlier register / shared-memory accesses before the wgmma instructions that follow.
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most N of this warpgroup's committed wgmma groups are still in flight
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Shared-memory matrix descriptor for a K-major fp16 tile stored as rows of 128 bytes with the 128-byte swizzle (what a
// TMA box of 64 fp16 x R rows with CU_TENSOR_MAP_SWIZZLE_128B writes): 8-row groups are 1024 bytes apart (SBO); LBO is
// unused for swizzled K-major layouts. Field layout of the PTX ISA wgmma matrix descriptor; the tile must start on a
// 1024-byte boundary (base offset 0). Advancing K by 16 fp16 inside the swizzled row adds 32 bytes to the start address.
__device__ __forceinline__ uint64_t wgmma_desc_kmajor_sw128(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((smem_addr & 0x3FFFFu) >> 4);  // start address  [0,14)
  d |= static_cast<uint64_t>(1) << 16;                      // LBO (ignored)  [16,30)
  d |= static_cast<uint64_t>(1024 >> 4) << 32;              // SBO = 1024 B   [32,46)
  d |= static_cast<uint64_t>(1) << 62;                      // SWIZZLE_128B   [62,64)
  return d;
}

}  // namespace pe
