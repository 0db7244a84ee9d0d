// extern "C" surface of libpipeedge_b200.so (declared in include/pipeedge_b200.h): thin wrappers that
// validate, forward to the kernels' host launchers and translate failures into PE_ERR_* codes plus a
// thread-local message.
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>

#include "../../include/pipeedge_b200.h"
#include "common.cuh"

namespace pe {

static thread_local char g_error[512] = "";
static std::atomic<uint64_t> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

int check_cuda(cudaError_t err, const char* what) {
  if (err == cudaSuccess) return PE_OK;
  set_error("CUDA error %d (%s) in %s", static_cast<int>(err), cudaGetErrorString(err), what);
  cudaGetLastError();  // consume it: a stale error must not be blamed on the next, unrelated call
  return PE_ERR_CUDA;
}

bool pdl_enabled() {
  static int cached = -1;
  if (cached < 0) {
    const char* e = getenv("PE_NO_PDL");
    cached = (e != nullptr && e[0] == '1') ? 0 : 1;
  }
  return cached == 1;
}

void count_launches(int n) { g_launches.fetch_add(static_cast<uint64_t>(n), std::memory_order_relaxed); }
uint64_t launch_count_now() { return g_launches.load(std::memory_order_relaxed); }

// The library is built for sm_90a only (wgmma / TMA / cluster PTX, compute capability 9.0): refuse anything else loudly.
int require_sm90() {
  static int cached = 1;  // 1 = unknown
  if (cached == 1) {
    int dev = 0, major = 0;
    if (cudaGetDevice(&dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) {
      set_error("no CUDA device available: pipeedge_b200 has no CPU fallback");
      cudaGetLastError();
      return PE_ERR_DEVICE;
    }
    if (major != 9) {
      set_error("device compute capability major %d is not 9 (sm_90a required)", major);
      return PE_ERR_DEVICE;
    }
    cached = PE_OK;
  }
  return cached;
}

int linear_impl(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n, int k,
                int epilogue, int rows_per_item, int out_item_rows, int out_row_offset, int resid_per_item,
                int static_w, cudaStream_t stream);
int linear_ln_impl(const void* a, const void* w, const void* bias, const void* resid, const void* gamma, const void* beta,
                   float eps, void* out_f32, int f32_is_ln, void* out_f16, int m, int n, int k, int static_w,
                   cudaStream_t stream);
int linear_ln_cluster(int n);
int linear_simt_impl(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n, int k,
                     int epilogue, cudaStream_t stream);
int layernorm_impl(const void* x, const void* resid, const void* gamma, const void* beta, float eps, void* sum_out,
                   void* out_f32, void* out_f16, int rows, int hidden, cudaStream_t stream);
int attention_impl(const void* qkv, void* ctx, int batch, int tokens, int heads, int head_dim, cudaStream_t stream);
int cast_impl(const void* src, void* dst, size_t n, bool to_half, cudaStream_t stream);
size_t quant_words(size_t n, int bit);
size_t quant_workspace_bytes(int items, size_t n);
int quant_encode_impl(const void* x, int items, size_t n, int bit, int clamp, void* codes, void* scale, void* shift,
                      void* alpha, void* work, cudaStream_t stream);
int quant_stats_impl(const void* x, int items, size_t n, int bit, int clamp, void* scale, void* shift, void* alpha,
                     void* work, cudaStream_t stream);
int quant_decode_impl(const void* codes, int items, size_t n, int bit, const void* scale, const void* shift, void* out,
                      cudaStream_t stream);
float clamp_factor(int bit, int gelu);
void set_gemm_trace(void* buf);
int gemm_plan_query(int m, int n, int k, int epilogue, int* out6);

}  // namespace pe

extern "C" {

int pe_abi_version(void) { return PE_ABI_VERSION; }
const char* pe_last_error(void) { return pe::g_error; }
uint64_t pe_launch_count(void) { return pe::g_launches.load(std::memory_order_relaxed); }

int pe_layernorm(const void* x, const void* gamma, const void* beta, float eps, void* out_f32, void* out_f16, int rows,
                 int hidden, void* stream) {
  int rc = pe::require_sm90();
  if (rc != PE_OK) return rc;
  return pe::layernorm_impl(x, nullptr, gamma, beta, eps, nullptr, out_f32, out_f16, rows, hidden,
                            static_cast<cudaStream_t>(stream));
}

int pe_residual_layernorm(const void* y, const void* resid, const void* gamma, const void* beta, float eps,
                          void* sum_out, void* out_f32, void* out_f16, int rows, int hidden, void* stream) {
  int rc = pe::require_sm90();
  if (rc != PE_OK) return rc;
  return pe::layernorm_impl(y, resid, gamma, beta, eps, sum_out, out_f32, out_f16, rows, hidden,
                            static_cast<cudaStream_t>(stream));
}

int pe_linear(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n, int k,
              int epilogue, void* stream) {
  return pe::linear_impl(a, w, bias, resid, out, m, n, k, epilogue & 0xff, 0, 0, 0, 0,
                         /*static_w=*/(epilogue & PE_EPI_STATIC_W) != 0 ? 1 : 0, static_cast<cudaStream_t>(stream));
}

int pe_linear_residual_layernorm(const void* a, const void* w, const void* bias, const void* resid, const void* gamma,
                                 const void* beta, float eps, void* out_f32, int f32_is_ln, void* out_f16, int m, int n,
                                 int k, int static_w, void* stream) {
  return pe::linear_ln_impl(a, w, bias, resid, gamma, beta, eps, out_f32, f32_is_ln, out_f16, m, n, k, static_w,
                            static_cast<cudaStream_t>(stream));
}

int pe_linear_ln_cluster(int n) { return pe::linear_ln_cluster(n); }

int pe_debug_linear_simt(const void* a, const void* w, const void* bias, const void* resid, void* out, int m, int n,
                         int k, int epilogue, void* stream) {
  int rc = pe::require_sm90();
  if (rc != PE_OK) return rc;
  return pe::linear_simt_impl(a, w, bias, resid, out, m, n, k, epilogue, static_cast<cudaStream_t>(stream));
}

int pe_debug_gemm_trace(void* buf) {
  pe::set_gemm_trace(buf);
  return PE_OK;
}

int pe_debug_gemm_plan(int m, int n, int k, int epilogue, int* out6) { return pe::gemm_plan_query(m, n, k, epilogue, out6); }

int pe_attention(const void* qkv, void* ctx, int batch, int tokens, int heads, int head_dim, void* stream) {
  int rc = pe::require_sm90();
  if (rc != PE_OK) return rc;
  return pe::attention_impl(qkv, ctx, batch, tokens, heads, head_dim, static_cast<cudaStream_t>(stream));
}

int pe_cast_f32_to_f16(const void* src, void* dst, size_t n, void* stream) {
  int rc = pe::require_sm90();
  if (rc != PE_OK) return rc;
  return pe::cast_impl(src, dst, n, true, static_cast<cudaStream_t>(stream));
}

int pe_cast_f16_to_f32(const void* src, void* dst, size_t n, void* stream) {
  int rc = pe::require_sm90();
  if (rc != PE_OK) return rc;
  return pe::cast_impl(src, dst, n, false, static_cast<cudaStream_t>(stream));
}

size_t pe_quant_words(size_t n, int bit) { return pe::quant_words(n, bit); }
size_t pe_quant_workspace_bytes(int items, size_t n) { return pe::quant_workspace_bytes(items, n); }
float pe_quant_clamp_factor(int bit, int gelu) { return pe::clamp_factor(bit, gelu); }

int pe_quant_encode(const void* x, int items, size_t n, int bit, int clamp, void* codes, void* scale, void* shift,
                    void* alpha, void* work, void* stream) {
  int rc = pe::require_sm90();
  if (rc != PE_OK) return rc;
  return pe::quant_encode_impl(x, items, n, bit, clamp, codes, scale, shift, alpha, work,
                               static_cast<cudaStream_t>(stream));
}

int pe_quant_alpha(const void* x, int items, size_t n, int bit, int clamp, void* scale, void* shift, void* alpha,
                   void* work, void* stream) {
  int rc = pe::require_sm90();
  if (rc != PE_OK) return rc;
  return pe::quant_stats_impl(x, items, n, bit, clamp, scale, shift, alpha, work, static_cast<cudaStream_t>(stream));
}

int pe_quant_decode(const void* codes, int items, size_t n, int bit, const void* scale, const void* shift, void* out,
                    void* stream) {
  int rc = pe::require_sm90();
  if (rc != PE_OK) return rc;
  return pe::quant_decode_impl(codes, items, n, bit, scale, shift, out, static_cast<cudaStream_t>(stream));
}

}  // extern "C"
