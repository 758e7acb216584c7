// C-ABI glue: error text, tunables, device query, linear-layer back-end dispatch.
#include <stdarg.h>
#include <string.h>

#include "common.cuh"

namespace dlrm {

static thread_local char g_err[512] = "";
static int g_tunables[TUNE_COUNT] = {0};

char* err_buf() { return g_err; }

int set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return -1;
}

int get_tunable(int id) { return (id >= 0 && id < TUNE_COUNT) ? g_tunables[id] : 0; }

static unsigned* g_err_word[64] = {nullptr};

unsigned* err_word_device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  if (!g_err_word[dev]) {
    // the only allocation this library ever makes: 4 bytes per device, outside any stream capture
    cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
    cudaThreadExchangeStreamCaptureMode(&mode);
    unsigned* p = nullptr;
    if (cudaMalloc(&p, 256) == cudaSuccess && cudaMemset(p, 0, 256) == cudaSuccess) g_err_word[dev] = p;
    cudaThreadExchangeStreamCaptureMode(&mode);
    (void)cudaGetLastError();
  }
  return g_err_word[dev];
}

int simt_linear_fwd(const float*, long long, const float*, long long, const float*, float*, long long,
                    long long, long long, long long, int, cudaStream_t);
int simt_linear_dgrad(const float*, long long, const float*, long long, const float*, long long, int,
                      float*, long long, long long, long long, long long, cudaStream_t);
int simt_linear_wgrad(const float*, long long, const float*, long long, float*, long long, float*,
                      long long, long long, long long, cudaStream_t);

}  // namespace dlrm

extern "C" int dlrm_b200_abi_version(void) { return DLRM_B200_ABI_VERSION; }
extern "C" const char* dlrm_b200_last_error(void) { return dlrm::err_buf(); }

extern "C" int dlrm_b200_set_tunable(int id, int value) {
  if (id < 0 || id >= dlrm::TUNE_COUNT) return dlrm::set_error("set_tunable: id=%d", id);
  dlrm::g_tunables[id] = value;
  return 0;
}

extern "C" int dlrm_b200_check_device_errors(void* stream) {
  using namespace dlrm;
  unsigned* w = err_word_device();
  if (!w) return 0;
  unsigned h = 0;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  DLRM_CUDA(cudaMemcpyAsync(&h, w, sizeof(h), cudaMemcpyDeviceToHost, st));
  DLRM_CUDA(cudaStreamSynchronize(st));
  if (h) {
    DLRM_CUDA(cudaMemsetAsync(w, 0, sizeof(h), st));
    if (h & 1u) return set_error("an embedding index was outside its table (index out of range in self; the access was "
                                 "redirected to row 0 / skipped, no memory outside the tables was touched)");
    return set_error("device error word = 0x%x", h);
  }
  return 0;
}

extern "C" int dlrm_b200_device_info(int device, int* sm_count, int* cc_major, int* cc_minor) {
  cudaDeviceProp prop;
  DLRM_CUDA(cudaGetDeviceProperties(&prop, device));
  if (sm_count) *sm_count = prop.multiProcessorCount;
  if (cc_major) *cc_major = prop.major;
  if (cc_minor) *cc_minor = prop.minor;
  if (prop.major != 9 || prop.minor != 0)
    return dlrm::set_error("device %d is sm_%d%d; libdlrm_b200 is built for sm_90a (H100) only", device,
                           prop.major, prop.minor);
  return 0;
}

extern "C" int dlrm_b200_linear_fwd(const float* X, int64_t ldx, const float* W, int64_t ldw,
                                    const float* bias, float* Y, int64_t ldy, int64_t M, int64_t N,
                                    int64_t K, int act, int backend, void* stream) {
  using namespace dlrm;
  if (M < 0 || N < 0 || K < 0) return set_error("linear_fwd: negative shape");
  if (act < DLRM_ACT_NONE || act > DLRM_ACT_SIGMOID) return set_error("linear_fwd: act=%d", act);
  if (M == 0 || N == 0) return 0;
  if (!X || !W || !Y) return set_error("linear_fwd: NULL pointer");
  if (backend == DLRM_GEMM_SIMT_FP32)
    return simt_linear_fwd(X, ldx, W, ldw, bias, Y, ldy, M, N, K, act, static_cast<cudaStream_t>(stream));
  return set_error("linear_fwd: backend %d is not available through the fp32-pointer entry point", backend);
}

extern "C" int dlrm_b200_linear_dgrad(const float* dY, int64_t lddy, const float* W, int64_t ldw,
                                      const float* Xact, int64_t ldxa, int act_prev, float* dX,
                                      int64_t lddx, int64_t M, int64_t N, int64_t K, int backend,
                                      void* stream) {
  using namespace dlrm;
  if (M == 0 || K == 0) return 0;
  if (!dY || !W || !dX) return set_error("linear_dgrad: NULL pointer");
  if (act_prev != DLRM_ACT_NONE && !Xact) return set_error("linear_dgrad: act_prev without Xact");
  if (backend == DLRM_GEMM_SIMT_FP32)
    return simt_linear_dgrad(dY, lddy, W, ldw, Xact, ldxa, act_prev, dX, lddx, M, N, K,
                             static_cast<cudaStream_t>(stream));
  return set_error("linear_dgrad: backend %d is not available through the fp32-pointer entry point", backend);
}

extern "C" int dlrm_b200_linear_wgrad(const float* dY, int64_t lddy, const float* X, int64_t ldx,
                                      float* dW, int64_t lddw, float* dbias, int64_t M, int64_t N,
                                      int64_t K, int backend, void* stream) {
  using namespace dlrm;
  if (N == 0) return 0;
  if (!dY || !X || !dW) return set_error("linear_wgrad: NULL pointer");
  if (backend == DLRM_GEMM_SIMT_FP32)
    return simt_linear_wgrad(dY, lddy, X, ldx, dW, lddw, dbias, M, N, K, static_cast<cudaStream_t>(stream));
  return set_error("linear_wgrad: backend %d is not available through the fp32-pointer entry point", backend);
}
