// C-ABI dispatch of the fp32 linear layers (K3): skinny-K stream kernels for in-features <= 16, otherwise the exact-fp32
// SIMT tile kernel.  (Big layers run on the tensor cores through gcbf_linear_*_h, gemm_wgmma_f16.cu.)  Reference op site: gcbf/nn/mlp.py:44-47 (nn.Linear + ReLU chain).
#include <cuda_fp16.h>

#include "common.cuh"

namespace gcbf {
int launch_simt_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma,
                    float* Y, int ldy, int M, int N, int K, int act, cudaStream_t st);
int launch_simt_dgrad(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma,
                      const float* relu_src, int ld_relu, float* dX, int lddx, int M, int N, int K, int accumulate,
                      cudaStream_t st);
int launch_simt_wgrad(const float* dZ, int lddz, const float* X, int ldx, const float* inv_sigma, float* dW, int lddw,
                      float* db, int M, int N, int K, int accumulate, cudaStream_t st);
bool skinny_supported(int K);
int launch_skinny_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, float* Y,
                      int ldy, int M, int N, int K, int act, uint32_t* amax_out, cudaStream_t st);
int launch_skinny_fwd_emit(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, __half* Yh, int ld_h,
                           uint32_t* tile_amax, int amax_stride, int M, int N, int K, int act, cudaStream_t st);
bool tiny_supported(int N, int K);
bool fewrows_supported(int M, int N, int K);
int launch_fewrows_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, float* Y, int ldy, int M,
                       int N, int K, int act, cudaStream_t st);
int launch_fewrows_dgrad(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma, const float* relu_src, int ld_relu,
                         float* dX, int lddx, int M, int N, int K, int accumulate, cudaStream_t st);
bool fewrows_narrow_supported(int M, int N, int K);
int launch_fewrows_dgrad_narrow(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma, const float* relu_src, int ld_relu,
                                float* dX, int lddx, int M, int N, int K, int accumulate, cudaStream_t st);
int launch_fewrows_wgrad(const float* dZ, int lddz, const float* X, int ldx, const float* inv_sigma, float* dW, int lddw, float* db, int M, int N,
                         int K, int accumulate, cudaStream_t st);
int launch_tiny_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, float* Y, int ldy,
                    int M, int N, int K, int act, cudaStream_t st);
int launch_tiny_dgrad(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma, const float* relu_src,
                      int ld_relu, float* dX, int lddx, int M, int N, int K, int accumulate, cudaStream_t st);
int launch_skinny_dgrad(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma, const float* relu_src,
                        int ld_relu, float* dX, int lddx, int M, int N, int K, int accumulate, cudaStream_t st);
int launch_skinny_wgrad(const float* dZ, int lddz, const float* X, int ldx, const float* inv_sigma, float* dW, int lddw,
                        float* db, int M, int N, int K, int accumulate, cudaStream_t st);
}  // namespace gcbf

using namespace gcbf;

static thread_local int g_last_impl = 0;
extern "C" int gcbf_last_gemm_impl(void) { return g_last_impl; }

extern "C" int gcbf_has_wgmma(void) {
#ifdef GCBF_WITH_WGMMA
  return 1;
#else
  return 0;
#endif
}

extern "C" int gcbf_amax_f32(const float* src, int ld, int rows, int cols, void* amax_slot, int accumulate, void* stream);

extern "C" int gcbf_linear_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias,
                               const float* inv_sigma, float* Y, int ldy, int M, int N, int K, int act, int impl,
                               void* out_amax, void* stream) {
  GCBF_REQUIRE(M >= 0 && N > 0 && K > 0 && ldx >= K && ldw >= K && ldy >= N, "gcbf_linear_fwd: bad sizes M=%d N=%d K=%d", M, N, K);
  GCBF_REQUIRE(act >= GCBF_ACT_NONE && act <= GCBF_ACT_TANH, "gcbf_linear_fwd: act %d", act);
  cudaStream_t st = as_stream(stream);
  if (out_amax) GCBF_CUDA_OK(cudaMemsetAsync(out_amax, 0, 4, st));
  if (M == 0) return GCBF_OK;
  GCBF_REQUIRE(X && W && Y, "gcbf_linear_fwd: null pointer");
  if (impl == 2) { set_error("gcbf_linear_fwd: the wgmma path has its own entry point (gcbf_linear_fwd_h)"); return GCBF_E_UNSUPPORTED; }
  if (impl == 0 && skinny_supported(K) && N >= 64 && M >= 64) {   // K <= 16: HBM-bound stream, not a GEMM tile
    g_last_impl = 3;
    return launch_skinny_fwd(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, reinterpret_cast<uint32_t*>(out_amax), st);
  }
  int rc;
  if (impl == 0 && tiny_supported(N, K)) {                         // N <= 32: row-streaming kernel
    g_last_impl = 4;
    rc = launch_tiny_fwd(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, st);
  } else if (impl == 0 && fewrows_supported(M, N, K)) {           // M <= 64: a stream over the weights, not a tile grid
    g_last_impl = 5;
    rc = launch_fewrows_fwd(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, st);
  } else {
    g_last_impl = 1;
    rc = launch_simt_fwd(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, st);
  }
  if (rc == GCBF_OK && out_amax) rc = gcbf_amax_f32(Y, ldy, M, N, out_amax, 1, stream);
  return rc;
}

extern "C" int gcbf_linear_bwd_data(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma,
                                    const float* relu_src, int ld_relu, float* dX, int lddx, int M, int N, int K,
                                    int accumulate, int impl, void* stream) {
  GCBF_REQUIRE(M >= 0 && N > 0 && K > 0 && lddz >= N && ldw >= K && lddx >= K, "gcbf_linear_bwd_data: bad sizes M=%d N=%d K=%d", M, N, K);
  GCBF_REQUIRE(!relu_src || ld_relu >= K, "gcbf_linear_bwd_data: ld_relu");
  if (M == 0) return GCBF_OK;
  GCBF_REQUIRE(dZ && W && dX, "gcbf_linear_bwd_data: null pointer");
  cudaStream_t st = as_stream(stream);
  if (impl == 2) { set_error("gcbf_linear_bwd_data: the wgmma path has its own entry point (gcbf_linear_bwd_data_h)"); return GCBF_E_UNSUPPORTED; }
  if (impl == 0 && skinny_supported(K) && N >= 64 && M >= 64) {
    g_last_impl = 3;
    return launch_skinny_dgrad(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, st);
  }
  if (impl == 0 && tiny_supported(N, K)) {
    g_last_impl = 4;
    return launch_tiny_dgrad(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, st);
  }
  if (impl == 0 && fewrows_supported(M, K, N)) {
    g_last_impl = 5;
    return launch_fewrows_dgrad(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, st);
  }
  if (impl == 0 && fewrows_narrow_supported(M, N, K)) {            // M <= 64 rows, K <= 32 inputs: d edge_attr of a single small graph
    g_last_impl = 5;
    return launch_fewrows_dgrad_narrow(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, st);
  }
  g_last_impl = 1;
  return launch_simt_dgrad(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, st);
}

extern "C" int gcbf_linear_bwd_weight(const float* dZ, int lddz, const float* X, int ldx, const float* inv_sigma,
                                      float* dW, int lddw, float* db, int M, int N, int K, int accumulate, int impl,
                                      void* stream) {
  GCBF_REQUIRE(M >= 0 && N > 0 && K > 0 && lddz >= N && ldx >= K && lddw >= K, "gcbf_linear_bwd_weight: bad sizes M=%d N=%d K=%d", M, N, K);
  GCBF_REQUIRE(dW, "gcbf_linear_bwd_weight: null dW");
  cudaStream_t st = as_stream(stream);
  if (M == 0) {
    if (!accumulate) {
      GCBF_CUDA_OK(cudaMemset2DAsync(dW, (size_t)lddw * 4, 0, (size_t)K * 4, N, st));
      if (db) GCBF_CUDA_OK(cudaMemsetAsync(db, 0, (size_t)N * 4, st));
    }
    return GCBF_OK;
  }
  GCBF_REQUIRE(dZ && X, "gcbf_linear_bwd_weight: null pointer");
  if (impl == 2) { set_error("gcbf_linear_bwd_weight: the wgmma path has its own entry point (gcbf_linear_bwd_weight_h)"); return GCBF_E_UNSUPPORTED; }
  if (impl == 0 && skinny_supported(K) && N >= 64 && M >= 64) {
    g_last_impl = 3;
    return launch_skinny_wgrad(dZ, lddz, X, ldx, inv_sigma, dW, lddw, db, M, N, K, accumulate, st);
  }
  if (impl == 0 && fewrows_supported(M, N, K)) {
    g_last_impl = 5;
    return launch_fewrows_wgrad(dZ, lddz, X, ldx, inv_sigma, dW, lddw, db, M, N, K, accumulate, st);
  }
  g_last_impl = 1;
  return launch_simt_wgrad(dZ, lddz, X, ldx, inv_sigma, dW, lddw, db, M, N, K, accumulate, st);
}

// The skinny-K forward (in-features <= 16: the first phi layer) writing its output as a tile-scaled fp16 companion only -- for a
// tensor-core layer that follows (no fp32 copy, no amax / split pass).  Yh: tile-scaled descriptor (amax strides (ceil(N/256), 1)).
extern "C" int gcbf_linear_fwd_emit(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, int act,
                                    const gcbf_h16* Yh, int M, int N, int K, void* stream) {
  GCBF_REQUIRE(M > 0 && N > 0 && K > 0 && skinny_supported(K) && ldx >= K && ldw >= K, "gcbf_linear_fwd_emit: bad sizes M=%d N=%d K=%d (K <= 16)", M, N, K);
  GCBF_REQUIRE(X && W && Yh && Yh->buf && Yh->amax && Yh->rows == M && Yh->cols == N && Yh->ld >= N && (Yh->ld & 7) == 0 &&
                   (reinterpret_cast<uintptr_t>(Yh->buf) & 15) == 0 && Yh->amax_row_stride == ceil_div(N, 256) && Yh->amax_col_stride == 1,
               "gcbf_linear_fwd_emit: companion descriptor");
  GCBF_REQUIRE(act >= GCBF_ACT_NONE && act <= GCBF_ACT_TANH, "gcbf_linear_fwd_emit: act %d", act);
  g_last_impl = 3;
  return launch_skinny_fwd_emit(X, ldx, W, ldw, bias, inv_sigma, reinterpret_cast<__half*>(Yh->buf), Yh->ld, reinterpret_cast<uint32_t*>(Yh->amax),
                                Yh->amax_row_stride, M, N, K, act, as_stream(stream));
}
