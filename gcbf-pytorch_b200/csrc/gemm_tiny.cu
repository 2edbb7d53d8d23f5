// Tiny-output linear layers: out-features N <= 32 (gate 128 -> 1, heads 128 -> 32 -> 1 | 2; reference gcbf/nn/gnn.py:17-19,
// gcbf/algo/gcbf.py:30-35, gcbf/controller/gnn_controller.py:27).  A 128 x 128 GEMM tile would be > 75 % padding and these
// layers are pure HBM streams over the [M, K] side, so:
//   fwd   : Y[M,N]  = act(alpha * X[M,K] W[N,K]^T + b)     warp = row, lanes sweep K (coalesced), W in shared memory,
//                                                          one shuffle reduction per output column
//   dgrad : dX[M,K] (+)= alpha * dZ[M,N] W[N,K] (* mask)   warp = row, lane n holds dZ[m][n], broadcast by shuffle
//   colsum: db[N]   = sum_m dZ[m][n]                       thread = row, N register accumulators (bias gradient)
// The weight gradient of these layers stays on the SIMT tile kernel (a real [N,K] x M reduction).
#include "common.cuh"

namespace gcbf {

constexpr int TINY_MAX_N = 32;
constexpr int TINY_MAX_K = 256;

bool tiny_supported(int N, int K) { return N <= TINY_MAX_N && K <= TINY_MAX_K; }

// W[N,K] -> shared [N][KP] (KP = KI*32, zero padded)
template <int KI>
__device__ __forceinline__ void load_w(float* wsm, const float* __restrict__ W, int ldw, int N, int K) {
  constexpr int KP = KI * 32;
  for (int i = threadIdx.x; i < N * KP; i += blockDim.x) {
    const int n = i / KP, k = i % KP;
    wsm[i] = (k < K) ? __ldg(W + (size_t)n * ldw + k) : 0.f;
  }
  __syncthreads();
}

template <int KI>
__global__ void __launch_bounds__(256) tiny_fwd_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ W, int ldw,
                                                       const float* __restrict__ bias, const float* __restrict__ alpha_p,
                                                       float* __restrict__ Y, int ldy, int M, int N, int K, int act) {
  constexpr int KP = KI * 32;
  extern __shared__ float wsm[];
  load_w<KI>(wsm, W, ldw, N, K);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  const float b = (bias && lane < N) ? __ldg(bias + lane) : 0.f;
  for (int row = blockIdx.x * 8 + warp; row < M; row += gridDim.x * 8) {
    float x[KI];
#pragma unroll
    for (int i = 0; i < KI; ++i) {
      const int k = lane + 32 * i;
      x[i] = (k < K) ? __ldg(X + (size_t)row * ldx + k) : 0.f;
    }
    float out = 0.f;
    for (int n = 0; n < N; ++n) {
      float p = 0.f;
#pragma unroll
      for (int i = 0; i < KI; ++i) p = fmaf(x[i], wsm[n * KP + lane + 32 * i], p);
      p = warp_sum(p);
      if (lane == n) out = p;
    }
    if (lane < N) {
      float y = fmaf(alpha, out, b);
      if (act == GCBF_ACT_RELU) y = fmaxf(y, 0.f);
      else if (act == GCBF_ACT_TANH) y = tanhf(y);
      Y[(size_t)row * ldy + lane] = y;
    }
  }
}

template <int KI>
__global__ void __launch_bounds__(256) tiny_dgrad_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ W,
                                                         int ldw, const float* __restrict__ alpha_p,
                                                         const float* __restrict__ relu_src, int ld_relu, float* __restrict__ dX,
                                                         int lddx, int M, int N, int K, int accumulate) {
  constexpr int KP = KI * 32;
  extern __shared__ float wsm[];
  load_w<KI>(wsm, W, ldw, N, K);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  for (int row = blockIdx.x * 8 + warp; row < M; row += gridDim.x * 8) {
    const float dz = (lane < N) ? __ldg(dZ + (size_t)row * lddz + lane) : 0.f;
    float acc[KI];
#pragma unroll
    for (int i = 0; i < KI; ++i) acc[i] = 0.f;
    for (int n = 0; n < N; ++n) {
      const float d = __shfl_sync(0xffffffffu, dz, n);
#pragma unroll
      for (int i = 0; i < KI; ++i) acc[i] = fmaf(d, wsm[n * KP + lane + 32 * i], acc[i]);
    }
#pragma unroll
    for (int i = 0; i < KI; ++i) {
      const int k = lane + 32 * i;
      if (k < K) {
        float v = alpha * acc[i];
        if (relu_src && !(__ldg(relu_src + (size_t)row * ld_relu + k) > 0.f)) v = 0.f;
        float* dst = dX + (size_t)row * lddx + k;
        *dst = accumulate ? *dst + v : v;
      }
    }
  }
}

// column sums of a narrow matrix (N <= 32): thread = row (N loads that stay in the same L1 lines), block reduction,
// one atomic per column per block
__global__ void __launch_bounds__(256) colsum_narrow_kernel(const float* __restrict__ dZ, int ld, int M, int N,
                                                            float* __restrict__ db) {
  __shared__ float part[8][TINY_MAX_N];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float s[TINY_MAX_N];
#pragma unroll
  for (int n = 0; n < TINY_MAX_N; ++n) s[n] = 0.f;
  for (int r = blockIdx.x * 256 + threadIdx.x; r < M; r += gridDim.x * 256) {
    const float* p = dZ + (size_t)r * ld;
#pragma unroll
    for (int n = 0; n < TINY_MAX_N; ++n)
      if (n < N) s[n] += __ldg(p + n);
  }
#pragma unroll
  for (int n = 0; n < TINY_MAX_N; ++n) {
    if (n < N) {
      const float t = warp_sum(s[n]);
      if (lane == 0) part[warp][n] = t;
    }
  }
  __syncthreads();
  if (threadIdx.x < N) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) t += part[w][threadIdx.x];
    db[(size_t)blockIdx.x * N + threadIdx.x] = t;      // this block's partial; summed in order by add_partials
  }
}

int launch_colsum_narrow(const float* dZ, int ld, int M, int N, float* db, int accumulate, cudaStream_t st) {
  const int blocks = (int)imax64(1, imin64(ceil_div(M, 256), 2 * kNumSMs));
  float* part = nullptr;
  GCBF_CUDA_OK(scratch_alloc((void**)&part, (size_t)blocks * N * 4, st));
  colsum_narrow_kernel<<<blocks, 256, 0, st>>>(dZ, ld, M, N, part);
  GCBF_LAUNCH_OK();
  GCBF_CUDA_OK(add_partials(part, blocks, 1, N, db, N, accumulate, st));
  GCBF_CUDA_OK(scratch_free(part, st));
  return GCBF_OK;
}

template <int KI>
static int tiny_fwd_t(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, float* Y, int ldy,
                      int M, int N, int K, int act, cudaStream_t st) {
  const int blocks = (int)imax64(1, imin64(ceil_div(M, 8), 8 * kNumSMs));
  tiny_fwd_kernel<KI><<<blocks, 256, (size_t)N * KI * 32 * 4, st>>>(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

template <int KI>
static int tiny_dgrad_t(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma, const float* relu_src,
                        int ld_relu, float* dX, int lddx, int M, int N, int K, int accumulate, cudaStream_t st) {
  const int blocks = (int)imax64(1, imin64(ceil_div(M, 8), 8 * kNumSMs));
  tiny_dgrad_kernel<KI><<<blocks, 256, (size_t)N * KI * 32 * 4, st>>>(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K,
                                                                    accumulate);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

int launch_tiny_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, float* Y, int ldy,
                    int M, int N, int K, int act, cudaStream_t st) {
  const int ki = ceil_div(K, 32);
  if (ki <= 1) return tiny_fwd_t<1>(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, st);
  if (ki <= 2) return tiny_fwd_t<2>(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, st);
  if (ki <= 4) return tiny_fwd_t<4>(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, st);
  return tiny_fwd_t<8>(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, st);
}

int launch_tiny_dgrad(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma, const float* relu_src,
                      int ld_relu, float* dX, int lddx, int M, int N, int K, int accumulate, cudaStream_t st) {
  const int ki = ceil_div(K, 32);
  if (ki <= 1) return tiny_dgrad_t<1>(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, st);
  if (ki <= 2) return tiny_dgrad_t<2>(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, st);
  if (ki <= 4) return tiny_dgrad_t<4>(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, st);
  return tiny_dgrad_t<8>(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, st);
}

}  // namespace gcbf
