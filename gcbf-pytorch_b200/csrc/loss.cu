// K6 losses of GCBF.update (reference gcbf/algo/gcbf.py:164-218) in two passes so that data-parallel
// ranks can all-reduce the 9 partial sums in between and reproduce the single-process masked MEANS:
//   pass 1 (loss_partials): per-rank sums / counts in double
//   pass 2 (loss_grads)   : d loss/d h, d loss/d h_next, d loss/d actions with the (global) denominators,
//                           plus the scalar losses and accuracies.
// and the M x M "acc/derivative" statistic of gcbf.py:209 as an exact tiled pair count.
#include "common.cuh"

namespace gcbf {

// value of h_dot as the reference forms it (gcbf.py:202-205): residue = (hdn - hd).detach(); hd = residue + hd
__device__ __forceinline__ float hdot_value(float h, float hn, float hnn, float dt) {
  const float hd = __fsub_rn(hn, h) / dt;
  const float hdn = __fsub_rn(hnn, h) / dt;
  return __fadd_rn(__fsub_rn(hdn, hd), hd);
}

__global__ void loss_partials_kernel(const float* __restrict__ h, const float* __restrict__ hn,
                                     const float* __restrict__ hnn, const float* __restrict__ act, int ad,
                                     const uint8_t* __restrict__ safe, const uint8_t* __restrict__ unsafe, int64_t M,
                                     float alpha, float eps, float dt, double* __restrict__ partial,
                                     float* __restrict__ hdot_out, const float* __restrict__ hdot_in) {
  double acc[9] = {0, 0, 0, 0, 0, 0, 0, 0, 0};
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < M; i += (int64_t)gridDim.x * blockDim.x) {
    const float hi = h[i];
    if (unsafe[i]) {                                    // gcbf.py:168-177
      acc[GCBF_LP_SUM_UNSAFE] += fmaxf(__fadd_rn(hi, eps), 0.f);
      acc[GCBF_LP_CNT_UNSAFE] += 1.0;
      acc[GCBF_LP_OK_UNSAFE] += (hi < 0.f) ? 1.0 : 0.0;
    }
    if (safe[i]) {                                      // gcbf.py:180-189
      acc[GCBF_LP_SUM_SAFE] += fmaxf(__fadd_rn(-hi, eps), 0.f);
      acc[GCBF_LP_CNT_SAFE] += 1.0;
      acc[GCBF_LP_OK_SAFE] += (hi >= 0.f) ? 1.0 : 0.0;
    }
    // gcbf.py:207; hdot_in: the analytic h_dot (GCBF.params['h_dot'] = 'analytic') instead of the finite difference
    const float hd = hdot_in ? hdot_in[i] : hdot_value(hi, hn[i], hnn[i], dt);
    if (hdot_out) hdot_out[i] = hd;
    acc[GCBF_LP_SUM_HDOT] += fmaxf(__fadd_rn(__fsub_rn(-hd, __fmul_rn(alpha, hi)), eps), 0.f);
    acc[GCBF_LP_CNT_ALL] += 1.0;
    float s = 0.f;
    for (int k = 0; k < ad; ++k) { const float u = act[i * ad + k]; s = __fadd_rn(s, __fmul_rn(u, u)); }
    acc[GCBF_LP_SUM_ACT] += s;                          // gcbf.py:212
  }
  __shared__ double sm[9][8];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const double v = warp_sum(acc[k]);
    if (lane == 0) sm[k][wid] = v;
  }
  __syncthreads();
  if (threadIdx.x < 9) {
    double t = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += sm[threadIdx.x][w];
    atomicAdd(partial + threadIdx.x, t);
  }
}

__global__ void loss_grads_kernel(const float* __restrict__ h, const float* __restrict__ hn,
                                  const float* __restrict__ hnn, const float* __restrict__ act, int ad,
                                  const uint8_t* __restrict__ safe, const uint8_t* __restrict__ unsafe, int64_t M,
                                  float alpha, float eps, float dt, float cu, float cs, float ch, float ca,
                                  const double* __restrict__ partial, float* __restrict__ d_h,
                                  float* __restrict__ d_hn, float* __restrict__ d_act, float* __restrict__ scalars,
                                  const float* __restrict__ hdot_in, float* __restrict__ d_hdot) {
  const double cnt_u = partial[GCBF_LP_CNT_UNSAFE], cnt_s = partial[GCBF_LP_CNT_SAFE], cnt = partial[GCBF_LP_CNT_ALL];
  const float inv_u = cnt_u > 0 ? (float)(1.0 / cnt_u) : 0.f;
  const float inv_s = cnt_s > 0 ? (float)(1.0 / cnt_s) : 0.f;
  const float inv_m = cnt > 0 ? (float)(1.0 / cnt) : 0.f;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    const float lu = cnt_u > 0 ? (float)(partial[GCBF_LP_SUM_UNSAFE] / cnt_u) : 0.f;   // empty mask: loss 0, acc 1
    const float ls = cnt_s > 0 ? (float)(partial[GCBF_LP_SUM_SAFE] / cnt_s) : 0.f;
    const float lh = cnt > 0 ? (float)(partial[GCBF_LP_SUM_HDOT] / cnt) : 0.f;
    const float la = cnt > 0 ? (float)(partial[GCBF_LP_SUM_ACT] / cnt) : 0.f;
    scalars[0] = lu; scalars[1] = ls; scalars[2] = lh; scalars[3] = la;
    scalars[4] = cnt_u > 0 ? (float)(partial[GCBF_LP_OK_UNSAFE] / cnt_u) : 1.f;
    scalars[5] = cnt_s > 0 ? (float)(partial[GCBF_LP_OK_SAFE] / cnt_s) : 1.f;
    scalars[6] = cu * lu + cs * ls + ch * lh + ca * la;                                 // gcbf.py:215-218
    scalars[7] = (float)cnt;
  }
  if (i >= M) return;
  const float hi = h[i];
  float g = 0.f;
  if (unsafe[i] && __fadd_rn(hi, eps) > 0.f) g += cu * inv_u;
  if (safe[i] && __fadd_rn(-hi, eps) > 0.f) g -= cs * inv_s;
  const float hd = hdot_in ? hdot_in[i] : hdot_value(hi, hn[i], hnn[i], dt);
  const bool on = __fadd_rn(__fsub_rn(-hd, __fmul_rn(alpha, hi)), eps) > 0.f;
  float gn = 0.f;
  if (hdot_in) {
    // analytic h_dot: d/dh of relu(-h_dot - alpha*h + eps) = -alpha ; d/dh_dot = -1
    const float w = on ? ch * inv_m : 0.f;
    g -= w * alpha;
    d_hdot[i] = -w;
  } else if (on) {
    const float w = ch * inv_m;
    // d/dh of relu(-(h_next - h)/dt - alpha*h + eps) = +1/dt - alpha ; d/dh_next = -1/dt   (the re-linked
    // h_next_new enters only through the detached residue)
    g += w / dt - w * alpha;
    gn = -(w / dt);
  }
  d_h[i] = g;
  if (d_hn) d_hn[i] = gn;
  for (int k = 0; k < ad; ++k) d_act[i * ad + k] = ca * inv_m * 2.f * act[i * ad + k];
}

// count of (row i, col j) with hdot[j] + alpha*h[i] >= 0.  One thread per row, columns staged in smem.
__global__ void __launch_bounds__(256) pair_count_kernel(const float* __restrict__ hdot, int64_t mc,
                                                         const float* __restrict__ h, int64_t mr, float alpha,
                                                         unsigned long long* __restrict__ count) {
  __shared__ float tile[1024];
  __shared__ unsigned long long wsum[8];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const float ah = (i < mr) ? __fmul_rn(alpha, h[i]) : 0.f;
  unsigned long long c = 0;
  for (int64_t j0 = (int64_t)blockIdx.y * 1024; j0 < mc; j0 += (int64_t)gridDim.y * 1024) {
    __syncthreads();
    for (int t = threadIdx.x; t < 1024; t += blockDim.x) tile[t] = (j0 + t < mc) ? hdot[j0 + t] : -INFINITY;
    __syncthreads();
    if (i < mr) {
      unsigned int cc = 0;
#pragma unroll 8
      for (int t = 0; t < 1024; ++t) cc += (__fadd_rn(tile[t], ah) >= 0.f) ? 1u : 0u;
      c += cc;
    }
  }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int w = 0; w < 8; ++w) t += wsum[w];
    atomicAdd(count, t);
  }
}

}  // namespace gcbf

using namespace gcbf;

extern "C" int gcbf_loss_partials(const float* h, const float* h_next, const float* h_next_new, const float* action,
                                  int action_dim, const uint8_t* safe, const uint8_t* unsafe, int64_t M, float alpha,
                                  float eps, float dt, double* partial, float* hdot_out, void* stream) {
  GCBF_REQUIRE(partial && M >= 0 && action_dim >= 0, "gcbf_loss_partials: bad arguments");
  cudaStream_t st = as_stream(stream);
  GCBF_CUDA_OK(cudaMemsetAsync(partial, 0, GCBF_LP_SIZE * sizeof(double), st));
  if (M == 0) return GCBF_OK;
  GCBF_REQUIRE(h && h_next && h_next_new && action && safe && unsafe, "gcbf_loss_partials: null pointer");
  const int grid = (int)imin64(ceil_div(M, 256), 4 * kNumSMs);
  loss_partials_kernel<<<grid, 256, 0, st>>>(h, h_next, h_next_new, action, action_dim, safe, unsafe, M, alpha, eps, dt,
                                            partial, hdot_out, nullptr);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_loss_grads(const float* h, const float* h_next, const float* h_next_new, const float* action,
                               int action_dim, const uint8_t* safe, const uint8_t* unsafe, int64_t M, float alpha,
                               float eps, float dt, float coef_unsafe, float coef_safe, float coef_hdot,
                               float coef_action, const double* partial, float* d_h, float* d_h_next, float* d_action,
                               float* scalars, void* stream) {
  GCBF_REQUIRE(partial && scalars && M >= 0, "gcbf_loss_grads: bad arguments");
  GCBF_REQUIRE(M == 0 || (h && h_next && h_next_new && action && safe && unsafe && d_h && d_h_next && d_action),
               "gcbf_loss_grads: null pointer");
  loss_grads_kernel<<<max(1, ceil_div(M, 256)), 256, 0, as_stream(stream)>>>(
      h, h_next, h_next_new, action, action_dim, safe, unsafe, M, alpha, eps, dt, coef_unsafe, coef_safe, coef_hdot,
      coef_action, partial, d_h, d_h_next, d_action, scalars, nullptr, nullptr);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

// the same two passes with the analytic h_dot as an input (GCBF.params['h_dot'] = 'analytic'): same partial layout, scalars and masked
// means; d_hdot replaces d_h_next
extern "C" int gcbf_loss_partials_hdot(const float* h, const float* hdot, const float* action, int action_dim, const uint8_t* safe,
                                       const uint8_t* unsafe, int64_t M, float alpha, float eps, double* partial, void* stream) {
  GCBF_REQUIRE(partial && M >= 0 && action_dim >= 0, "gcbf_loss_partials_hdot: bad arguments");
  if (M > 0) GCBF_REQUIRE(h && hdot && action && safe && unsafe, "gcbf_loss_partials_hdot: null pointer");
  cudaStream_t st = as_stream(stream);
  GCBF_CUDA_OK(cudaMemsetAsync(partial, 0, GCBF_LP_SIZE * sizeof(double), st));
  if (M == 0) return GCBF_OK;
  const int grid = (int)imin64(ceil_div(M, 256), 4 * kNumSMs);
  loss_partials_kernel<<<grid, 256, 0, st>>>(h, nullptr, nullptr, action, action_dim, safe, unsafe, M, alpha, eps, 1.f, partial, nullptr, hdot);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_loss_grads_hdot(const float* h, const float* hdot, const float* action, int action_dim, const uint8_t* safe,
                                    const uint8_t* unsafe, int64_t M, float alpha, float eps, float coef_unsafe, float coef_safe,
                                    float coef_hdot, float coef_action, const double* partial, float* d_h, float* d_hdot, float* d_action,
                                    float* scalars, void* stream) {
  GCBF_REQUIRE(partial && scalars && M >= 0 && action_dim >= 0, "gcbf_loss_grads_hdot: bad arguments");
  GCBF_REQUIRE(M == 0 || (h && hdot && action && safe && unsafe && d_h && d_hdot && d_action), "gcbf_loss_grads_hdot: null pointer");
  loss_grads_kernel<<<max(1, ceil_div(M, 256)), 256, 0, as_stream(stream)>>>(
      h, nullptr, nullptr, action, action_dim, safe, unsafe, M, alpha, eps, 1.f, coef_unsafe, coef_safe, coef_hdot, coef_action, partial,
      d_h, nullptr, d_action, scalars, hdot, d_hdot);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_pair_count(const float* hdot, int64_t m_cols, const float* h, int64_t m_rows, float alpha,
                               unsigned long long* count, void* stream) {
  GCBF_REQUIRE(count && m_cols >= 0 && m_rows >= 0, "gcbf_pair_count: bad arguments");
  cudaStream_t st = as_stream(stream);
  GCBF_CUDA_OK(cudaMemsetAsync(count, 0, sizeof(unsigned long long), st));
  if (m_cols == 0 || m_rows == 0) return GCBF_OK;
  GCBF_REQUIRE(hdot && h, "gcbf_pair_count: null pointer");
  const int gx = ceil_div(m_rows, 256);
  int gy = max(1, min(ceil_div(m_cols, 1024), (4 * kNumSMs) / gx));
  dim3 grid(gx, gy);
  pair_count_kernel<<<grid, 256, 0, st>>>(hdot, m_cols, h, m_rows, alpha, count);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}
