// Skinny linear layers: in-features K <= 16 -- the first phi layer, cat[x_i, x_j, e_ij] (12..14 wide) -> 2048
// (reference gcbf/nn/gnn.py:31, gcbf/nn/mlp.py:44-47).  These are HBM-bound streams over the [M, 2048] side
// (E x 2048 x 4 B = 198 MB at config C2) with 2*K flops per element, so they get dedicated kernels instead of a
// 128x128 GEMM tile that would be 90 % padding:
//   fwd   : Y[M,N]  = act(alpha * X[M,K] W[N,K]^T + b)       thread = 4 output columns (16-byte stores), X rows broadcast
//                                                            from smem; optional fused max|Y| for the next layer's fp16 split
//   dgrad : dX[M,K] = alpha * dZ[M,N] W[N,K]                 warp = 4 rows, lanes sweep N against W^T staged in smem,
//                                                            shuffle-reduce the K sums
//   wgrad : dW[N,K] += alpha * dZ^T X ; db[N] += colsum(dZ)  thread = column n, rows split over blockIdx.y
#include <cuda_fp16.h>

#include "common.cuh"

namespace gcbf {

constexpr int SK = 16;          // max in-features handled here
constexpr int SK_ROWS = 64;     // rows staged per block iteration

constexpr int SKF_COLS = 4;     // output columns per thread in the forward kernel (one 16-byte store per row)

__global__ void __launch_bounds__(256) skinny_fwd_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ W,
                                                         int ldw, const float* __restrict__ bias,
                                                         const float* __restrict__ alpha_p, float* __restrict__ Y, int ldy,
                                                         int M, int N, int K, int act, int rows_per_block,
                                                         uint32_t* __restrict__ amax_out, int vec_ok) {
  __shared__ __align__(16) float xs[SK_ROWS][SK];
  const int n0 = (blockIdx.x * 256 + threadIdx.x) * SKF_COLS;
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  float w[SKF_COLS][SK], b[SKF_COLS];
#pragma unroll
  for (int c = 0; c < SKF_COLS; ++c) {
#pragma unroll
    for (int k = 0; k < SK; ++k) w[c][k] = (n0 + c < N && k < K) ? __ldg(W + (size_t)(n0 + c) * ldw + k) * alpha : 0.f;
    b[c] = (n0 + c < N && bias) ? __ldg(bias + n0 + c) : 0.f;
  }
  float ymax = 0.f;
  const int m_begin = blockIdx.y * rows_per_block, m_end = min(M, m_begin + rows_per_block);
  for (int m0 = m_begin; m0 < m_end; m0 += SK_ROWS) {
    __syncthreads();
    for (int i = threadIdx.x; i < SK_ROWS * SK; i += 256) {
      const int r = i / SK, k = i % SK;
      xs[r][k] = (m0 + r < m_end && k < K) ? X[(size_t)(m0 + r) * ldx + k] : 0.f;
    }
    __syncthreads();
    if (n0 < N) {
      const int rows = min(SK_ROWS, m_end - m0);
      for (int r = 0; r < rows; ++r) {
        const float4* xr = reinterpret_cast<const float4*>(xs[r]);
        float y[SKF_COLS];
#pragma unroll
        for (int c = 0; c < SKF_COLS; ++c) y[c] = 0.f;
#pragma unroll
        for (int q = 0; q < SK / 4; ++q) {
          const float4 v = xr[q];
#pragma unroll
          for (int c = 0; c < SKF_COLS; ++c) {
            y[c] = fmaf(v.x, w[c][4 * q], y[c]); y[c] = fmaf(v.y, w[c][4 * q + 1], y[c]);
            y[c] = fmaf(v.z, w[c][4 * q + 2], y[c]); y[c] = fmaf(v.w, w[c][4 * q + 3], y[c]);
          }
        }
#pragma unroll
        for (int c = 0; c < SKF_COLS; ++c) {
          y[c] += b[c];
          if (act == GCBF_ACT_RELU) y[c] = fmaxf(y[c], 0.f);
          else if (act == GCBF_ACT_TANH) y[c] = tanhf(y[c]);
          if (n0 + c < N) ymax = fmaxf(ymax, fabsf(y[c]));
        }
        float* dst = Y + (size_t)(m0 + r) * ldy + n0;
        if (vec_ok && n0 + SKF_COLS <= N) {
          *reinterpret_cast<float4*>(dst) = make_float4(y[0], y[1], y[2], y[3]);
        } else {
#pragma unroll
          for (int c = 0; c < SKF_COLS; ++c)
            if (n0 + c < N) dst[c] = y[c];
        }
      }
    }
  }
  if (amax_out) {   // max|Y| for the fp16 split of the next (tensor-core) layer; non-negative floats order like uints
    const uint32_t m = __reduce_max_sync(0xffffffffu, __float_as_uint(ymax));
    if ((threadIdx.x & 31) == 0 && m) atomicMax(amax_out, m);
  }
}

// The same layer writing its output directly as a tile-scaled fp16 [hi|lo] companion (the format the tensor-core epilogues emit,
// gemm_wgmma_f16.cu): a block owns one 128-row x 256-column tile; with K <= 16 an output costs 2*K flops, so the tile is computed
// TWICE -- once for its exact max|y| (the tile's scale), once to convert and store -- instead of writing fp32, re-reading it for an
// amax pass and again for a split pass (12 B/element of HBM traffic become 4).
__device__ __forceinline__ uint32_t skinny_scale_bits(uint32_t amax_bits) {     // == th::scale_bits_from_amax
  const int e = (int)((amax_bits >> 23) & 0xffu);
  if (e == 0 || e == 255) return 0x3f800000u;
  int se = 127 + 14 - (e - 127);
  se = se < 2 ? 2 : (se > 252 ? 252 : se);
  return (uint32_t)se << 23;
}

__global__ void __launch_bounds__(512, 1) skinny_fwd_emit_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ W, int ldw,
                                                                 const float* __restrict__ bias, const float* __restrict__ alpha_p,
                                                                 __half* __restrict__ Yh, int ld_h, uint32_t* __restrict__ tile_amax,
                                                                 int amax_stride, int M, int N, int K, int act) {
  // A block (512 threads = 16 warps, one per SM) owns one 256-column tile and walks down the 128-row tiles: its 2 x 16 weights per
  // thread are loaded ONCE, the next row tile's inputs are prefetched into registers while the current one is computed.  thread = 2
  // adjacent columns x 32 rows; the 64 results stay in registers between the tile maximum and the conversion.  (v1 recomputed the
  // tile for the conversion pass and re-loaded the weights per tile: 1.08 ms per 206 k-row launch; v2 kept 4 x 32 results per thread in
  // 231 registers -> 8 warps per SM: 0.87 ms.)
  __shared__ __align__(16) float xs[128][SK];
  __shared__ uint32_t wmax[2][16];
  const int cg = threadIdx.x & 127, rg = threadIdx.x >> 7;            // 128 column pairs x 4 row groups of 32
  const int n0 = blockIdx.x * 256 + cg * 2;
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  float w[2][SK], b[2];
#pragma unroll
  for (int c = 0; c < 2; ++c) {
#pragma unroll
    for (int k = 0; k < SK; ++k) w[c][k] = (n0 + c < N && k < K) ? __ldg(W + (size_t)(n0 + c) * ldw + k) * alpha : 0.f;
    b[c] = (n0 + c < N && bias) ? __ldg(bias + n0 + c) : 0.f;
  }
  const int row_tiles = (M + 127) / 128;
  const size_t plane = (size_t)M * ld_h;
  const bool vec = (n0 + 2 <= N);
  float pre[4];                                                       // 128 x 16 staged inputs / 512 threads
  auto prefetch = [&](int rt) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int i = threadIdx.x + 512 * j, r = i / SK, k = i % SK;
      const int row = rt * 128 + r;
      pre[j] = (rt < row_tiles && row < M && k < K) ? __ldg(X + (size_t)row * ldx + k) : 0.f;
    }
  };
  prefetch(blockIdx.y);
  int par = 0;
  for (int rt = blockIdx.y; rt < row_tiles; rt += gridDim.y, par ^= 1) {
    const int m0 = rt * 128;
    __syncthreads();                                                  // the previous tile's reads of xs are done
#pragma unroll
    for (int j = 0; j < 4; ++j) { const int i = threadIdx.x + 512 * j; xs[i / SK][i % SK] = pre[j]; }
    __syncthreads();
    prefetch(rt + gridDim.y);                                         // in flight during the compute below
    const int rows = min(128, M - m0);
    float y[32][2];
    float ymax = 0.f;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const float4* xr = reinterpret_cast<const float4*>(xs[rg * 32 + i]);
      float t0 = 0.f, t1 = 0.f;
#pragma unroll
      for (int q = 0; q < SK / 4; ++q) {
        const float4 v = xr[q];
        t0 = fmaf(v.x, w[0][4 * q], t0); t0 = fmaf(v.y, w[0][4 * q + 1], t0); t0 = fmaf(v.z, w[0][4 * q + 2], t0); t0 = fmaf(v.w, w[0][4 * q + 3], t0);
        t1 = fmaf(v.x, w[1][4 * q], t1); t1 = fmaf(v.y, w[1][4 * q + 1], t1); t1 = fmaf(v.z, w[1][4 * q + 2], t1); t1 = fmaf(v.w, w[1][4 * q + 3], t1);
      }
      t0 += b[0]; t1 += b[1];
      if (act == GCBF_ACT_RELU) { t0 = fmaxf(t0, 0.f); t1 = fmaxf(t1, 0.f); }
      else if (act == GCBF_ACT_TANH) { t0 = tanhf(t0); t1 = tanhf(t1); }
      const bool row_in = rg * 32 + i < rows;
      if (!row_in || n0 >= N) t0 = 0.f;
      if (!row_in || n0 + 1 >= N) t1 = 0.f;
      y[i][0] = t0; y[i][1] = t1;
      ymax = fmaxf(ymax, fmaxf(fabsf(t0), fabsf(t1)));
    }
    {
      const uint32_t m = __reduce_max_sync(0xffffffffu, __float_as_uint(ymax));   // non-negative floats order like uints
      if ((threadIdx.x & 31) == 0) wmax[par][threadIdx.x >> 5] = m;
    }
    __syncthreads();
    uint32_t tm = 0;
#pragma unroll
    for (int i = 0; i < 16; ++i) tm = max(tm, wmax[par][i]);
    const float s = __uint_as_float(skinny_scale_bits(tm));
    if (threadIdx.x == 0) tile_amax[(size_t)rt * amax_stride + blockIdx.x] = tm;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int r = rg * 32 + i;
      if (r < rows) {
        const float y0 = y[i][0] * s, y1 = y[i][1] * s;
        const __half2 h = __floats2half2_rn(y0, y1);
        const float2 hf = __half22float2(h);
        const __half2 l = __floats2half2_rn(__fsub_rn(y0, hf.x), __fsub_rn(y1, hf.y));
        __half* d = Yh + (size_t)(m0 + r) * ld_h + n0;
        if (vec) {
          *reinterpret_cast<__half2*>(d) = h;
          *reinterpret_cast<__half2*>(d + plane) = l;
        } else if (n0 < N) {
          d[0] = __low2half(h);
          d[plane] = __low2half(l);
        }
      }
    }
  }
}

constexpr int SKD_NCHUNK = 512;   // columns of W staged per pass: [SK][512] floats = 32 KB of shared memory

__global__ void __launch_bounds__(256) skinny_dgrad_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ W,
                                                           int ldw, const float* __restrict__ alpha_p,
                                                           const float* __restrict__ relu_src, int ld_relu,
                                                           float* __restrict__ dX, int lddx, int M, int N, int K, int accumulate,
                                                           int rows_per_block, int vec_ok) {
  __shared__ __align__(16) float wt[SK][SKD_NCHUNK + 4];   // W^T chunk: wt[k][n] -> lanes read consecutive n (16-byte reads, conflict free)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int m_begin = blockIdx.x * rows_per_block, m_end = min(M, m_begin + rows_per_block);
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  constexpr int RPW = 4;                   // rows per warp per pass (independent accumulators -> loads in flight)
  for (int mb = m_begin; mb < m_end; mb += 8 * RPW) {
    float acc[RPW][SK];
#pragma unroll
    for (int r = 0; r < RPW; ++r)
#pragma unroll
      for (int k = 0; k < SK; ++k) acc[r][k] = 0.f;
    for (int nc = 0; nc < N; nc += SKD_NCHUNK) {
      __syncthreads();
      for (int i = threadIdx.x; i < SK * SKD_NCHUNK; i += 256) {
        const int n = i / SK, k = i % SK;       // consecutive threads read consecutive k of one weight row
        wt[k][n] = (nc + n < N && k < K) ? __ldg(W + (size_t)(nc + n) * ldw + k) : 0.f;
      }
      __syncthreads();
      const int nlim = min(SKD_NCHUNK, N - nc);
      if (vec_ok && (nlim & 3) == 0) {
        for (int n = lane * 4; n < nlim; n += 128) {       // 16-byte loads: 512 B of a dZ row per warp instruction
          float4 z[RPW];
#pragma unroll
          for (int r = 0; r < RPW; ++r) {
            const int m = mb + warp * RPW + r;
            z[r] = (m < m_end) ? __ldg(reinterpret_cast<const float4*>(dZ + (size_t)m * lddz + nc + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
          }
#pragma unroll
          for (int k = 0; k < SK; ++k) {
            const float4 w4 = *reinterpret_cast<const float4*>(&wt[k][n]);
            const float w0 = w4.x, w1 = w4.y, w2 = w4.z, w3 = w4.w;
#pragma unroll
            for (int r = 0; r < RPW; ++r)
              acc[r][k] = fmaf(z[r].w, w3, fmaf(z[r].z, w2, fmaf(z[r].y, w1, fmaf(z[r].x, w0, acc[r][k]))));
          }
        }
      } else {
        for (int n = lane; n < nlim; n += 32) {
          float z[RPW];
#pragma unroll
          for (int r = 0; r < RPW; ++r) {
            const int m = mb + warp * RPW + r;
            z[r] = (m < m_end) ? __ldg(dZ + (size_t)m * lddz + nc + n) : 0.f;
          }
#pragma unroll
          for (int k = 0; k < SK; ++k) {
            const float wv = wt[k][n];
#pragma unroll
            for (int r = 0; r < RPW; ++r) acc[r][k] = fmaf(z[r], wv, acc[r][k]);
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < RPW; ++r) {
      const int m = mb + warp * RPW + r;
#pragma unroll
      for (int k = 0; k < SK; ++k) {
        const float s = warp_sum(acc[r][k]);
        if (lane == k && k < K && m < m_end) {
          float v = alpha * s;
          if (relu_src && !(relu_src[(size_t)m * ld_relu + k] > 0.f)) v = 0.f;
          float* dst = dX + (size_t)m * lddx + k;
          *dst = accumulate ? *dst + v : v;
        }
      }
    }
  }
}

// data-grad with the WHOLE W^T resident in shared memory (N <= 3072: 16 x (N + 4) floats <= 197 KB): persistent blocks stage it once
// and stream their rows -- the chunked kernel above re-stages 128 KB of W per 32 rows, half as much again as the dZ bytes it reads
constexpr int SKD_RPW = 8;
__global__ void __launch_bounds__(256, 1) skinny_dgrad_full_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ W, int ldw,
                                                                   const float* __restrict__ alpha_p, const float* __restrict__ relu_src,
                                                                   int ld_relu, float* __restrict__ dX, int lddx, int M, int N, int K,
                                                                   int accumulate) {
  extern __shared__ __align__(16) float wt_full[];                 // [SK][N + 4]
  const int pitch = N + 4;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < SK * N; i += 256) {
    const int n = i / SK, k = i % SK;
    wt_full[k * pitch + n] = (k < K) ? __ldg(W + (size_t)n * ldw + k) : 0.f;
  }
  __syncthreads();
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  for (int mb = blockIdx.x * (8 * SKD_RPW); mb < M; mb += gridDim.x * (8 * SKD_RPW)) {
    const int m0 = mb + warp * SKD_RPW;
    float acc[SKD_RPW][SK];
#pragma unroll
    for (int r = 0; r < SKD_RPW; ++r)
#pragma unroll
      for (int k = 0; k < SK; ++k) acc[r][k] = 0.f;
    for (int n = lane * 4; n < N; n += 128) {
      float4 z[SKD_RPW];
#pragma unroll
      for (int r = 0; r < SKD_RPW; ++r)
        z[r] = (m0 + r < M) ? __ldg(reinterpret_cast<const float4*>(dZ + (size_t)(m0 + r) * lddz + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int k = 0; k < SK; ++k) {
        const float4 w4 = *reinterpret_cast<const float4*>(&wt_full[k * pitch + n]);
#pragma unroll
        for (int r = 0; r < SKD_RPW; ++r)
          acc[r][k] = fmaf(z[r].w, w4.w, fmaf(z[r].z, w4.z, fmaf(z[r].y, w4.y, fmaf(z[r].x, w4.x, acc[r][k]))));
      }
    }
#pragma unroll
    for (int r = 0; r < SKD_RPW; ++r) {
      const int m = m0 + r;
#pragma unroll
      for (int k = 0; k < SK; ++k) {
        const float sum = warp_sum(acc[r][k]);
        if (lane == k && k < K && m < M) {
          float v = alpha * sum;
          if (relu_src && !(relu_src[(size_t)m * ld_relu + k] > 0.f)) v = 0.f;
          float* dst = dX + (size_t)m * lddx + k;
          *dst = accumulate ? *dst + v : v;
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) skinny_wgrad_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ X,
                                                           int ldx, const float* __restrict__ alpha_p, float* __restrict__ dW,
                                                           int lddw, float* __restrict__ db, int M, int N, int K,
                                                           int rows_per_block) {
  __shared__ __align__(16) float xs[SK_ROWS][SK];
  const int n = blockIdx.x * 256 + threadIdx.x;
  float acc[SK];
#pragma unroll
  for (int k = 0; k < SK; ++k) acc[k] = 0.f;
  float accb = 0.f;
  const int m_begin = blockIdx.y * rows_per_block, m_end = min(M, m_begin + rows_per_block);
  for (int m0 = m_begin; m0 < m_end; m0 += SK_ROWS) {
    __syncthreads();
    for (int i = threadIdx.x; i < SK_ROWS * SK; i += 256) {
      const int r = i / SK, k = i % SK;
      xs[r][k] = (m0 + r < m_end && k < K) ? X[(size_t)(m0 + r) * ldx + k] : 0.f;
    }
    __syncthreads();
    if (n < N) {
      const int rows = min(SK_ROWS, m_end - m0);     // rows beyond `rows` are zero in xs, so reading dZ row 0 for them is harmless
      for (int r = 0; r < rows; r += 8) {
        float z[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) z[u] = (r + u < rows) ? __ldg(dZ + (size_t)(m0 + r + u) * lddz + n) : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const float4* xr = reinterpret_cast<const float4*>(xs[r + u]);
          accb += z[u];
#pragma unroll
          for (int q = 0; q < SK / 4; ++q) {
            const float4 v = xr[q];
            acc[4 * q] = fmaf(z[u], v.x, acc[4 * q]); acc[4 * q + 1] = fmaf(z[u], v.y, acc[4 * q + 1]);
            acc[4 * q + 2] = fmaf(z[u], v.z, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(z[u], v.w, acc[4 * q + 3]);
          }
        }
      }
    }
  }
  if (n < N) {
    const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
    // this row block's partials (dW_part [row block][N][K], db_part [row block][N]); summed in order by add_partials
#pragma unroll
    for (int k = 0; k < SK; ++k)
      if (k < K) dW[((size_t)blockIdx.y * N + n) * K + k] = alpha * acc[k];
    if (db) db[(size_t)blockIdx.y * N + n] = accb;
  }
}

bool skinny_supported(int K) { return K <= SK; }

int launch_skinny_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, float* Y,
                      int ldy, int M, int N, int K, int act, uint32_t* amax_out, cudaStream_t st) {
  const int col_blocks = ceil_div(N, 256 * SKF_COLS);
  int row_blocks = max(1, min(ceil_div(M, SK_ROWS), (12 * kNumSMs) / col_blocks));   // ~6 resident blocks per SM hide the X-tile loads
  const int rpb = ceil_div(ceil_div(M, row_blocks), SK_ROWS) * SK_ROWS;
  row_blocks = ceil_div(M, rpb);
  const int vec_ok = ((ldy & 3) == 0 && (reinterpret_cast<uintptr_t>(Y) & 15) == 0) ? 1 : 0;
  skinny_fwd_kernel<<<dim3(col_blocks, row_blocks), 256, 0, st>>>(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, rpb,
                                                                  amax_out, vec_ok);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

int launch_skinny_fwd_emit(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, __half* Yh, int ld_h,
                           uint32_t* tile_amax, int amax_stride, int M, int N, int K, int act, cudaStream_t st) {
  const int col_tiles = ceil_div(N, 256), row_tiles = ceil_div(M, 128);
  const int gy = max(1, min(row_tiles, kNumSMs / col_tiles));          // persistent: about one 512-thread block per SM
  skinny_fwd_emit_kernel<<<dim3(col_tiles, gy), 512, 0, st>>>(X, ldx, W, ldw, bias, inv_sigma, Yh, ld_h, tile_amax, amax_stride, M, N, K, act);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

int launch_skinny_dgrad(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma, const float* relu_src,
                        int ld_relu, float* dX, int lddx, int M, int N, int K, int accumulate, cudaStream_t st) {
  const int vec_ok = ((lddz & 3) == 0 && (reinterpret_cast<uintptr_t>(dZ) & 15) == 0) ? 1 : 0;
  if (vec_ok && (N & 3) == 0 && N <= 3072 && M >= 4096) {
    const size_t smem = (size_t)SK * (N + 4) * sizeof(float);
    static bool attr_set = false;
    if (!attr_set) {
      GCBF_CUDA_OK(cudaFuncSetAttribute(skinny_dgrad_full_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SK * (3072 + 4) * (int)sizeof(float)));
      attr_set = true;
    }
    skinny_dgrad_full_kernel<<<kNumSMs, 256, smem, st>>>(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate);
    GCBF_LAUNCH_OK();
    return GCBF_OK;
  }
  const int rpb = 32;                       // 8 warps x 4 rows: W^T is staged once per block
  const int blocks = ceil_div(M, rpb);
  skinny_dgrad_kernel<<<blocks, 256, 0, st>>>(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K, accumulate, rpb, vec_ok);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

int launch_skinny_wgrad(const float* dZ, int lddz, const float* X, int ldx, const float* inv_sigma, float* dW, int lddw,
                        float* db, int M, int N, int K, int accumulate, cudaStream_t st) {
  const int col_blocks = ceil_div(N, 256);
  int row_blocks = max(1, min(ceil_div(M, 4 * SK_ROWS), (4 * kNumSMs) / col_blocks));
  const int rpb = ceil_div(ceil_div(M, row_blocks), SK_ROWS) * SK_ROWS;
  row_blocks = ceil_div(M, rpb);
  float* part = nullptr;
  GCBF_CUDA_OK(scratch_alloc((void**)&part, (size_t)row_blocks * N * (K + 1) * 4, st));
  float* db_part = part + (size_t)row_blocks * N * K;
  skinny_wgrad_kernel<<<dim3(col_blocks, row_blocks), 256, 0, st>>>(dZ, lddz, X, ldx, inv_sigma, part, lddw, db ? db_part : nullptr, M, N, K, rpb);
  GCBF_LAUNCH_OK();
  GCBF_CUDA_OK(add_partials(part, row_blocks, N, K, dW, lddw, accumulate, st));
  if (db) GCBF_CUDA_OK(add_partials(db_part, row_blocks, 1, N, db, N, accumulate, st));
  GCBF_CUDA_OK(scratch_free(part, st));
  return GCBF_OK;
}

}  // namespace gcbf
