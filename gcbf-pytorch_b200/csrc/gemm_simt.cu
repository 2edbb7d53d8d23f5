// fp32 SIMT GEMM with fused epilogues -- the exact-fp32 implementation of the linear layers of gcbf.nn.MLP
// (reference gcbf/nn/mlp.py:44-47).  Used for every shape the wgmma path does not take (odd K such as
// the 12..14-wide first phi layer, the tiny gate / head layers) and as the numerical cross-check of the
// tensor-core kernel.  One kernel, three operand layouts:
//
//     C(m, n) = sum_k A(m, k) * B(n, k)
//
//   forward    A = X  [M,K] (k contiguous)   B = W  [N,K] (k contiguous)      C = Y  [M,N]
//   data grad  A = dZ [M,N] (k contiguous)   B = W  [N,K] (n-out contiguous)  C = dX [M,K]
//   weight grad A = dZ [M,N] (m-out contig.) B = X  [M,K] (n-out contiguous)  C = dW [N,K]   (split-K)
//
// Tile 128x128x16, 256 threads, 8x8 register micro-tile, register-prefetch double buffering.
#include "common.cuh"

namespace gcbf {

constexpr int BM = 128, BN = 128, BK = 16, NT = 256;
constexpr int LDS = BM + 4;  // smem row pitch (floats): keeps float4 alignment, breaks the worst conflicts

enum EpiMode { EPI_FWD = 0, EPI_DGRAD = 1, EPI_WGRAD = 2 };

struct Epi {
  int mode;
  const float* alpha;     // device scalar or nullptr (== 1)
  const float* bias;      // [N] or nullptr            (FWD)
  int act;                // GCBF_ACT_*                (FWD)
  const float* relu_src;  // [M, ld_relu] or nullptr   (DGRAD)
  int ld_relu;
  int accumulate;         // WGRAD / DGRAD: add into C
  size_t split_stride;    // WGRAD split-K: contraction split z writes the slice C + z * split_stride
};

// Load one BK x 128 operand tile into registers (8 floats per thread).
// KC = true : global is [row][k] (k contiguous)  -> thread owns 2 x float4 along k for rows r, r+64
// KC = false: global is [k][row] (row contiguous)-> thread owns 2 x float4 along rows for k, k+8
template <bool KC>
__device__ __forceinline__ void load_tile(const float* __restrict__ P, int ld, int row0, int nrows, int k0,
                                          int kend, bool vec_ok, float (&r)[8]) {
  const int t = threadIdx.x;
  if (KC) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = row0 + (t >> 2) + 64 * i;
      const int k = k0 + (t & 3) * 4;
      const float* src = P + (size_t)row * ld + k;
      if (row < nrows && vec_ok && k + 3 < kend) {
        const float4 v = *reinterpret_cast<const float4*>(src);
        r[4 * i + 0] = v.x; r[4 * i + 1] = v.y; r[4 * i + 2] = v.z; r[4 * i + 3] = v.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) r[4 * i + j] = (row < nrows && k + j < kend) ? src[j] : 0.f;
      }
    }
  } else {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int k = k0 + (t >> 5) + 8 * i;
      const int row = row0 + (t & 31) * 4;
      const float* src = P + (size_t)k * ld + row;
      if (k < kend && vec_ok && row + 3 < nrows) {
        const float4 v = *reinterpret_cast<const float4*>(src);
        r[4 * i + 0] = v.x; r[4 * i + 1] = v.y; r[4 * i + 2] = v.z; r[4 * i + 3] = v.w;
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j) r[4 * i + j] = (k < kend && row + j < nrows) ? src[j] : 0.f;
      }
    }
  }
}

template <bool KC>
__device__ __forceinline__ void store_tile(float* __restrict__ S, const float (&r)[8]) {
  const int t = threadIdx.x;
  if (KC) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int row = (t >> 2) + 64 * i;
      const int k = (t & 3) * 4;
#pragma unroll
      for (int j = 0; j < 4; ++j) S[(k + j) * LDS + row] = r[4 * i + j];
    }
  } else {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int k = (t >> 5) + 8 * i;
      const int row = (t & 31) * 4;
      *reinterpret_cast<float4*>(&S[k * LDS + row]) = make_float4(r[4 * i], r[4 * i + 1], r[4 * i + 2], r[4 * i + 3]);
    }
  }
}

template <bool A_KC, bool B_KC>
__global__ void __launch_bounds__(NT) gemm_simt_kernel(const float* __restrict__ A, int lda,
                                                       const float* __restrict__ B, int ldb,
                                                       float* __restrict__ C, int ldc, int M, int N, int K,
                                                       int k_chunk, Epi ep) {
  __shared__ __align__(16) float As[BK * LDS];
  __shared__ __align__(16) float Bs[BK * LDS];
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * k_chunk;
  const int kend = min(K, kbeg + k_chunk);
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const bool a_vec = ((lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(A) & 15) == 0);
  const bool b_vec = ((ldb & 3) == 0) && ((reinterpret_cast<uintptr_t>(B) & 15) == 0);

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float ra[8], rb[8];
  if (kbeg < kend) {
    load_tile<A_KC>(A, lda, m0, M, kbeg, kend, a_vec, ra);
    load_tile<B_KC>(B, ldb, n0, N, kbeg, kend, b_vec, rb);
  }
  for (int k0 = kbeg; k0 < kend; k0 += BK) {
    __syncthreads();  // previous tile fully consumed
    store_tile<A_KC>(As, ra);
    store_tile<B_KC>(Bs, rb);
    __syncthreads();
    if (k0 + BK < kend) {
      load_tile<A_KC>(A, lda, m0, M, k0 + BK, kend, a_vec, ra);
      load_tile<B_KC>(B, ldb, n0, N, k0 + BK, kend, b_vec, rb);
    }
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[k * LDS + ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[k * LDS + 64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[k * LDS + tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[k * LDS + 64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
  }

  // ---- epilogue -----------------------------------------------------------------------------------
  const float alpha = ep.alpha ? __ldg(ep.alpha) : 1.f;
  const bool c_vec = ((ldc & 3) == 0) && ((reinterpret_cast<uintptr_t>(C) & 15) == 0);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    if (m >= M) continue;
#pragma unroll
    for (int jh = 0; jh < 2; ++jh) {
      const int n = n0 + jh * 64 + tx * 4;
      if (n >= N) continue;
      float v[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) v[j] = alpha * acc[i][jh * 4 + j];
      const int nv = min(4, N - n);
      if (ep.mode == EPI_FWD) {
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          if (j < nv) {
            float y = v[j] + (ep.bias ? __ldg(ep.bias + n + j) : 0.f);
            if (ep.act == GCBF_ACT_RELU) y = fmaxf(y, 0.f);
            else if (ep.act == GCBF_ACT_TANH) y = tanhf(y);
            v[j] = y;
          }
        }
      } else if (ep.mode == EPI_DGRAD) {
        if (ep.relu_src) {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (j < nv) v[j] = (__ldg(ep.relu_src + (size_t)m * ep.ld_relu + n + j) > 0.f) ? v[j] : 0.f;
        }
      }
      float* dst = C + (size_t)blockIdx.z * ep.split_stride + (size_t)m * ldc + n;
      if (ep.accumulate) {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j < nv) dst[j] += v[j];
      } else if (nv == 4 && c_vec) {
        *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
      } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (j < nv) dst[j] = v[j];
      }
    }
  }
}

// column sums of dZ[M,N] -> db[N]; one block column-tile of 32 columns x 8 row-lanes, loop over rows.
__global__ void colsum_kernel(const float* __restrict__ dZ, int ld, int M, int N, float* __restrict__ db,
                              int accumulate, int rows_per_block) {
  __shared__ float part[8][33];
  const int col = blockIdx.x * 32 + threadIdx.x;
  const int r0 = blockIdx.y * rows_per_block;
  const int r1 = min(M, r0 + rows_per_block);
  float s = 0.f;
  if (col < N)
    for (int r = r0 + threadIdx.y; r < r1; r += 8) s += dZ[(size_t)r * ld + col];
  part[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && col < N) {
    float t = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) t += part[i][threadIdx.x];
    if (gridDim.y > 1) db[(size_t)blockIdx.y * N + col] = t;     // row block's partial; summed in order by add_partials
    else if (accumulate) db[col] += t;
    else db[col] = t;
  }
}

__global__ void act_bwd_kernel(const float* __restrict__ dY, const float* __restrict__ Y, float* __restrict__ dZ,
                               int64_t count, int act) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const float y = Y[i], g = dY[i];
  float d = g;
  if (act == GCBF_ACT_TANH) d = g * (1.f - y * y);
  else if (act == GCBF_ACT_RELU) d = (y > 0.f) ? g : 0.f;
  dZ[i] = d;
}

int launch_colsum_narrow(const float* dZ, int ld, int M, int N, float* db, int accumulate, cudaStream_t st);

int launch_colsum(const float* dZ, int ld, int M, int N, float* db, int accumulate, cudaStream_t st) {
  if (N <= 32) return launch_colsum_narrow(dZ, ld, M, N, db, accumulate, st);
  int rsplit = (int)imin64(64, imax64(1, (int64_t)M / 2048));
  int rows_per_block = ceil_div(M, rsplit);
  rsplit = ceil_div(M, rows_per_block);
  dim3 g2(ceil_div(N, 32), rsplit), b2(32, 8);
  if (rsplit == 1) {
    colsum_kernel<<<g2, b2, 0, st>>>(dZ, ld, M, N, db, accumulate, rows_per_block);
    GCBF_LAUNCH_OK();
    return GCBF_OK;
  }
  float* part = nullptr;
  GCBF_CUDA_OK(scratch_alloc((void**)&part, (size_t)rsplit * N * 4, st));
  colsum_kernel<<<g2, b2, 0, st>>>(dZ, ld, M, N, part, accumulate, rows_per_block);
  GCBF_LAUNCH_OK();
  GCBF_CUDA_OK(add_partials(part, rsplit, 1, N, db, N, accumulate, st));
  GCBF_CUDA_OK(scratch_free(part, st));
  return GCBF_OK;
}

int launch_simt_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma,
                    float* Y, int ldy, int M, int N, int K, int act, cudaStream_t st) {
  Epi ep{};
  ep.mode = EPI_FWD; ep.alpha = inv_sigma; ep.bias = bias; ep.act = act;
  dim3 grid(ceil_div(N, BN), ceil_div(M, BM), 1);
  gemm_simt_kernel<true, true><<<grid, NT, 0, st>>>(X, ldx, W, ldw, Y, ldy, M, N, K, ceil_div(K, BK) * BK, ep);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

int launch_simt_dgrad(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma,
                      const float* relu_src, int ld_relu, float* dX, int lddx, int M, int N, int K,
                      int accumulate, cudaStream_t st) {
  Epi ep{};
  ep.mode = EPI_DGRAD; ep.alpha = inv_sigma; ep.relu_src = relu_src; ep.ld_relu = ld_relu; ep.accumulate = accumulate;
  // C = dX [M, K]; reduction over N.  A = dZ (k-contiguous), B(n=kout, k=nred) = W[nred*ldw + kout].
  dim3 grid(ceil_div(K, BN), ceil_div(M, BM), 1);
  gemm_simt_kernel<true, false><<<grid, NT, 0, st>>>(dZ, lddz, W, ldw, dX, lddx, M, K, N, ceil_div(N, BK) * BK, ep);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

int launch_simt_wgrad(const float* dZ, int lddz, const float* X, int ldx, const float* inv_sigma, float* dW,
                      int lddw, float* db, int M, int N, int K, int accumulate, cudaStream_t st) {
  // C = dW [N, K]; reduction over M rows.  A(m=nout, k=row) = dZ[row*lddz + nout], B(n=kout, k=row) = X[row*ldx + kout].
  const int tiles = ceil_div(N, BM) * ceil_div(K, BN);
  int splits = 1;
  if (tiles < 2 * kNumSMs) splits = min(ceil_div(M, 4 * BK), max(1, (2 * kNumSMs) / tiles));
  int k_chunk = ceil_div(ceil_div(M, splits), BK) * BK;
  splits = ceil_div(M, k_chunk);
  Epi ep{};
  ep.mode = EPI_WGRAD; ep.alpha = inv_sigma; ep.accumulate = accumulate;
  dim3 grid(ceil_div(K, BN), ceil_div(N, BM), splits);
  if (splits == 1) {
    gemm_simt_kernel<false, false><<<grid, NT, 0, st>>>(dZ, lddz, X, ldx, dW, lddw, N, K, M, k_chunk, ep);
    GCBF_LAUNCH_OK();
  } else {
    // each contraction split writes its own [N][K] slice; the slices are summed in order
    float* part = nullptr;
    GCBF_CUDA_OK(scratch_alloc((void**)&part, (size_t)splits * N * K * 4, st));
    ep.accumulate = 0;
    ep.split_stride = (size_t)N * K;
    gemm_simt_kernel<false, false><<<grid, NT, 0, st>>>(dZ, lddz, X, ldx, part, K, N, K, M, k_chunk, ep);
    GCBF_LAUNCH_OK();
    GCBF_CUDA_OK(add_partials(part, splits, N, K, dW, lddw, accumulate, st));
    GCBF_CUDA_OK(scratch_free(part, st));
  }
  if (db) return launch_colsum(dZ, lddz, M, N, db, accumulate, st);
  return GCBF_OK;
}

}  // namespace gcbf

extern "C" int gcbf_act_bwd(const float* dY, const float* Y, float* dZ, int64_t count, int act, void* stream) {
  GCBF_REQUIRE(dY && Y && dZ && count >= 0, "gcbf_act_bwd: bad arguments");
  if (count == 0) return GCBF_OK;
  gcbf::act_bwd_kernel<<<gcbf::ceil_div(count, 256), 256, 0, gcbf::as_stream(stream)>>>(dY, Y, dZ, count, act);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}
