// Linear layers with FEW ROWS (M <= 64): the rollout-time forward of a single graph (reference gcbf/algo/gcbf.py:128-139: 16 agents,
// ~45 edges per env step) and the plumbing config C1.  With so few rows a layer is a stream over its WEIGHTS (2048 x 2048 fp32 = 16 MB,
// resident in the 50 MB L2 from one pass to the next), not a GEMM tile problem: a 128 x 128 tile grid puts 16 CTAs on 132 SMs.
//   fwd   : Y[M,N]   = act(alpha * X W^T + b)      warp = 2 output columns, lanes split K (16-byte loads of W rows), shuffle-reduce
//   dgrad : dX[M,K] (+)= alpha * dZ W (* mask)      thread = 4 consecutive k (16-byte loads of W rows), N split over blockIdx.y,
//                                                   partial sums (already masked / scaled: both are linear) added atomically
//   wgrad : dW[N,K] (+)= alpha * dZ^T X             thread = (n, 4 consecutive k): a streaming write of dW, X / dZ tiles in smem
// Exact fp32 FFMA arithmetic like gemm_simt.cu (different summation order).
//
// Round 2: the 16-byte-aligned shapes (every hidden layer) run the TILED kernels below instead -- one CTA owns all (<= 64) rows x 16
// output columns, stages X / W chunks in shared memory with cp.async (two stages), 4 x 4 register tiles, the contraction split
// four ways inside the CTA and up to eight ways across a thread-block CLUSTER whose partial tiles are summed through distributed shared
// memory by rank 0 (no atomics, no scratch buffer, no second launch, deterministic).  The launch list of GCBF.apply on one 16-agent
// graph showed the first version at 110-310 us per 2048-wide layer (latency-bound: 8 warps per SM, every lane issuing its own X loads);
// the tiled kernels are FFMA-issue bound.  The kernels above stay as the fallback for unaligned shapes.
#include <cooperative_groups.h>

#include "common.cuh"

namespace cg = cooperative_groups;

namespace gcbf {

constexpr int FR_MAX_M = 64;
constexpr int FR_MT = 16;           // rows per register tile

bool fewrows_supported(int M, int N, int K) { return M >= 1 && M <= FR_MAX_M && N >= 64 && K >= 32; }

// ---- forward -------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) fewrows_fwd_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ W, int ldw,
                                                          const float* __restrict__ bias, const float* __restrict__ alpha_p,
                                                          float* __restrict__ Y, int ldy, int M, int N, int K, int act, int vec_ok) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = (blockIdx.x * 8 + warp) * 2;
  if (n0 >= N) return;
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  const bool two = n0 + 1 < N;
  const float* w0 = W + (size_t)n0 * ldw;
  const float* w1 = W + (size_t)(two ? n0 + 1 : n0) * ldw;
  for (int m0 = 0; m0 < M; m0 += FR_MT) {
    float acc0[FR_MT], acc1[FR_MT];
#pragma unroll
    for (int r = 0; r < FR_MT; ++r) { acc0[r] = 0.f; acc1[r] = 0.f; }
    if (vec_ok) {
      for (int k = lane * 4; k < K; k += 128) {
        const float4 a = __ldg(reinterpret_cast<const float4*>(w0 + k));
        const float4 b = __ldg(reinterpret_cast<const float4*>(w1 + k));
#pragma unroll
        for (int r = 0; r < FR_MT; ++r) {
          if (m0 + r < M) {
            const float4 x = __ldg(reinterpret_cast<const float4*>(X + (size_t)(m0 + r) * ldx + k));
            acc0[r] = fmaf(x.x, a.x, acc0[r]); acc0[r] = fmaf(x.y, a.y, acc0[r]); acc0[r] = fmaf(x.z, a.z, acc0[r]); acc0[r] = fmaf(x.w, a.w, acc0[r]);
            acc1[r] = fmaf(x.x, b.x, acc1[r]); acc1[r] = fmaf(x.y, b.y, acc1[r]); acc1[r] = fmaf(x.z, b.z, acc1[r]); acc1[r] = fmaf(x.w, b.w, acc1[r]);
          }
        }
      }
    } else {
      for (int k = lane; k < K; k += 32) {
        const float a = __ldg(w0 + k), b = __ldg(w1 + k);
#pragma unroll
        for (int r = 0; r < FR_MT; ++r) {
          if (m0 + r < M) {
            const float x = __ldg(X + (size_t)(m0 + r) * ldx + k);
            acc0[r] = fmaf(x, a, acc0[r]);
            acc1[r] = fmaf(x, b, acc1[r]);
          }
        }
      }
    }
#pragma unroll
    for (int r = 0; r < FR_MT; ++r) { acc0[r] = warp_sum(acc0[r]); acc1[r] = warp_sum(acc1[r]); }
    // lane r writes row m0 + r (both columns)
#pragma unroll
    for (int r = 0; r < FR_MT; ++r) {
      if (lane == r && m0 + r < M) {
        float y0 = alpha * acc0[r] + (bias ? __ldg(bias + n0) : 0.f);
        float y1 = alpha * acc1[r] + ((bias && two) ? __ldg(bias + n0 + 1) : 0.f);
        if (act == GCBF_ACT_RELU) { y0 = fmaxf(y0, 0.f); y1 = fmaxf(y1, 0.f); }
        else if (act == GCBF_ACT_TANH) { y0 = tanhf(y0); y1 = tanhf(y1); }
        float* d = Y + (size_t)(m0 + r) * ldy + n0;
        d[0] = y0;
        if (two) d[1] = y1;
      }
    }
  }
}

// ---- data gradient -------------------------------------------------------------------------------------------------------------
constexpr int FRD_NSLICE = 32;      // rows of W (contraction indices) per block

__global__ void __launch_bounds__(128) fewrows_dgrad_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ W, int ldw,
                                                            const float* __restrict__ alpha_p, const float* __restrict__ relu_src,
                                                            int ld_relu, float* __restrict__ dX, int lddx, int M, int N, int K, int m0) {
  __shared__ float dzs[FR_MT][FRD_NSLICE];
  const int k = (blockIdx.x * 128 + threadIdx.x) * 4;
  const int nb = blockIdx.y * FRD_NSLICE, ne = min(N, nb + FRD_NSLICE);
  for (int i = threadIdx.x; i < FR_MT * FRD_NSLICE; i += 128) {
    const int r = i / FRD_NSLICE, n = i % FRD_NSLICE;
    dzs[r][n] = (m0 + r < M && nb + n < N) ? dZ[(size_t)(m0 + r) * lddz + nb + n] : 0.f;
  }
  __syncthreads();
  if (k >= K) return;
  const bool full = (k + 3 < K) && ((ldw & 3) == 0) && ((reinterpret_cast<uintptr_t>(W) & 15) == 0);
  float acc[FR_MT][4];
#pragma unroll
  for (int r = 0; r < FR_MT; ++r) { acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f; }
  for (int n = nb; n < ne; ++n) {
    float4 w;
    const float* wr = W + (size_t)n * ldw + k;
    if (full) w = __ldg(reinterpret_cast<const float4*>(wr));
    else { w.x = wr[0]; w.y = (k + 1 < K) ? wr[1] : 0.f; w.z = (k + 2 < K) ? wr[2] : 0.f; w.w = (k + 3 < K) ? wr[3] : 0.f; }
#pragma unroll
    for (int r = 0; r < FR_MT; ++r) {
      const float z = dzs[r][n - nb];
      acc[r][0] = fmaf(z, w.x, acc[r][0]); acc[r][1] = fmaf(z, w.y, acc[r][1]);
      acc[r][2] = fmaf(z, w.z, acc[r][2]); acc[r][3] = fmaf(z, w.w, acc[r][3]);
    }
  }
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
#pragma unroll
  for (int r = 0; r < FR_MT; ++r) {
    if (m0 + r >= M) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (k + j >= K) continue;
      float v = alpha * acc[r][j];
      if (relu_src && !(relu_src[(size_t)(m0 + r) * ld_relu + k + j] > 0.f)) v = 0.f;      // mask and alpha are linear: applied per partial
      dX[((size_t)blockIdx.y * M + m0 + r) * lddx + k + j] = v;      // this contraction slice's partial ([slices][M][K]), summed in order
    }
  }
}

// ---- weight gradient -----------------------------------------------------------------------------------------------------------
constexpr int FRW_KT = 128, FRW_NT = 32;

__global__ void __launch_bounds__(256) fewrows_wgrad_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ X, int ldx,
                                                            const float* __restrict__ alpha_p, float* __restrict__ dW, int lddw, int M,
                                                            int N, int K, int accumulate) {
  __shared__ __align__(16) float xs[FR_MAX_M][FRW_KT];
  __shared__ float zs[FR_MAX_M][FRW_NT + 1];
  const int k0 = blockIdx.x * FRW_KT, n0 = blockIdx.y * FRW_NT;
  for (int i = threadIdx.x; i < M * FRW_KT; i += 256) {
    const int r = i / FRW_KT, c = i % FRW_KT;
    xs[r][c] = (k0 + c < K) ? X[(size_t)r * ldx + k0 + c] : 0.f;
  }
  for (int i = threadIdx.x; i < M * FRW_NT; i += 256) {
    const int r = i / FRW_NT, c = i % FRW_NT;
    zs[r][c] = (n0 + c < N) ? dZ[(size_t)r * lddz + n0 + c] : 0.f;
  }
  __syncthreads();
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  const int kc = (threadIdx.x & 31) * 4;
  const bool vec = ((lddw & 3) == 0) && ((reinterpret_cast<uintptr_t>(dW) & 15) == 0) && (k0 + kc + 3 < K);
#pragma unroll
  for (int pass = 0; pass < FRW_NT / 8; ++pass) {
    const int nl = pass * 8 + (threadIdx.x >> 5);
    const int n = n0 + nl;
    if (n >= N || k0 + kc >= K) continue;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    for (int m = 0; m < M; ++m) {
      const float z = zs[m][nl];
      const float4 x = *reinterpret_cast<const float4*>(&xs[m][kc]);
      acc.x = fmaf(z, x.x, acc.x); acc.y = fmaf(z, x.y, acc.y); acc.z = fmaf(z, x.z, acc.z); acc.w = fmaf(z, x.w, acc.w);
    }
    acc.x *= alpha; acc.y *= alpha; acc.z *= alpha; acc.w *= alpha;
    float* d = dW + (size_t)n * lddw + k0 + kc;
    if (vec) {
      if (accumulate) { const float4 o = *reinterpret_cast<const float4*>(d); acc.x += o.x; acc.y += o.y; acc.z += o.z; acc.w += o.w; }
      *reinterpret_cast<float4*>(d) = acc;
    } else {
      const float v[4] = {acc.x, acc.y, acc.z, acc.w};
      for (int j = 0; j < 4; ++j)
        if (k0 + kc + j < K) d[j] = accumulate ? d[j] + v[j] : v[j];
    }
  }
}


// ---- tiled kernels (aligned shapes) ----------------------------------------------------------------------------------------------
constexpr int FT_BN = 16;                 // output columns per CTA
constexpr int FT_KC = 128;                // contraction elements per stage
constexpr int FT_LD = FT_KC + 4;          // shared-memory row pitch in floats (132 % 32 = 4: conflict-free 16-byte row-strided loads)
constexpr int FT_FWD_STAGE = (FR_MAX_M + FT_BN) * FT_LD;                         // floats per stage: X rows then W rows
constexpr size_t FT_FWD_SMEM = (size_t)2 * FT_FWD_STAGE * sizeof(float);         // 84,480 B
constexpr int FT_DG_STAGE = FT_KC * FR_MAX_M + FT_KC * FT_BN;                    // dZ^T [128][64] then W [128][16]
constexpr size_t FT_DG_SMEM = (size_t)2 * FT_DG_STAGE * sizeof(float);           // 81,920 B

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  const int sz = valid ? 16 : 0;          // src-size 0: the 16 bytes are zero-filled, nothing is read
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gsrc), "r"(sz) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

// sum the four in-CTA contraction groups, then the cluster's CTAs (rank 0 reads its peers' tiles over DSMEM); returns this thread's
// float4 of the [64 x 16] tile (row = t / 4, columns 4 * (t % 4) ...) -- valid on cluster rank 0 only
__device__ __forceinline__ float4 ft_reduce(float (&acc)[4][4], float* smem, int row_of_i_stride, int row_base) {
  cg::cluster_group cluster = cg::this_cluster();
  const int t = threadIdx.x, kg = t >> 6;
  float* red = smem;                                     // [4][64][16]
  float* part = smem + 4 * FR_MAX_M * FT_BN;             // [64][16]: this CTA's tile
  const int tc = t & 3;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int row = row_base + i * row_of_i_stride;
    *reinterpret_cast<float4*>(&red[(kg * FR_MAX_M + row) * FT_BN + tc * 4]) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
  }
  __syncthreads();
  float4 s = *reinterpret_cast<const float4*>(&red[t * 4]);
#pragma unroll
  for (int g = 1; g < 4; ++g) {
    const float4 o = *reinterpret_cast<const float4*>(&red[g * FR_MAX_M * FT_BN + t * 4]);
    s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
  }
  const unsigned S = cluster.num_blocks();
  if (S > 1) {
    *reinterpret_cast<float4*>(&part[t * 4]) = s;
    cluster.sync();
    if (cluster.block_rank() == 0) {
      for (unsigned r = 1; r < S; ++r) {
        const float4 o = *reinterpret_cast<const float4*>(cluster.map_shared_rank(part, r) + t * 4);
        s.x += o.x; s.y += o.y; s.z += o.z; s.w += o.w;
      }
    }
    cluster.sync();                                      // peers keep their shared memory alive until rank 0 has read it
  }
  return s;
}

// Y[M, N] = act(alpha * X W^T + b); grid (ceil(N / 16), S), cluster (1, S, 1): CTA y owns contraction range [y * k_per_cta, ...)
__global__ void __launch_bounds__(256) fewrows_fwd_tiled_kernel(const float* __restrict__ X, int ldx, const float* __restrict__ W, int ldw,
                                                                const float* __restrict__ bias, const float* __restrict__ alpha_p,
                                                                float* __restrict__ Y, int ldy, int M, int N, int K, int act, int k_per_cta) {
  extern __shared__ __align__(16) float ft_smem[];
  const int t = threadIdx.x, kg = t >> 6, tt = t & 63, tc = tt & 3, tr = tt >> 2;
  const int n0 = blockIdx.x * FT_BN;
  const int k_lo = blockIdx.y * k_per_cta, k_hi = min(K, k_lo + k_per_cta);
  const int nchunks = k_hi > k_lo ? (k_hi - k_lo + FT_KC - 1) / FT_KC : 0;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }

  auto load = [&](int c, int buf) {
    float* xs = ft_smem + buf * FT_FWD_STAGE;
    float* ws = xs + FR_MAX_M * FT_LD;
    const int kb = k_lo + c * FT_KC;
#pragma unroll
    for (int u = 0; u < 8; ++u) {                        // X: 64 rows x 32 float4
      const int idx = t + 256 * u, row = idx >> 5, k = kb + (idx & 31) * 4;
      const bool ok = row < M && k < k_hi;
      cp_async16(&xs[row * FT_LD + (idx & 31) * 4], ok ? X + (size_t)row * ldx + k : X, ok);
    }
#pragma unroll
    for (int u = 0; u < 2; ++u) {                        // W: 16 rows x 32 float4
      const int idx = t + 256 * u, col = idx >> 5, k = kb + (idx & 31) * 4;
      const bool ok = n0 + col < N && k < k_hi;
      cp_async16(&ws[col * FT_LD + (idx & 31) * 4], ok ? W + (size_t)(n0 + col) * ldw + k : W, ok);
    }
    cp_async_commit();
  };

  if (nchunks > 0) load(0, 0);
  for (int c = 0; c < nchunks; ++c) {
    const int buf = c & 1;
    if (c + 1 < nchunks) { load(c + 1, buf ^ 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();
    const float* xs = ft_smem + buf * FT_FWD_STAGE;
    const float* ws = xs + FR_MAX_M * FT_LD;
#pragma unroll
    for (int q = 0; q < 8; ++q) {                        // this contraction group's 32 of the stage's 128 elements
      const int k4 = (kg * 8 + q) * 4;
      float4 w[4], x[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) w[j] = *reinterpret_cast<const float4*>(&ws[(tc * 4 + j) * FT_LD + k4]);
#pragma unroll
      for (int i = 0; i < 4; ++i) x[i] = *reinterpret_cast<const float4*>(&xs[(tr + 16 * i) * FT_LD + k4]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          acc[i][j] = fmaf(x[i].x, w[j].x, acc[i][j]); acc[i][j] = fmaf(x[i].y, w[j].y, acc[i][j]);
          acc[i][j] = fmaf(x[i].z, w[j].z, acc[i][j]); acc[i][j] = fmaf(x[i].w, w[j].w, acc[i][j]);
        }
    }
    __syncthreads();                                     // the stage is overwritten by the load issued in the next iteration
  }
  const float4 s = ft_reduce(acc, ft_smem, 16, tr);
  if (cg::this_cluster().block_rank() != 0) return;
  const int row = t >> 2, col = n0 + (t & 3) * 4;
  if (row >= M) return;
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  const float v[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (col + j >= N) break;
    float y = alpha * v[j] + (bias ? __ldg(bias + col + j) : 0.f);
    if (act == GCBF_ACT_RELU) y = fmaxf(y, 0.f);
    else if (act == GCBF_ACT_TANH) y = tanhf(y);
    Y[(size_t)row * ldy + col + j] = y;
  }
}

// dX[M, K] (+)= alpha * dZ W (* mask); grid (ceil(K / 16), S), cluster (1, S, 1): CTA y owns the contraction rows [y * n_per_cta, ...) of W
__global__ void __launch_bounds__(256) fewrows_dgrad_tiled_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ W, int ldw,
                                                                  const float* __restrict__ alpha_p, const float* __restrict__ relu_src,
                                                                  int ld_relu, float* __restrict__ dX, int lddx, int M, int N, int K,
                                                                  int accumulate, int n_per_cta) {
  extern __shared__ __align__(16) float ft_smem[];
  const int t = threadIdx.x, kg = t >> 6, tt = t & 63, tc = tt & 3, tr = tt >> 2;
  const int k0 = blockIdx.x * FT_BN;
  const int n_lo = blockIdx.y * n_per_cta, n_hi = min(N, n_lo + n_per_cta);
  const int nchunks = n_hi > n_lo ? (n_hi - n_lo + FT_KC - 1) / FT_KC : 0;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }
  const int zr = t & 63, zq = t >> 6;                    // dZ staging: thread = (row, one of four float4 columns per 16 contraction elements)
  float4 zreg[8];

  auto load_w = [&](int c, int buf) {                    // W rows [nb, nb + 128) x 16 columns: 4 float4 per row
    float* ws = ft_smem + buf * FT_DG_STAGE + FT_KC * FR_MAX_M;
    const int nb = n_lo + c * FT_KC;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int idx = t + 256 * u, nn = idx >> 2, k = k0 + (idx & 3) * 4;
      const bool ok = nb + nn < n_hi && k < K;
      cp_async16(&ws[nn * FT_BN + (idx & 3) * 4], ok ? W + (size_t)(nb + nn) * ldw + k : W, ok);
    }
    cp_async_commit();
  };
  auto load_z = [&](int c) {                             // dZ[row][nb + 16 u + 4 zq ...] -> registers
    const int nb = n_lo + c * FT_KC;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int n = nb + (u * 4 + zq) * 4;
      zreg[u] = (zr < M && n < n_hi) ? __ldg(reinterpret_cast<const float4*>(dZ + (size_t)zr * lddz + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_z = [&](int buf) {                          // transposed: zs[n][row], consecutive threads = consecutive rows
    float* zs = ft_smem + buf * FT_DG_STAGE;
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const int nn = (u * 4 + zq) * 4;
      zs[(nn + 0) * FR_MAX_M + zr] = zreg[u].x; zs[(nn + 1) * FR_MAX_M + zr] = zreg[u].y;
      zs[(nn + 2) * FR_MAX_M + zr] = zreg[u].z; zs[(nn + 3) * FR_MAX_M + zr] = zreg[u].w;
    }
  };

  if (nchunks > 0) { load_w(0, 0); load_z(0); store_z(0); }
  for (int c = 0; c < nchunks; ++c) {
    const int buf = c & 1;
    if (c + 1 < nchunks) { load_w(c + 1, buf ^ 1); load_z(c + 1); cp_async_wait<1>(); } else { cp_async_wait<0>(); }
    __syncthreads();
    const float* zs = ft_smem + buf * FT_DG_STAGE;
    const float* ws = zs + FT_KC * FR_MAX_M;
#pragma unroll 8
    for (int q = 0; q < 32; ++q) {                       // this contraction group's 32 of the stage's 128 rows of W
      const int nn = kg * 32 + q;
      const float4 z = *reinterpret_cast<const float4*>(&zs[nn * FR_MAX_M + tr * 4]);
      const float4 w = *reinterpret_cast<const float4*>(&ws[nn * FT_BN + tc * 4]);
      const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        acc[i][0] = fmaf(zz[i], w.x, acc[i][0]); acc[i][1] = fmaf(zz[i], w.y, acc[i][1]);
        acc[i][2] = fmaf(zz[i], w.z, acc[i][2]); acc[i][3] = fmaf(zz[i], w.w, acc[i][3]);
      }
    }
    if (c + 1 < nchunks) store_z(buf ^ 1);               // the other stage was released by the barrier at the end of the previous iteration
    __syncthreads();
  }
  const float4 s = ft_reduce(acc, ft_smem, 1, tr * 4);
  if (cg::this_cluster().block_rank() != 0) return;
  const int row = t >> 2, col = k0 + (t & 3) * 4;
  if (row >= M) return;
  const float alpha = alpha_p ? __ldg(alpha_p) : 1.f;
  const float v[4] = {s.x, s.y, s.z, s.w};
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    if (col + j >= K) break;
    float g = alpha * v[j];
    if (relu_src && !(relu_src[(size_t)row * ld_relu + col + j] > 0.f)) g = 0.f;
    float* d = dX + (size_t)row * lddx + col + j;
    *d = accumulate ? *d + g : g;
  }
}

// dX[M, K] (+)= alpha * dZ W (* mask) for a NARROW input (K <= 32: the first phi layer, whose input gradient is d edge_attr): one block
// per row, threads = (k, contraction lane), partial sums reduced through shared memory
__global__ void __launch_bounds__(256) fewrows_dgrad_narrow_kernel(const float* __restrict__ dZ, int lddz, const float* __restrict__ W, int ldw,
                                                                   const float* __restrict__ alpha_p, const float* __restrict__ relu_src,
                                                                   int ld_relu, float* __restrict__ dX, int lddx, int N, int K, int KP,
                                                                   int accumulate) {
  __shared__ float part[256];
  const int m = blockIdx.x, t = threadIdx.x;
  const int k = t % KP, lane = t / KP, lanes = 256 / KP;
  float acc = 0.f;
  if (k < K) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;         // four independent load / FMA chains per thread
    int n = lane;
    for (; n + 3 * lanes < N; n += 4 * lanes) {
      const float z0 = __ldg(dZ + (size_t)m * lddz + n), z1 = __ldg(dZ + (size_t)m * lddz + n + lanes);
      const float z2 = __ldg(dZ + (size_t)m * lddz + n + 2 * lanes), z3 = __ldg(dZ + (size_t)m * lddz + n + 3 * lanes);
      const float w0 = __ldg(W + (size_t)n * ldw + k), w1 = __ldg(W + (size_t)(n + lanes) * ldw + k);
      const float w2 = __ldg(W + (size_t)(n + 2 * lanes) * ldw + k), w3 = __ldg(W + (size_t)(n + 3 * lanes) * ldw + k);
      a0 = fmaf(z0, w0, a0); a1 = fmaf(z1, w1, a1); a2 = fmaf(z2, w2, a2); a3 = fmaf(z3, w3, a3);
    }
    for (; n < N; n += lanes) a0 = fmaf(__ldg(dZ + (size_t)m * lddz + n), __ldg(W + (size_t)n * ldw + k), a0);
    acc = (a0 + a1) + (a2 + a3);
  }
  part[t] = acc;
  __syncthreads();
  for (int s = lanes >> 1; s > 0; s >>= 1) {
    if (lane < s) part[t] += part[t + s * KP];
    __syncthreads();
  }
  if (lane == 0 && k < K) {
    float g = (alpha_p ? __ldg(alpha_p) : 1.f) * part[t];
    if (relu_src && !(relu_src[(size_t)m * ld_relu + k] > 0.f)) g = 0.f;
    float* d = dX + (size_t)m * lddx + k;
    *d = accumulate ? *d + g : g;
  }
}

// contraction split over a cluster: enough CTAs to cover the SMs, at least one 128-element stage per CTA, at most 8 (portable cluster size)
static int ft_split(int tiles, int contraction) {
  int S = 1;
  while (S < 8 && tiles * S * 2 <= 2 * kNumSMs && contraction / (2 * S) >= FT_KC) S *= 2;
  return S;
}

template <typename... Args>
static int ft_launch(void (*kernel)(Args...), dim3 grid, int S, size_t smem, cudaStream_t st, Args... args) {
  static thread_local void* configured[4] = {nullptr, nullptr, nullptr, nullptr};
  bool done = false;
  for (void* p : configured) done |= (p == (void*)kernel);
  if (!done) {
    GCBF_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (void*& p : configured) if (!p) { p = (void*)kernel; break; }
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(256); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1; attr[0].val.clusterDim.y = S; attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  GCBF_CUDA_OK(cudaLaunchKernelEx(&cfg, kernel, args...));
  return GCBF_OK;
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int launch_colsum(const float* dZ, int lddz, int M, int N, float* db, int accumulate, cudaStream_t st);

int launch_fewrows_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, float* Y, int ldy, int M,
                       int N, int K, int act, cudaStream_t st) {
  const int vec_ok = ((K & 3) == 0 && (ldx & 3) == 0 && (ldw & 3) == 0 && (reinterpret_cast<uintptr_t>(X) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(W) & 15) == 0) ? 1 : 0;
  if (vec_ok) {
    const int tiles = ceil_div(N, FT_BN), S = ft_split(tiles, K);
    const int k_per_cta = ceil_div(ceil_div(K, S), FT_KC) * FT_KC;
    return ft_launch(fewrows_fwd_tiled_kernel, dim3(tiles, S), S, FT_FWD_SMEM, st, X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, k_per_cta);
  }
  fewrows_fwd_kernel<<<ceil_div(N, 16), 256, 0, st>>>(X, ldx, W, ldw, bias, inv_sigma, Y, ldy, M, N, K, act, vec_ok);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

int launch_fewrows_dgrad(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma, const float* relu_src, int ld_relu,
                         float* dX, int lddx, int M, int N, int K, int accumulate, cudaStream_t st) {
  if ((K & 3) == 0 && (N & 3) == 0 && (lddz & 3) == 0 && (ldw & 3) == 0 && aligned16(dZ) && aligned16(W)) {
    const int tiles = ceil_div(K, FT_BN), S = ft_split(tiles, N);
    const int n_per_cta = ceil_div(ceil_div(N, S), FT_KC) * FT_KC;
    return ft_launch(fewrows_dgrad_tiled_kernel, dim3(tiles, S), S, FT_DG_SMEM, st, dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, M, N, K,
                     accumulate, n_per_cta);
  }
  const int slices = ceil_div(N, FRD_NSLICE);
  float* part = nullptr;
  GCBF_CUDA_OK(scratch_alloc((void**)&part, (size_t)slices * M * K * 4, st));
  for (int m0 = 0; m0 < M; m0 += FR_MT) {
    fewrows_dgrad_kernel<<<dim3(ceil_div(K, 512), slices), 128, 0, st>>>(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, part, K, M, N, K, m0);
    GCBF_LAUNCH_OK();
  }
  GCBF_CUDA_OK(add_partials(part, slices, M, K, dX, lddx, accumulate, st));
  GCBF_CUDA_OK(scratch_free(part, st));
  return GCBF_OK;
}

bool fewrows_narrow_supported(int M, int N, int K) { return M >= 1 && M <= FR_MAX_M && K >= 1 && K <= 32 && N >= 64; }

int launch_fewrows_dgrad_narrow(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma, const float* relu_src, int ld_relu,
                                float* dX, int lddx, int M, int N, int K, int accumulate, cudaStream_t st) {
  int KP = 1;
  while (KP < K) KP *= 2;
  fewrows_dgrad_narrow_kernel<<<M, 256, 0, st>>>(dZ, lddz, W, ldw, inv_sigma, relu_src, ld_relu, dX, lddx, N, K, KP, accumulate);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

int launch_fewrows_wgrad(const float* dZ, int lddz, const float* X, int ldx, const float* inv_sigma, float* dW, int lddw, float* db, int M, int N,
                         int K, int accumulate, cudaStream_t st) {
  fewrows_wgrad_kernel<<<dim3(ceil_div(K, FRW_KT), ceil_div(N, FRW_NT)), 256, 0, st>>>(dZ, lddz, X, ldx, inv_sigma, dW, lddw, M, N, K, accumulate);
  GCBF_LAUNCH_OK();
  if (db) return launch_colsum(dZ, lddz, M, N, db, accumulate, st);
  return GCBF_OK;
}

}  // namespace gcbf
