// Shared helpers for libgcbf_b200 (sm_90a).  Error reporting, launch checks, warp reductions.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include "gcbf_b200.h"

namespace gcbf {

void set_error(const char* fmt, ...);

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

// Stream-ordered scratch for per-block partial results, and their sum in a fixed order (reduce.cu):
// target[r * ldt + c] = (accumulate ? target[r * ldt + c] : 0) + part[0][r][c] + part[1][r][c] + ...   (parts of rows x cols each)
cudaError_t scratch_alloc(void** p, size_t bytes, cudaStream_t st);
cudaError_t scratch_free(void* p, cudaStream_t st);
cudaError_t add_partials(const float* part, int parts, int rows, int cols, float* target, int ldt, int accumulate, cudaStream_t st);

// d_states += the VJP of edge_attr like gcbf_edge_attr_bwd, summed in a fixed order (graph.cu); needs the batch's node count
int edge_attr_bwd_ordered(int env, const float* states, int ld_state, const int64_t* edge_index, int64_t num_edges, int num_nodes,
                          const float* d_edge_attr, float* d_states, cudaStream_t st);

// in-place single-block exclusive scan of `count` int32 values, data[count] <- total (graph.cu; shared with macbf.cu)
cudaError_t exclusive_scan_i32(int32_t* data, int count, cudaStream_t st);

#define GCBF_REQUIRE(cond, ...)                 \
  do {                                          \
    if (!(cond)) {                              \
      ::gcbf::set_error(__VA_ARGS__);           \
      return GCBF_E_INVALID;                    \
    }                                           \
  } while (0)

#define GCBF_CUDA_OK(expr)                                                                   \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess) {                                                                 \
      ::gcbf::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return GCBF_E_CUDA;                                                                    \
    }                                                                                        \
  } while (0)

#define GCBF_LAUNCH_OK() GCBF_CUDA_OK(cudaGetLastError())

constexpr int kNumSMs = 132;  // H100 SXM

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ int warp_sum_int(int v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

inline int ceil_div(int64_t a, int64_t b) { return (int)((a + b - 1) / b); }
inline int64_t imin64(int64_t a, int64_t b) { return a < b ? a : b; }
inline int64_t imax64(int64_t a, int64_t b) { return a > b ? a : b; }

}  // namespace gcbf
