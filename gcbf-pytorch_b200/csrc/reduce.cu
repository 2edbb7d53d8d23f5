// Deterministic cross-block sums.  A kernel whose blocks each produce a partial result for the same outputs (split-K GEMMs,
// column sums over row blocks, scatters over edges) writes its partials into stream-ordered scratch and add_partials adds them
// in a fixed order, so results do not depend on which block finishes first (float atomics would make them run-dependent).
#include <mutex>

#include "common.cuh"

namespace gcbf {

// The library's own stream-ordered pool per device (the process's default pool and its settings are left alone); freed scratch
// stays cached in it rather than going back to the driver at every synchronisation.
static std::mutex g_pool_mutex;
static cudaMemPool_t g_pools[64];

cudaError_t scratch_alloc(void** p, size_t bytes, cudaStream_t st) {
  int dev = 0;
  if (cudaError_t e = cudaGetDevice(&dev)) return e;
  if (dev < 0 || dev >= 64) return cudaErrorInvalidDevice;
  cudaMemPool_t pool;
  {
    std::lock_guard<std::mutex> lock(g_pool_mutex);
    if (!g_pools[dev]) {
      cudaMemPoolProps props = {};
      props.allocType = cudaMemAllocationTypePinned;
      props.location.type = cudaMemLocationTypeDevice;
      props.location.id = dev;
      if (cudaError_t e = cudaMemPoolCreate(&g_pools[dev], &props)) return e;
      uint64_t keep = UINT64_MAX;
      cudaMemPoolSetAttribute(g_pools[dev], cudaMemPoolAttrReleaseThreshold, &keep);
    }
    pool = g_pools[dev];
  }
  return cudaMallocFromPoolAsync(p, bytes < 256 ? 256 : bytes, pool, st);
}

cudaError_t scratch_free(void* p, cudaStream_t st) { return cudaFreeAsync(p, st); }

__global__ void add_partials_kernel(const float* __restrict__ part, int parts, int64_t n, int cols, float* __restrict__ target,
                                    int ldt, int accumulate) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float* t = target + (i / cols) * ldt + (i % cols);
    float s = accumulate ? *t : 0.f;
    for (int p = 0; p < parts; ++p) s += part[(int64_t)p * n + i];
    *t = s;
  }
}

cudaError_t add_partials(const float* part, int parts, int rows, int cols, float* target, int ldt, int accumulate, cudaStream_t st) {
  const int64_t n = (int64_t)rows * cols;
  if (n == 0) return cudaSuccess;
  add_partials_kernel<<<(int)imin64(ceil_div(n, 256), 8 * kNumSMs), 256, 0, st>>>(part, parts, n, cols, target, ldt, accumulate);
  return cudaGetLastError();
}

}  // namespace gcbf
