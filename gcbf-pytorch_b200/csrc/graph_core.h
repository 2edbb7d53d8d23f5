// Per-element arithmetic of the graph build, written once for device and host: the K1 pair rule (radius_graph_kernel in graph.cu
// and the probe graphs of field.cu) and the K2 edge-feature map g(s) (edge_attr_fwd_kernel in graph.cu and field.cu).
// tests/host_driver/field_host.cpp compiles the same functions with g++ -ffp-contract=off for the CPU test-suite.
//   metric 0 (SimpleCar -> torch_cluster.radius_graph, reference gcbf/env/simple_car.py:32-33,249-252):
//       d2 = 0; d2 = d2 + (dx*dx) for each dim, NO fma contraction;  hit = d2 < r*r
//   metric 1 (DubinsCar / SimpleDrone, gcbf/env/dubins_car.py:730-746, simple_drone.py:316-333):
//       torch.norm on CPU accumulates acc = fma(d, d, acc) per dim, then sqrt;  hit = sqrtf(acc) < r
#pragma once
#include <math.h>
#include <stdint.h>

#include "gcbf_b200.h"

#if defined(__CUDACC__)
#define GCBF_GHD __host__ __device__ __forceinline__
#else
#define GCBF_GHD inline
#endif

namespace gcbf {
namespace graph {

#if defined(__CUDA_ARCH__)
GCBF_GHD float add_rn(float a, float b) { return __fadd_rn(a, b); }
GCBF_GHD float sub_rn(float a, float b) { return __fsub_rn(a, b); }
GCBF_GHD float mul_rn(float a, float b) { return __fmul_rn(a, b); }
GCBF_GHD float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
GCBF_GHD float sqrt_rn(float a) { return __fsqrt_rn(a); }
#else
GCBF_GHD float add_rn(float a, float b) { return a + b; }
GCBF_GHD float sub_rn(float a, float b) { return a - b; }
GCBF_GHD float mul_rn(float a, float b) { return a * b; }
GCBF_GHD float fma_rn(float a, float b, float c) { return fmaf(a, b, c); }
GCBF_GHD float sqrt_rn(float a) { return sqrtf(a); }
#endif

// is node j (position pj) a neighbour of node i (position pi)?  r2 = r * r rounded to fp32
GCBF_GHD bool pair_hit(const float* pi, const float* pj, int pos_dim, float r, float r2, int metric) {
  if (metric == 0) {
    float d2 = 0.f;
    for (int d = 0; d < pos_dim; ++d) {
      const float diff = sub_rn(pi[d], pj[d]);
      d2 = add_rn(d2, mul_rn(diff, diff));
    }
    return d2 < r2;
  }
  float acc = 0.f;
  for (int d = 0; d < pos_dim; ++d) {
    const float diff = sub_rn(pi[d], pj[d]);
    acc = fma_rn(diff, diff, acc);
  }
  return sqrt_rn(acc) < r;
}

// g(s) of the edge features: edge_attr = g(s_src) - g(s_dst)
template <int ENV>
GCBF_GHD void edge_feat(const float* s, float* f) {
  if (ENV == GCBF_ENV_DUBINS_CAR) {
    // reference gcbf/env/dubins_car.py:724-728: [x, y, theta, v*cos(theta), v*sin(theta)]
    f[0] = s[0]; f[1] = s[1]; f[2] = s[2];
    f[3] = mul_rn(s[3], cosf(s[2]));
    f[4] = mul_rn(s[3], sinf(s[2]));
  } else if (ENV == GCBF_ENV_SIMPLE_CAR) {
    f[0] = s[0]; f[1] = s[1]; f[2] = s[2]; f[3] = s[3];
  } else {
    f[0] = s[0]; f[1] = s[1]; f[2] = s[2]; f[3] = s[3]; f[4] = s[4]; f[5] = s[5];
  }
}

}  // namespace graph
}  // namespace gcbf
