// Per-element arithmetic of the CBF level-set field (reference plot_cbf_contour, gcbf/trainer/utils.py:226-298), written once for device
// and host: field.cu's probe-graph kernels (field_kernels.cuh) are loops around these functions, tests/host_driver/field_host.cpp
// compiles them with g++ -ffp-contract=off for the CPU test-suite.
//
// A probe t = (graph b, agent slot ai, grid row iy, grid column ix), numbered in that nesting: t = ((b * A + ai) * ny + iy) * nx + ix.
// Its state s'_t is s_{b, agents[ai]} with state[x_dim] = xs[ix] and state[y_dim] = ys[iy] (the grid values are already fp32, as
// the reference's write into the fp32 state tensor rounds them, utils.py:266-267).  A probe edge j -> t carries g(s_j) - g(s'_t).
#pragma once
#include "graph_core.h"

namespace gcbf {
namespace field {

struct ProbeIdx {
  int64_t b;     // graph
  int ai;        // slot in the probed-agent list
  int iy, ix;    // grid row / column
};

GCBF_GHD ProbeIdx probe_index(int64_t t, int num_probe_agents, int nx, int ny) {
  ProbeIdx p;
  p.ix = (int)(t % nx);
  t /= nx;
  p.iy = (int)(t % ny);
  t /= ny;
  p.ai = (int)(t % num_probe_agents);
  p.b = t / num_probe_agents;
  return p;
}

// s' = s with s'[x_dim] = vx, s'[y_dim] = vy (state_dim <= 6)
GCBF_GHD void probe_state(const float* s, int state_dim, int x_dim, float vx, int y_dim, float vy, float* out) {
  for (int k = 0; k < state_dim; ++k) out[k] = s[k];
  out[x_dim] = vx;
  out[y_dim] = vy;
}

template <int ENV> struct EnvDims;
template <> struct EnvDims<GCBF_ENV_SIMPLE_CAR> { static constexpr int SD = 4, ED = 4; };
template <> struct EnvDims<GCBF_ENV_DUBINS_CAR> { static constexpr int SD = 4, ED = 5; };
template <> struct EnvDims<GCBF_ENV_SIMPLE_DRONE> { static constexpr int SD = 6, ED = 6; };

// edge feature of the probe edge j -> t given g(s'_t) (computed once per probe): g(s_j) - g(s'_t)
template <int ENV>
GCBF_GHD void probe_edge_attr(const float* s_src, const float* g_probe, float* out) {
  constexpr int ED = EnvDims<ENV>::ED;
  float f[ED];
  graph::edge_feat<ENV>(s_src, f);
  for (int k = 0; k < ED; ++k) out[k] = graph::sub_rn(f[k], g_probe[k]);
}

}  // namespace field
}  // namespace gcbf
