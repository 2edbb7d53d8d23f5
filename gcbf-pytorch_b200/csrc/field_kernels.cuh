// Kernel bodies of the probe-graph builder (field.cu).  One warp per probe, grid-stride over probes; the 32 lanes of a warp sweep a
// probe's sources in ascending order and a ballot + popc ranks the hits, so every probe's edges come out in ascending source order
// without a sort and without atomics (the scheme of the K1 radius-graph kernel, graph.cu).  Counting and filling are two passes around
// an exclusive scan of the per-probe counts.
//
// Host build (tests/host_driver/field_grid.cpp with cuda_emu.h): a "warp" is one thread there (no warp intrinsics on the emulated
// grid), so the same bodies run with a warp width of 1.
#pragma once
#include "field_core.h"

namespace gcbf {
namespace field {

#if defined(__CUDA_ARCH__)
constexpr int kProbeWarp = 32;
__device__ __forceinline__ unsigned probe_ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
__device__ __forceinline__ int probe_popc(unsigned m) { return __popc(m); }
#else
constexpr int kProbeWarp = 1;
__device__ inline unsigned probe_ballot(bool p) { return p ? 1u : 0u; }
__device__ inline int probe_popc(unsigned m) { return m & 1u; }
#endif

// What the probes are made of.  Graph layout: num_graphs graphs of N nodes, agents first; states [num_graphs * N, ld].
struct ProbeGrid {
  const float* states; int ld; int state_dim;
  int num_graphs, N;
  const int32_t* agents; int A;          // probed agents (local ids, agents first in every graph)
  int x_dim, y_dim; const float* xs; const float* ys; int nx, ny;
  int pos_dim; float r; int metric;      // relink: the K1 pair rule
  int relink;                            // 0: the in-edges of the given graph (fixed), 1: every node j != a inside the radius of s'_t
  const int32_t* rowptr; const int64_t* edge_index;   // the given graph (fixed mode): CSR over all nodes, target-sorted [2, E]
};

// s'_t and the node it replaces
__device__ inline int64_t probe_load(const ProbeGrid& g, int64_t t, ProbeIdx* pi, float* sp) {
  const ProbeIdx p = probe_index(t, g.A, g.nx, g.ny);
  const int64_t node = p.b * g.N + g.agents[p.ai];
  probe_state(g.states + node * g.ld, g.state_dim, g.x_dim, g.xs[p.ix], g.y_dim, g.ys[p.iy], sp);
  *pi = p;
  return node;
}

// counts[t] = number of sources of probe t, t in [0, T)
__global__ void probe_count_kernel(ProbeGrid g, int64_t T, int32_t* __restrict__ counts) {
  const int64_t gt = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = (int)(gt % kProbeWarp);
  const int64_t nw = (int64_t)gridDim.x * blockDim.x / kProbeWarp;
  for (int64_t t = gt / kProbeWarp; t < T; t += nw) {
    ProbeIdx p;
    float sp[6];
    const int64_t node = probe_load(g, t, &p, sp);
    if (!g.relink) {
      if (lane == 0) counts[t] = g.rowptr[node + 1] - g.rowptr[node];
      continue;
    }
    const int a = g.agents[p.ai];
    const int64_t base = p.b * g.N;
    const float r2 = graph::mul_rn(g.r, g.r);
    int total = 0;
    for (int j0 = 0; j0 < g.N; j0 += kProbeWarp) {
      const int j = j0 + lane;
      bool hit = false;
      if (j < g.N && j != a) hit = graph::pair_hit(sp, g.states + (base + j) * g.ld, g.pos_dim, g.r, r2, g.metric);
      total += probe_popc(probe_ballot(hit));
    }
    if (lane == 0) counts[t] = total;
  }
}

// The edges of probes [t0, t0 + T): rowptr_local[i] (exclusive scan of their counts) is where probe t0 + i's edges start.  Writes
// edge_index [2, E_out] with source = src_off + original node id, target = tgt_off + i, edge_attr [E_out, ED] and, if x_out is not
// null, the probe's x row x_out[i * nd ..] = x of the probed agent.
template <int ENV>
__global__ void probe_fill_kernel(ProbeGrid g, int64_t t0, int T, const int32_t* __restrict__ rowptr_local, int64_t src_off, int64_t tgt_off,
                                  const float* __restrict__ x, int nd, float* __restrict__ x_out, int64_t* __restrict__ ei_out,
                                  int64_t E_out, float* __restrict__ ea_out) {
  constexpr int ED = EnvDims<ENV>::ED;
  const int64_t gt = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = (int)(gt % kProbeWarp);
  const int64_t nw = (int64_t)gridDim.x * blockDim.x / kProbeWarp;
  for (int64_t i = gt / kProbeWarp; i < T; i += nw) {
    ProbeIdx p;
    float sp[6], gp[6];
    const int64_t node = probe_load(g, t0 + i, &p, sp);
    graph::edge_feat<ENV>(sp, gp);
    const int64_t tgt = tgt_off + i;
    if (x_out)
      for (int c = lane; c < nd; c += kProbeWarp) x_out[i * nd + c] = x[node * nd + c];
    int64_t out = rowptr_local[i];
    if (!g.relink) {
      const int64_t beg = g.rowptr[node];
      const int deg = g.rowptr[node + 1] - g.rowptr[node];
      for (int k = lane; k < deg; k += kProbeWarp) {
        const int64_t src = g.edge_index[beg + k];
        ei_out[out + k] = src_off + src;
        ei_out[E_out + out + k] = tgt;
        probe_edge_attr<ENV>(g.states + src * g.ld, gp, ea_out + (out + k) * ED);
      }
      continue;
    }
    const int a = g.agents[p.ai];
    const int64_t base = p.b * g.N;
    const float r2 = graph::mul_rn(g.r, g.r);
    for (int j0 = 0; j0 < g.N; j0 += kProbeWarp) {
      const int j = j0 + lane;
      bool hit = false;
      if (j < g.N && j != a) hit = graph::pair_hit(sp, g.states + (base + j) * g.ld, g.pos_dim, g.r, r2, g.metric);
      const unsigned m = probe_ballot(hit);
      if (hit) {
        const int64_t pos = out + probe_popc(m & ((1u << lane) - 1u));
        ei_out[pos] = src_off + base + j;
        ei_out[E_out + pos] = tgt;
        probe_edge_attr<ENV>(g.states + (base + j) * g.ld, gp, ea_out + pos * ED);
      }
      out += probe_popc(m);
    }
  }
}

}  // namespace field
}  // namespace gcbf
