// Kernel bodies of the two-hop probe-graph builder of the CBF-condition field (condition.cu).  One warp per probe, grid-stride over
// probes, in the scheme of the level-set field's probe graphs (field_kernels.cuh): the lanes sweep candidate sources in ascending order
// and a ballot + popc ranks the hits, so every target's edges come out in the copy's order without a sort and without atomics.  The
// agent sources of a' are then visited one by one, in order, and the whole warp sweeps each one's in-edges in G'.  Counting and
// filling are two passes around an exclusive scan of the per-probe counts.
//
// Host build (tests/host_driver/condition_grid.cpp with cuda_emu.h): a "warp" is one thread there, as in field_kernels.cuh.
#pragma once
#include "condition_core.h"

namespace gcbf {
namespace cond {

// warp helpers as in field_kernels.cuh (whose kernels are not included here: one definition per library)
#if defined(__CUDA_ARCH__)
constexpr int kProbeWarp = 32;
__device__ __forceinline__ unsigned probe_ballot(bool p) { return __ballot_sync(0xffffffffu, p); }
__device__ __forceinline__ int probe_popc(unsigned m) { return __popc(m); }
__device__ __forceinline__ int cond_lowbit(unsigned m) { return __ffs((int)m) - 1; }
#else
constexpr int kProbeWarp = 1;
__device__ inline unsigned probe_ballot(bool p) { return p ? 1u : 0u; }
__device__ inline int probe_popc(unsigned m) { return m & 1u; }
__device__ inline int cond_lowbit(unsigned m) { return __builtin_ctz(m); }
#endif

// what the probes are made of: the field's ProbeGrid (field_kernels.cuh) plus the agent count
struct ProbeGrid {
  const float* states; int ld; int state_dim;
  int num_graphs, N;
  const int32_t* agents; int A;
  int x_dim, y_dim; const float* xs; const float* ys; int nx, ny;
  int pos_dim; float r; int metric;
  int relink;
  const int32_t* rowptr; const int64_t* edge_index;
};

// s'_t and the node it replaces
__device__ inline int64_t probe_load(const ProbeGrid& g, int64_t t, field::ProbeIdx* pi, float* sp) {
  const field::ProbeIdx p = field::probe_index(t, g.A, g.nx, g.ny);
  const int64_t node = p.b * g.N + g.agents[p.ai];
  field::probe_state(g.states + node * g.ld, g.state_dim, g.x_dim, g.xs[p.ix], g.y_dim, g.ys[p.iy], sp);
  *pi = p;
  return node;
}

struct CondGrid {
  ProbeGrid p;                       // states, graph sizes, probed agents, grid, pair rule, fixed / relink
  int n;                             // agents per graph (agents first)
};

// candidate k of the in-edges of a' (fixed: position k of a's CSR range; relink: node k of graph b): is it a source, and which node
__device__ inline bool moved_source(const CondGrid& c, const float* sp, int a, int64_t base, int64_t beg, int k, float r2, int64_t* src) {
  const ProbeGrid& g = c.p;
  if (!g.relink) {
    *src = g.edge_index[beg + k];
    return true;
  }
  *src = base + k;
  return k != a && graph::pair_hit(sp, g.states + (base + k) * g.ld, g.pos_dim, g.r, r2, g.metric);
}

// candidate k of the in-edges of j' (j = node jn): the given CSR range of j (fixed) or node k of graph b with a at s'_t (relink)
__device__ inline bool neighbour_source(const CondGrid& c, const float* sp, int64_t a_node, int64_t jn, int64_t base, int64_t beg, int k,
                                        float r2, int64_t* src) {
  const ProbeGrid& g = c.p;
  if (!g.relink) {
    *src = g.edge_index[beg + k];
    return true;
  }
  *src = base + k;
  return base + k != jn &&
         graph::pair_hit(g.states + jn * g.ld, cond_source_state(base + k, a_node, g.states, g.ld, sp), g.pos_dim, g.r, r2, g.metric);
}

// candidates of a target: its CSR degree (fixed) or the graph's node count (relink)
__device__ inline int candidates(const CondGrid& c, int64_t node) {
  return c.p.relink ? c.p.N : c.p.rowptr[node + 1] - c.p.rowptr[node];
}

// counts[t] = in-edges of a', counts[T + t] = j' rows, counts[2 T + t] = in-edges of all j' rows, t in [0, T)
__global__ void cond_count_kernel(CondGrid c, int64_t T, int32_t* __restrict__ counts) {
  const ProbeGrid& g = c.p;
  const int64_t gt = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = (int)(gt % kProbeWarp);
  const int64_t nw = (int64_t)gridDim.x * blockDim.x / kProbeWarp;
  const float r2 = graph::mul_rn(g.r, g.r);
  for (int64_t t = gt / kProbeWarp; t < T; t += nw) {
    field::ProbeIdx p;
    float sp[6];
    const int64_t node = probe_load(g, t, &p, sp);
    const int a = g.agents[p.ai];
    const int64_t base = p.b * g.N;
    const int64_t beg = g.relink ? 0 : g.rowptr[node];
    const int cand = candidates(c, node);
    int ea = 0, rows = 0, ej = 0;
    for (int k0 = 0; k0 < cand; k0 += kProbeWarp) {
      const int k = k0 + lane;
      int64_t src = 0;
      const bool hit = k < cand && moved_source(c, sp, a, base, beg, k, r2, &src);
      ea += probe_popc(probe_ballot(hit));
      unsigned ma = probe_ballot(hit && src - base < c.n);
      rows += probe_popc(ma);
      while (ma) {                                       // the agent sources, in order: their in-degree in G'
        const int kb = k0 + cond_lowbit(ma);
        ma &= ma - 1u;
        int64_t jn = 0;
        moved_source(c, sp, a, base, beg, kb, r2, &jn);
        const int64_t jbeg = g.relink ? 0 : g.rowptr[jn];
        const int jc = candidates(c, jn);
        for (int q0 = 0; q0 < jc; q0 += kProbeWarp) {
          const int q = q0 + lane;
          int64_t s2 = 0;
          ej += probe_popc(probe_ballot(q < jc && neighbour_source(c, sp, node, jn, base, jbeg, q, r2, &s2)));
        }
      }
    }
    if (lane == 0) {
      counts[t] = ea;
      counts[T + t] = rows;
      counts[2 * T + t] = ej;
    }
  }
}

// The rows and edges of probes [t0, t0 + Tc).  off[i], off[Tc + i], off[2 Tc + i] = where probe t0 + i's a' edges, j' rows and j'
// edges start (exclusive scans; the j' rows start at Tc, the j' edges after all a' edges: edges are target-sorted).  Writes, per row r
// (a' rows r = i): x_out[r] = x of the node, st_out[r] [state_dim] = its state in G', goal_out[r] [goal_dim] = its goal row, rows_out
// [r] = (kind, node id, probe id) if not null; edge_index [2, E_out] with target rows and source rows (cond_source_row); edge_attr
// [E_out, ED] = g(s_src) - g(s_tgt) in G'.
template <int ENV>
__global__ void cond_fill_kernel(CondGrid c, int64_t t0, int Tc, const int32_t* __restrict__ off, int64_t src_off,
                                 const float* __restrict__ x, int nd, const float* __restrict__ goal, int ld_goal, int goal_dim,
                                 int goal_gstride, float* __restrict__ x_out, float* __restrict__ st_out, float* __restrict__ goal_out,
                                 int64_t* __restrict__ rows_out, int64_t* __restrict__ ei_out, int64_t E_out, float* __restrict__ ea_out) {
  constexpr int ED = field::EnvDims<ENV>::ED;
  const ProbeGrid& g = c.p;
  const int sd = g.state_dim;
  const int64_t gt = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int lane = (int)(gt % kProbeWarp);
  const int64_t nw = (int64_t)gridDim.x * blockDim.x / kProbeWarp;
  const float r2 = graph::mul_rn(g.r, g.r);
  for (int64_t i = gt / kProbeWarp; i < Tc; i += nw) {
    field::ProbeIdx p;
    float sp[6], gp[6];
    const int64_t node = probe_load(g, t0 + i, &p, sp);
    graph::edge_feat<ENV>(sp, gp);
    const int a = g.agents[p.ai];
    const int64_t base = p.b * g.N;
    const int64_t beg = g.relink ? 0 : g.rowptr[node];
    const int cand = candidates(c, node);
    // the a' row
    const int64_t goal_b = p.b * goal_gstride;
    for (int k = lane; k < nd; k += kProbeWarp) x_out[i * nd + k] = x[node * nd + k];
    for (int k = lane; k < sd; k += kProbeWarp) st_out[i * sd + k] = sp[k];
    for (int k = lane; k < goal_dim; k += kProbeWarp) goal_out[i * goal_dim + k] = goal[(goal_b + a) * ld_goal + k];
    if (rows_out && lane == 0) { rows_out[i * 3] = kRowMoved; rows_out[i * 3 + 1] = node; rows_out[i * 3 + 2] = t0 + i; }
    int64_t out = off[i], jrow = off[Tc + i], jout = off[2 * Tc + i];
    for (int k0 = 0; k0 < cand; k0 += kProbeWarp) {
      const int k = k0 + lane;
      int64_t src = 0;
      const bool hit = k < cand && moved_source(c, sp, a, base, beg, k, r2, &src);
      const bool is_agent = hit && src - base < c.n;
      const unsigned m = probe_ballot(hit);
      unsigned ma = probe_ballot(is_agent);
      const unsigned below = (1u << lane) - 1u;
      if (hit) {                                         // the a' edge: an agent source is read from its j' row
        const int64_t pos = out + probe_popc(m & below);
        ei_out[pos] = cond_source_row(src, node, true, is_agent, i, jrow + probe_popc(ma & below), src_off);
        ei_out[E_out + pos] = i;
        field::probe_edge_attr<ENV>(g.states + src * g.ld, gp, ea_out + pos * ED);
      }
      out += probe_popc(m);
      while (ma) {                                       // the j' rows and their in-edges, in a'-edge order
        const int kb = k0 + cond_lowbit(ma);
        ma &= ma - 1u;
        int64_t jn = 0;
        moved_source(c, sp, a, base, beg, kb, r2, &jn);
        const float* sj = g.states + jn * g.ld;
        float gj[6];
        graph::edge_feat<ENV>(sj, gj);
        for (int q = lane; q < nd; q += kProbeWarp) x_out[jrow * nd + q] = x[jn * nd + q];
        for (int q = lane; q < sd; q += kProbeWarp) st_out[jrow * sd + q] = sj[q];
        for (int q = lane; q < goal_dim; q += kProbeWarp) goal_out[jrow * goal_dim + q] = goal[(goal_b + (jn - base)) * ld_goal + q];
        if (rows_out && lane == 0) { rows_out[jrow * 3] = kRowNeighbour; rows_out[jrow * 3 + 1] = jn; rows_out[jrow * 3 + 2] = t0 + i; }
        const int64_t jbeg = g.relink ? 0 : g.rowptr[jn];
        const int jc = candidates(c, jn);
        for (int q0 = 0; q0 < jc; q0 += kProbeWarp) {
          const int q = q0 + lane;
          int64_t s2 = 0;
          const bool h2 = q < jc && neighbour_source(c, sp, node, jn, base, jbeg, q, r2, &s2);
          const unsigned m2 = probe_ballot(h2);
          if (h2) {
            const int64_t pos = jout + probe_popc(m2 & below);
            ei_out[pos] = cond_source_row(s2, node, false, false, i, 0, src_off);
            ei_out[E_out + pos] = jrow;
            field::probe_edge_attr<ENV>(cond_source_state(s2, node, g.states, g.ld, sp), gj, ea_out + pos * ED);
          }
          jout += probe_popc(m2);
        }
        ++jrow;
      }
    }
  }
}

}  // namespace cond
}  // namespace gcbf
