// CBF level-set field (gcbf_cbf_field): h of chosen agents over a grid of two state dimensions, the data of the reference's
// plot_cbf_contour (gcbf/trainer/utils.py:226-298).  The reference batches n_mesh^2 full copies of the graph and keeps one agent's row;
// h_a depends only on a's in-edges and x_a, so here every grid point of every probed agent becomes ONE target node ("probe") with only
// its own in-edges:
//   1. count   one warp per probe: its edge count (fixed: the agent's in-degree; relink: K1 hits of the moved state)  -> counts[T]
//   2. sync    counts -> host (the call's one host sync), split [0, T) into chunks of <= max_probes probes and <= max_edges edges
//   3. sigma   ONE spectral-norm power iteration; every chunk uses its 1/sigma (the reference's single cbf(plot_data) call)
//   4. chunk   exclusive scan of the chunk's counts, fill (x rows, edge_index, edge_attr = g(s_j) - g(s'_t)), then the CBF chain of
//              net.cu over the chunk's probes only.  Node layout of a chunk: x rows [0, P) are the probes (P = probes of the largest
//              chunk; a chunk uses [0, Tc)), rows [P, P + B * N) are the original nodes, copied once per call.  The net runs over
//              Tc nodes -- aggregation, gamma and head on the probes alone -- while the edges' sources index the rows behind them
//              (edge_input reads x[source] directly; nothing else in the forward reads a source id).
// gcbf_cbf_field_probe_count / _fill export steps 1 and 4's fill for inspection, with the probe ids as targets.
#include <vector>

#include "chain.h"
#include "field_kernels.cuh"

namespace gcbf {
namespace chain {

// everything but the net: what the probe graphs need
static int check_field_grid(const gcbf_field_desc* d) {
  GCBF_REQUIRE(d, "gcbf_cbf_field: null descriptor");
  const gcbf_env_cfg& e = d->env;
  const int sd = e.env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4;
  GCBF_REQUIRE(e.env >= GCBF_ENV_SIMPLE_CAR && e.env <= GCBF_ENV_SIMPLE_DRONE, "gcbf_cbf_field: unknown env %d", e.env);
  GCBF_REQUIRE(d->state_dim == sd && d->ld_state >= sd, "gcbf_cbf_field: state_dim %d / ld_state %d (env needs %d)", d->state_dim, d->ld_state, sd);
  GCBF_REQUIRE(e.num_graphs >= 1 && e.num_agents >= 1 && e.nodes_per_graph >= e.num_agents, "gcbf_cbf_field: bad graph sizes");
  GCBF_REQUIRE(d->num_probe_agents >= 1 && d->agents, "gcbf_cbf_field: no agents to probe");
  GCBF_REQUIRE(d->x_dim >= 0 && d->x_dim < sd && d->y_dim >= 0 && d->y_dim < sd && d->x_dim != d->y_dim,
               "gcbf_cbf_field: dims (%d, %d) must be distinct and in [0, %d)", d->x_dim, d->y_dim, sd);
  GCBF_REQUIRE(d->nx >= 1 && d->ny >= 1 && d->xs && d->ys, "gcbf_cbf_field: empty grid");
  GCBF_REQUIRE(d->states && d->x, "gcbf_cbf_field: null states / x");
  GCBF_REQUIRE(d->pos_dim >= 1 && d->pos_dim <= 3 && (d->graph_metric == 0 || d->graph_metric == 1), "gcbf_cbf_field: pos_dim / metric");
  GCBF_REQUIRE(d->relink || (d->rowptr && (d->num_edges == 0 || d->edge_index)), "gcbf_cbf_field: fixed mode needs the graph's edges");
  GCBF_REQUIRE(d->num_edges >= 0, "gcbf_cbf_field: num_edges < 0");
  GCBF_REQUIRE(d->max_probes >= 1 && d->max_edges >= 1 && d->max_edges < (1ll << 31), "gcbf_cbf_field: chunk bounds (%d probes, %lld edges)",
               d->max_probes, (long long)d->max_edges);
  const int64_t T = (int64_t)e.num_graphs * d->num_probe_agents * d->nx * d->ny;
  const int64_t Nt = (int64_t)e.num_graphs * e.nodes_per_graph;
  GCBF_REQUIRE(T < (1ll << 31) && Nt + imin64(T, d->max_probes) < (1ll << 31), "gcbf_cbf_field: too many probes (%lld)", (long long)T);
  return 0;
}

static int check_field(const gcbf_field_desc* d) {
  GCBF_REQUIRE(d, "gcbf_cbf_field: null descriptor");
  if (int rc = check_net(&d->cbf)) return rc;
  GCBF_REQUIRE(d->cbf.n_head > 0 && d->cbf.head[d->cbf.n_head - 1].N == 1 && d->cbf.head_extra_dim == 0,
               "gcbf_cbf_field: the net must end in a one-column head (the CBF)");
  return check_field_grid(d);
}

struct FieldPlan {
  int64_t T, Nt;
  int P;            // probes of the largest chunk
  int64_t Emax;     // probe edges of the largest chunk
};

static FieldPlan field_plan(const gcbf_field_desc& d) {
  FieldPlan p;
  p.T = (int64_t)d.env.num_graphs * d.num_probe_agents * d.nx * d.ny;
  p.Nt = (int64_t)d.env.num_graphs * d.env.nodes_per_graph;
  p.P = (int)imin64(p.T, d.max_probes);
  // a probe has at most N - 1 sources (relink: the other nodes of its graph; fixed: the in-edges of an agent of a graph without
  // duplicate edges), so a chunk of P probes never needs more than P (N - 1) edges: the workspace scales with the call
  p.Emax = imax64(1, imin64(d.max_edges, (int64_t)p.P * (d.env.nodes_per_graph - 1)));
  return p;
}

static field::ProbeGrid probe_grid(const gcbf_field_desc& d) {
  field::ProbeGrid g;
  g.states = d.states; g.ld = d.ld_state; g.state_dim = d.state_dim;
  g.num_graphs = d.env.num_graphs; g.N = d.env.nodes_per_graph;
  g.agents = d.agents; g.A = d.num_probe_agents;
  g.x_dim = d.x_dim; g.y_dim = d.y_dim; g.xs = d.xs; g.ys = d.ys; g.nx = d.nx; g.ny = d.ny;
  g.pos_dim = d.pos_dim; g.r = d.comm_radius; g.metric = d.graph_metric; g.relink = d.relink ? 1 : 0;
  g.rowptr = d.rowptr; g.edge_index = d.edge_index;
  return g;
}

static int probe_grid_blocks(int64_t T) { return (int)imax64(1, imin64(ceil_div(T * 32, 256), 8 * 1024)); }

static int launch_count(const field::ProbeGrid& g, int64_t T, int32_t* counts, cudaStream_t st) {
  if (T == 0) return 0;
  field::probe_count_kernel<<<probe_grid_blocks(T), 256, 0, st>>>(g, T, counts);
  GCBF_LAUNCH_OK();
  return 0;
}

static int launch_fill(const field::ProbeGrid& g, int env, int64_t t0, int T, const int32_t* rowptr_local, int64_t src_off, int64_t tgt_off,
                       const float* x, int nd, float* x_out, int64_t* ei, int64_t E, float* ea, cudaStream_t st) {
  if (T == 0) return 0;
  const int grid = probe_grid_blocks(T);
  switch (env) {
    case GCBF_ENV_SIMPLE_CAR:
      field::probe_fill_kernel<GCBF_ENV_SIMPLE_CAR><<<grid, 256, 0, st>>>(g, t0, T, rowptr_local, src_off, tgt_off, x, nd, x_out, ei, E, ea); break;
    case GCBF_ENV_DUBINS_CAR:
      field::probe_fill_kernel<GCBF_ENV_DUBINS_CAR><<<grid, 256, 0, st>>>(g, t0, T, rowptr_local, src_off, tgt_off, x, nd, x_out, ei, E, ea); break;
    default:
      field::probe_fill_kernel<GCBF_ENV_SIMPLE_DRONE><<<grid, 256, 0, st>>>(g, t0, T, rowptr_local, src_off, tgt_off, x, nd, x_out, ei, E, ea); break;
  }
  GCBF_LAUNCH_OK();
  return 0;
}

struct FieldBufs {
  int32_t* counts; float* x; int32_t* rowptr; int64_t* ei; float* ea;
  const float* isg[4 * GCBF_MAX_MLP_LAYERS];
};

// allocations that live for the whole call (the sigma snapshot among them), in the order of the real run
static int field_outer(Run& R, const gcbf_field_desc& d, const FieldPlan& p, const gcbf_linear_desc* const* all, int nall, FieldBufs* b) {
  const int nd = d.cbf.node_dim, ed = d.cbf.edge_dim;
  b->counts = (int32_t*)R.ws.alloc((size_t)p.T * 4);
  const float *us[4 * GCBF_MAX_MLP_LAYERS], *vs[4 * GCBF_MAX_MLP_LAYERS];
  if (int rc = sn_power_iter(R, all, nall, false, b->isg, us, vs)) return rc;
  b->x = (float*)R.ws.alloc((size_t)(p.P + p.Nt) * nd * 4);
  b->rowptr = (int32_t*)R.ws.alloc((size_t)(p.P + 1) * 4);
  b->ei = (int64_t*)R.ws.alloc((size_t)2 * p.Emax * 8);
  b->ea = (float*)R.ws.alloc((size_t)p.Emax * ed * 4);
  return 0;
}

static size_t field_bytes(const gcbf_field_desc& d) {
  const FieldPlan p = field_plan(d);
  const gcbf_linear_desc* all[4 * GCBF_MAX_MLP_LAYERS];
  const int nall = collect_layers(d.cbf, all);
  Run R(nullptr, 0, nullptr, true);
  FieldBufs b;
  if (field_outer(R, d, p, all, nall, &b)) return 0;
  const size_t chunk = net_fwd_bytes(d.cbf, p.Emax, p.P, p.P, false, false);
  if (!chunk) return 0;
  return R.ws.off + chunk;
}

static int field_run(const gcbf_field_desc& d, float* h, int64_t* info, void* workspace, size_t bytes, cudaStream_t st) {
  const FieldPlan p = field_plan(d);
  const gcbf_linear_desc* all[4 * GCBF_MAX_MLP_LAYERS];
  const int nall = collect_layers(d.cbf, all);
  const int nd = d.cbf.node_dim;
  Run R(workspace, bytes, st, false);
  FieldBufs b;
  const field::ProbeGrid g = probe_grid(d);

  // buffers of the whole call; launches the one power iteration (3.)
  if (int rc = field_outer(R, d, p, all, nall, &b)) return rc;
  if (d.cbf.refresh_weights) { if (int rc = refresh_weight_companions(R, all, nall)) return rc; }
  if (R.ws.overflow) { set_error("gcbf_cbf_field: workspace overflow"); return GCBF_E_WORKSPACE; }
  // 1. counts of every probe
  if (int rc = launch_count(g, p.T, b.counts, st)) return rc;
  R.launched(1);
  std::vector<int32_t> counts((size_t)p.T);
  GCBF_CUDA_OK(cudaMemcpyAsync(counts.data(), b.counts, (size_t)p.T * 4, cudaMemcpyDeviceToHost, st));
  GCBF_CUDA_OK(cudaMemcpyAsync(b.x + (size_t)p.P * nd, d.x, (size_t)p.Nt * nd * 4, cudaMemcpyDeviceToDevice, st));   // the sources' x
  GCBF_CUDA_OK(cudaStreamSynchronize(st));                                                                          // 2. the one host sync

  gcbf_net_desc net = d.cbf;
  net.refresh_weights = 0;                                  // refreshed above, once
  uint8_t* chunk_base = R.ws.base + R.ws.off;
  const size_t chunk_cap = R.ws.cap - R.ws.off;
  int64_t chunks = 0, edges = 0;
  for (int64_t t0 = 0; t0 < p.T;) {
    int64_t E = 0, t1 = t0;
    while (t1 < p.T && t1 - t0 < p.P && E + counts[t1] <= p.Emax) E += counts[t1++];
    if (t1 == t0) {
      set_error("gcbf_cbf_field: probe %lld has %d edges > max_edges %lld (duplicate edges in the given graph?)", (long long)t0, counts[t0],
                (long long)p.Emax);
      return GCBF_E_INVALID;
    }
    const int Tc = (int)(t1 - t0);
    if (net_fwd_bytes(net, E, Tc, Tc, false, false) > chunk_cap) { set_error("gcbf_cbf_field: workspace too small for a chunk"); return GCBF_E_WORKSPACE; }
    GCBF_CUDA_OK(cudaMemcpyAsync(b.rowptr, b.counts + t0, (size_t)Tc * 4, cudaMemcpyDeviceToDevice, st));
    GCBF_CUDA_OK(exclusive_scan_i32(b.rowptr, Tc, st));     // rowptr[i] = first edge of probe t0 + i, rowptr[Tc] = E
    if (int rc = launch_fill(g, d.env.env, t0, Tc, b.rowptr, p.P, 0, d.x, nd, b.x, b.ei, E, b.ea, st)) return rc;
    R.launched(2);
    Run C(chunk_base, chunk_cap, st, false);
    if (int rc = net_forward(C, net, b.x, b.ea, b.ei, b.rowptr, E, Tc, nullptr, Tc, nullptr, h + t0, 1, nullptr, b.isg)) return rc;
    if (int rc = C.finish(0, "gcbf_cbf_field")) return rc;
    ++chunks;
    edges += E;
    t0 = t1;
  }
  if (info) { info[0] = chunks; info[1] = edges; }
  return R.finish(0, "gcbf_cbf_field");
}

}  // namespace chain
}  // namespace gcbf

using namespace gcbf;
using namespace gcbf::chain;

extern "C" size_t gcbf_cbf_field_workspace_bytes(const gcbf_field_desc* d) {
  if (check_field(d)) return 0;
  const size_t b = field_bytes(*d);
  return b ? b + 1024 : 0;
}

extern "C" int gcbf_cbf_field(const gcbf_field_desc* d, float* h, int64_t* info, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_field(d)) return rc;
  GCBF_REQUIRE(h, "gcbf_cbf_field: null output");
  GCBF_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "gcbf_cbf_field: workspace must be 256-byte aligned");
  const size_t need = field_bytes(*d);
  if (!need) { set_error("gcbf_cbf_field: could not size the workspace"); return GCBF_E_INVALID; }
  if (need > workspace_bytes) { set_error("gcbf_cbf_field: workspace too small (%zu needed, %zu given)", need, workspace_bytes); return GCBF_E_WORKSPACE; }
  return field_run(*d, h, info, workspace, workspace_bytes, as_stream(stream));
}

extern "C" int gcbf_cbf_field_probe_count(const gcbf_field_desc* d, int32_t* rowptr, void* stream) {
  if (int rc = check_field_grid(d)) return rc;
  GCBF_REQUIRE(rowptr, "gcbf_cbf_field_probe_count: null rowptr");
  const int64_t T = field_plan(*d).T;
  cudaStream_t st = as_stream(stream);
  if (int rc = launch_count(probe_grid(*d), T, rowptr, st)) return rc;
  GCBF_CUDA_OK(exclusive_scan_i32(rowptr, (int)T, st));
  return GCBF_OK;
}

extern "C" int gcbf_cbf_field_probe_fill(const gcbf_field_desc* d, const int32_t* rowptr, int64_t* edge_index, int64_t num_edges, float* edge_attr,
                                         void* stream) {
  if (int rc = check_field_grid(d)) return rc;
  GCBF_REQUIRE(rowptr && (num_edges == 0 || (edge_index && edge_attr)) && num_edges >= 0, "gcbf_cbf_field_probe_fill: bad arguments");
  if (num_edges == 0) return GCBF_OK;
  const int64_t T = field_plan(*d).T;
  return launch_fill(probe_grid(*d), d->env.env, 0, (int)T, rowptr, 0, 0, nullptr, 0, nullptr, edge_index, num_edges, edge_attr, as_stream(stream));
}
