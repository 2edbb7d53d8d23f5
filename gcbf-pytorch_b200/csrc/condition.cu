// CBF-condition field: the two-hop probe graphs of gcbf_cbf_condition_probe_count / _fill.  The kernels live in condition_kernels.cuh
// (shared with the host emulation of the CPU test-suite); this file holds the argument checks and launches.  The nets, the per-row
// closed loop and the tangent pass run over these graphs from Python (GCBF.cbf_condition_field), on the existing entry points.
#include "common.cuh"
#include "condition_kernels.cuh"

namespace gcbf {
namespace cond {

static int check_grid(const gcbf_field_desc* d, const char* who) {
  GCBF_REQUIRE(d, "%s: null descriptor", who);
  const gcbf_env_cfg& e = d->env;
  const int sd = e.env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4;
  GCBF_REQUIRE(e.env >= GCBF_ENV_SIMPLE_CAR && e.env <= GCBF_ENV_SIMPLE_DRONE, "%s: unknown env %d", who, e.env);
  GCBF_REQUIRE(d->state_dim == sd && d->ld_state >= sd, "%s: state_dim %d / ld_state %d (env needs %d)", who, d->state_dim, d->ld_state, sd);
  GCBF_REQUIRE(e.num_graphs >= 1 && e.num_agents >= 1 && e.nodes_per_graph >= e.num_agents, "%s: bad graph sizes", who);
  GCBF_REQUIRE(d->num_probe_agents >= 1 && d->agents, "%s: no agents to probe", who);
  GCBF_REQUIRE(d->x_dim >= 0 && d->x_dim < sd && d->y_dim >= 0 && d->y_dim < sd && d->x_dim != d->y_dim,
               "%s: dims (%d, %d) must be distinct and in [0, %d)", who, d->x_dim, d->y_dim, sd);
  GCBF_REQUIRE(d->nx >= 1 && d->ny >= 1 && d->xs && d->ys, "%s: empty grid", who);
  GCBF_REQUIRE(d->states, "%s: null states", who);
  GCBF_REQUIRE(d->pos_dim >= 1 && d->pos_dim <= 3 && (d->graph_metric == 0 || d->graph_metric == 1), "%s: pos_dim / metric", who);
  GCBF_REQUIRE(d->relink || (d->rowptr && (d->num_edges == 0 || d->edge_index)), "%s: fixed mode needs the graph's edges", who);
  const int64_t T = (int64_t)e.num_graphs * d->num_probe_agents * d->nx * d->ny;
  GCBF_REQUIRE(T < (1ll << 31) && (int64_t)e.num_graphs * e.nodes_per_graph < (1ll << 31), "%s: too many probes (%lld)", who, (long long)T);
  return 0;
}

static CondGrid cond_grid(const gcbf_field_desc& d) {
  CondGrid c;
  ProbeGrid& g = c.p;
  g.states = d.states; g.ld = d.ld_state; g.state_dim = d.state_dim;
  g.num_graphs = d.env.num_graphs; g.N = d.env.nodes_per_graph;
  g.agents = d.agents; g.A = d.num_probe_agents;
  g.x_dim = d.x_dim; g.y_dim = d.y_dim; g.xs = d.xs; g.ys = d.ys; g.nx = d.nx; g.ny = d.ny;
  g.pos_dim = d.pos_dim; g.r = d.comm_radius; g.metric = d.graph_metric; g.relink = d.relink ? 1 : 0;
  g.rowptr = d.rowptr; g.edge_index = d.edge_index;
  c.n = d.env.num_agents;
  return c;
}

static int probe_blocks(int64_t T) { return (int)imax64(1, imin64(ceil_div(T * 32, 256), 8 * 1024)); }

}  // namespace cond
}  // namespace gcbf

using namespace gcbf;
using namespace gcbf::cond;

extern "C" int gcbf_cbf_condition_probe_count(const gcbf_field_desc* d, int32_t* counts, void* stream) {
  if (int rc = check_grid(d, "gcbf_cbf_condition_probe_count")) return rc;
  GCBF_REQUIRE(counts, "gcbf_cbf_condition_probe_count: null counts");
  const int64_t T = (int64_t)d->env.num_graphs * d->num_probe_agents * d->nx * d->ny;
  cond_count_kernel<<<probe_blocks(T), 256, 0, as_stream(stream)>>>(cond_grid(*d), T, counts);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_cbf_condition_probe_fill(const gcbf_field_desc* d, const float* goal, int ld_goal, int goal_dim, int goal_per_graph,
                                             int64_t t0, int num_probes, const int32_t* offsets, int64_t src_off, float* x_out,
                                             float* states_out, float* goal_out, int64_t* rows_out, int64_t* edge_index, int64_t num_edges,
                                             float* edge_attr, void* stream) {
  const char* who = "gcbf_cbf_condition_probe_fill";
  if (int rc = check_grid(d, who)) return rc;
  const int64_t T = (int64_t)d->env.num_graphs * d->num_probe_agents * d->nx * d->ny;
  GCBF_REQUIRE(t0 >= 0 && num_probes >= 0 && t0 + num_probes <= T, "%s: probes [%lld, %lld) outside [0, %lld)", who, (long long)t0,
               (long long)(t0 + num_probes), (long long)T);
  GCBF_REQUIRE(num_edges >= 0 && num_edges < (1ll << 31) && src_off >= 0, "%s: num_edges %lld / src_off %lld", who, (long long)num_edges,
               (long long)src_off);
  GCBF_REQUIRE(goal_dim >= 0 && goal_dim <= 6 && ld_goal >= goal_dim && (goal_dim == 0 || goal), "%s: goal rows", who);
  if (num_probes == 0) return GCBF_OK;
  GCBF_REQUIRE(offsets && d->x && x_out && states_out && (goal_dim == 0 || goal_out) && (num_edges == 0 || (edge_index && edge_attr)),
               "%s: null pointer", who);
  const CondGrid c = cond_grid(*d);
  const int gs = goal_per_graph ? d->env.num_agents : 0;
  const int nd = d->cbf.node_dim;
  GCBF_REQUIRE(nd >= 1, "%s: d->cbf.node_dim must give the width of x", who);
  const int grid = probe_blocks(num_probes);
  cudaStream_t st = as_stream(stream);
  switch (d->env.env) {
    case GCBF_ENV_SIMPLE_CAR:
      cond_fill_kernel<GCBF_ENV_SIMPLE_CAR><<<grid, 256, 0, st>>>(c, t0, num_probes, offsets, src_off, d->x, nd, goal, ld_goal, goal_dim, gs,
                                                                   x_out, states_out, goal_out, rows_out, edge_index, num_edges, edge_attr);
      break;
    case GCBF_ENV_DUBINS_CAR:
      cond_fill_kernel<GCBF_ENV_DUBINS_CAR><<<grid, 256, 0, st>>>(c, t0, num_probes, offsets, src_off, d->x, nd, goal, ld_goal, goal_dim, gs,
                                                                   x_out, states_out, goal_out, rows_out, edge_index, num_edges, edge_attr);
      break;
    default:
      cond_fill_kernel<GCBF_ENV_SIMPLE_DRONE><<<grid, 256, 0, st>>>(c, t0, num_probes, offsets, src_off, d->x, nd, goal, ld_goal, goal_dim, gs,
                                                                     x_out, states_out, goal_out, rows_out, edge_index, num_edges, edge_attr);
      break;
  }
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}
