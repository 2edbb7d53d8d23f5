// TEST INFRASTRUCTURE ONLY: the two-hop probe-graph kernels of csrc/condition_kernels.cuh (count, fill) compiled as plain C++ and
// executed on an emulated 1-D grid (cuda_emu.h).  A "warp" is one thread there (condition_kernels.cuh builds with a warp width of 1 on
// the host), so this runs the kernels' probe / source loops and output placement, not the ballot ranks.
// Compiled by tests/test_cbf_condition_field_cpu.py with g++ -ffp-contract=off.
#include "cuda_emu.h"
#include "condition_kernels.cuh"

using namespace gcbf;

static cond::CondGrid make_grid(const float* states, int ld, int state_dim, int num_graphs, int N, int n, const int32_t* agents, int A,
                                int x_dim, int y_dim, const float* xs, const float* ys, int nx, int ny, int pos_dim, float r, int metric,
                                int relink, const int32_t* rowptr, const int64_t* edge_index) {
  cond::CondGrid c;
  cond::ProbeGrid& g = c.p;
  g.states = states; g.ld = ld; g.state_dim = state_dim; g.num_graphs = num_graphs; g.N = N; g.agents = agents; g.A = A;
  g.x_dim = x_dim; g.y_dim = y_dim; g.xs = xs; g.ys = ys; g.nx = nx; g.ny = ny; g.pos_dim = pos_dim; g.r = r; g.metric = metric;
  g.relink = relink; g.rowptr = rowptr; g.edge_index = edge_index;
  c.n = n;
  return c;
}

#define GRID_ARGS                                                                                                                      \
  const float *states, int ld, int state_dim, int num_graphs, int N, int n, const int32_t *agents, int A, int x_dim, int y_dim,       \
      const float *xs, const float *ys, int nx, int ny, int pos_dim, float r, int metric, int relink, const int32_t *rowptr,          \
      const int64_t *edge_index
#define GRID_PASS states, ld, state_dim, num_graphs, N, n, agents, A, x_dim, y_dim, xs, ys, nx, ny, pos_dim, r, metric, relink, rowptr, edge_index

extern "C" {

void grid_cond_count(int grid, int block, GRID_ARGS, int64_t T, int32_t* counts) {
  const cond::CondGrid c = make_grid(GRID_PASS);
  EMU_LAUNCH(grid, block, cond::cond_count_kernel, c, T, counts);
}

void grid_cond_fill(int grid, int block, int env, GRID_ARGS, int64_t t0, int Tc, const int32_t* off, int64_t src_off, const float* x, int nd,
                    const float* goal, int ld_goal, int goal_dim, int goal_gstride, float* x_out, float* st_out, float* goal_out,
                    int64_t* rows_out, int64_t* ei_out, int64_t E_out, float* ea_out) {
  const cond::CondGrid c = make_grid(GRID_PASS);
  switch (env) {
    case GCBF_ENV_SIMPLE_CAR:
      EMU_LAUNCH(grid, block, cond::cond_fill_kernel<GCBF_ENV_SIMPLE_CAR>, c, t0, Tc, off, src_off, x, nd, goal, ld_goal, goal_dim, goal_gstride,
                 x_out, st_out, goal_out, rows_out, ei_out, E_out, ea_out);
      break;
    case GCBF_ENV_DUBINS_CAR:
      EMU_LAUNCH(grid, block, cond::cond_fill_kernel<GCBF_ENV_DUBINS_CAR>, c, t0, Tc, off, src_off, x, nd, goal, ld_goal, goal_dim, goal_gstride,
                 x_out, st_out, goal_out, rows_out, ei_out, E_out, ea_out);
      break;
    default:
      EMU_LAUNCH(grid, block, cond::cond_fill_kernel<GCBF_ENV_SIMPLE_DRONE>, c, t0, Tc, off, src_off, x, nd, goal, ld_goal, goal_dim, goal_gstride,
                 x_out, st_out, goal_out, rows_out, ei_out, E_out, ea_out);
      break;
  }
}

}  // extern "C"
