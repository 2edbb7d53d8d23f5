// TEST INFRASTRUCTURE ONLY: the probe-graph kernels of csrc/field_kernels.cuh (count, fill) compiled as plain C++ and executed on an
// emulated 1-D grid (cuda_emu.h).  The emulated grid has no warp intrinsics: a "warp" is one thread there (field_kernels.cuh builds
// with a warp width of 1 on the host), so this runs the kernels' probe / source loops and output placement, not the ballot ranks.
// Compiled by tests/test_cbf_field_cpu.py with g++ -ffp-contract=off.
#include "cuda_emu.h"
#include "field_kernels.cuh"

using namespace gcbf;

static field::ProbeGrid make_grid(const float* states, int ld, int state_dim, int num_graphs, int N, const int32_t* agents, int A, int x_dim,
                                  int y_dim, const float* xs, const float* ys, int nx, int ny, int pos_dim, float r, int metric, int relink,
                                  const int32_t* rowptr, const int64_t* edge_index) {
  field::ProbeGrid g;
  g.states = states; g.ld = ld; g.state_dim = state_dim; g.num_graphs = num_graphs; g.N = N; g.agents = agents; g.A = A;
  g.x_dim = x_dim; g.y_dim = y_dim; g.xs = xs; g.ys = ys; g.nx = nx; g.ny = ny; g.pos_dim = pos_dim; g.r = r; g.metric = metric;
  g.relink = relink; g.rowptr = rowptr; g.edge_index = edge_index;
  return g;
}

extern "C" {

void grid_probe_count(int grid, int block, const float* states, int ld, int state_dim, int num_graphs, int N, const int32_t* agents, int A,
                      int x_dim, int y_dim, const float* xs, const float* ys, int nx, int ny, int pos_dim, float r, int metric, int relink,
                      const int32_t* rowptr, const int64_t* edge_index, int64_t T, int32_t* counts) {
  const field::ProbeGrid g = make_grid(states, ld, state_dim, num_graphs, N, agents, A, x_dim, y_dim, xs, ys, nx, ny, pos_dim, r, metric,
                                       relink, rowptr, edge_index);
  EMU_LAUNCH(grid, block, field::probe_count_kernel, g, T, counts);
}

void grid_probe_fill(int grid, int block, int env, const float* states, int ld, int state_dim, int num_graphs, int N, const int32_t* agents,
                     int A, int x_dim, int y_dim, const float* xs, const float* ys, int nx, int ny, int pos_dim, float r, int metric, int relink,
                     const int32_t* rowptr, const int64_t* edge_index, int64_t t0, int T, const int32_t* rowptr_local, int64_t src_off,
                     int64_t tgt_off, const float* x, int nd, float* x_out, int64_t* ei_out, int64_t E_chunk, float* ea_out) {
  const field::ProbeGrid g = make_grid(states, ld, state_dim, num_graphs, N, agents, A, x_dim, y_dim, xs, ys, nx, ny, pos_dim, r, metric,
                                       relink, rowptr, edge_index);
  switch (env) {
    case GCBF_ENV_SIMPLE_CAR:
      EMU_LAUNCH(grid, block, field::probe_fill_kernel<GCBF_ENV_SIMPLE_CAR>, g, t0, T, rowptr_local, src_off, tgt_off, x, nd, x_out, ei_out, E_chunk, ea_out); break;
    case GCBF_ENV_DUBINS_CAR:
      EMU_LAUNCH(grid, block, field::probe_fill_kernel<GCBF_ENV_DUBINS_CAR>, g, t0, T, rowptr_local, src_off, tgt_off, x, nd, x_out, ei_out, E_chunk, ea_out); break;
    default:
      EMU_LAUNCH(grid, block, field::probe_fill_kernel<GCBF_ENV_SIMPLE_DRONE>, g, t0, T, rowptr_local, src_off, tgt_off, x, nd, x_out, ei_out, E_chunk, ea_out); break;
  }
}

}  // extern "C"
