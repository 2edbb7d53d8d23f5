// TEST INFRASTRUCTURE ONLY: the element-wise backward kernels of csrc/jvp_kernels.cuh (state_dot_bwd_kernel, act_tangent_bwd_kernel)
// compiled as plain C++ and executed on an emulated 1-D grid (cuda_emu.h).  The attention backward kernel uses warp shuffles and is not
// emulated.  Compiled by tests/test_hdot_train_cpu.py with g++ -ffp-contract=off.
#include "cuda_emu.h"
#include "jvp_kernels.cuh"

extern "C" {

void grid_state_dot_bwd(int grid, int block, int env, int num_graphs, int N, int n, const float* states, int ld, const float* action,
                        const float* u_ref, const float* goal, int ld_goal, int goal_gstride, float action_lim, float dist2goal, int freeze,
                        const float* d_sdot, int ld_dsd, float* d_action, int accumulate) {
  EMU_LAUNCH(grid, block, gcbf::state_dot_bwd_kernel, env, num_graphs, N, n, states, ld, action, u_ref, goal, ld_goal, goal_gstride, action_lim,
             dist2goal, freeze, d_sdot, ld_dsd, d_action, accumulate);
}

void grid_act_tangent_bwd(int grid, int block, const float* dY, const float* dTY, const float* Y, const float* TZ, int64_t count, int act,
                          float* dZ, float* dTZ) {
  EMU_LAUNCH(grid, block, gcbf::act_tangent_bwd_kernel, dY, dTY, Y, TZ, count, act, dZ, dTZ);
}

}  // extern "C"
