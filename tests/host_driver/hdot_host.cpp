// TEST INFRASTRUCTURE ONLY: host build of the per-element functions of the analytic-h_dot backward kernels
// (gcbf-pytorch_b200/csrc/jvp_core.h); each function is the serial form of the corresponding kernel in csrc/jvp_kernels.cuh.
// Compiled by tests/test_hdot_train_cpu.py with g++ -ffp-contract=off.
#include <math.h>
#include <stdint.h>
#include "jvp_core.h"

using namespace gcbf::jvp;

extern "C" {

void host_act_tangent_bwd(const float* dY, const float* dTY, const float* Y, const float* TZ, int64_t count, int act, float* dZ, float* dTZ) {
  for (int64_t i = 0; i < count; ++i) act_tangent_vjp(act, dY[i], dTY[i], Y[i], act == 2 ? TZ[i] : 0.f, dZ + i, dTZ + i);
}

void host_state_dot_bwd(int env, int num_graphs, int N, int n, const float* states, int ld, const float* action, const float* u_ref, const float* goal,
                        int ld_goal, int goal_gstride, float action_lim, float dist2goal, int freeze, const float* d_sdot, int ld_dsd, float* d_action,
                        int accumulate) {
  const int sd = env == 2 ? 6 : 4, ad = env == 2 ? 3 : 2, pd = env == 2 ? 3 : 2;
  for (int64_t a = 0; a < (int64_t)num_graphs * n; ++a) {
    const int g = (int)(a / n), l = (int)(a % n);
    const int64_t node = (int64_t)g * N + l;
    float s[6] = {0, 0, 0, 0, 0, 0}, uc[3], dx[6] = {0, 0, 0, 0, 0, 0}, du[3];
    bool pass[3];
    for (int k = 0; k < sd; ++k) { s[k] = states[node * ld + k]; dx[k] = d_sdot[node * ld_dsd + k]; }
    const float* goal_row = (freeze && env != 0) ? goal + ((int64_t)g * goal_gstride + l) * ld_goal : nullptr;
    const bool frozen = agent_inputs(ad, pd, s, action + a * ad, u_ref + a * ad, goal_row, action_lim, dist2goal, uc, pass);
    state_dot_vjp(env, true, frozen, dx, du);
    for (int k = 0; k < ad; ++k) {
      const float v = pass[k] ? du[k] : 0.f;
      d_action[a * ad + k] = accumulate ? d_action[a * ad + k] + v : v;
    }
  }
}

// serial form of attn_tangent_bwd_kernel (the kernel's sums are warp-shuffle trees; these are left to right)
void host_attn_aggr_tangent_bwd(const float* msg, int ld_msg, const float* t_msg, int ld_tmsg, const float* att, const float* t_gate,
                                const int32_t* rowptr, int num_nodes, int C, const float* d_t_aggr, int ld_dta, float* d_t_msg, int ld_dtm,
                                float* d_t_gate, float* d_msg, int ld_dmsg, float* d_gate, int accumulate) {
  for (int i = 0; i < num_nodes; ++i) {
    const int beg = rowptr[i], end = rowptr[i + 1];
    const float* tau = d_t_aggr + (int64_t)i * ld_dta;
    float gbar = 0.f, P = 0.f, Q = 0.f, GP = 0.f;
    for (int e = beg; e < end; ++e) gbar += att[e] * t_gate[e];
    for (int e = beg; e < end; ++e) {
      float p = 0.f, q = 0.f;
      for (int c = 0; c < C; ++c) { p += msg[(int64_t)e * ld_msg + c] * tau[c]; q += t_msg[(int64_t)e * ld_tmsg + c] * tau[c]; }
      P += att[e] * p; Q += att[e] * q; GP += att[e] * t_gate[e] * p;
    }
    const float R = attn_tangent_vjp_R(Q, GP, gbar, P);
    for (int e = beg; e < end; ++e) {
      float p = 0.f, q = 0.f;
      for (int c = 0; c < C; ++c) {
        p += msg[(int64_t)e * ld_msg + c] * tau[c];
        q += t_msg[(int64_t)e * ld_tmsg + c] * tau[c];
        float dtm, dm;
        attn_tangent_vjp_cell(att[e], t_gate[e], gbar, tau[c], &dtm, &dm);
        d_t_msg[(int64_t)e * ld_dtm + c] = dtm;
        float* dmp = d_msg + (int64_t)e * ld_dmsg + c;
        *dmp = accumulate ? *dmp + dm : dm;
      }
      float dtg, dg;
      attn_tangent_vjp_edge(att[e], t_gate[e], gbar, p, q, P, R, &dtg, &dg);
      d_t_gate[e] = dtg;
      d_gate[e] = accumulate ? d_gate[e] + dg : dg;
    }
  }
}

}  // extern "C"
