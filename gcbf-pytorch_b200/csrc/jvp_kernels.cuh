// Kernels of the analytic h_dot pass (SURVEY 8f-3): grid-stride loops around the per-element functions of jvp_core.h.  Kept in a header
// of their own, free of CUDA runtime includes, so that tests/host_driver/jvp_grid.cpp can compile the SAME kernel bodies for the host
// on an emulated grid (tests/host_driver/cuda_emu.h) -- the build container has no GPU.
#pragma once
#include "gcbf_b200.h"
#include "jvp_core.h"

namespace gcbf {

__global__ void state_dot_kernel(int env, int num_graphs, int N, int n, const float* __restrict__ states, int ld,
                                 const float* __restrict__ action, const float* __restrict__ u_ref, const float* __restrict__ goal, int ld_goal,
                                 int goal_gstride, float action_lim, float speed_limit, float dist2goal, int freeze,
                                 float* __restrict__ out, int ld_out) {
  const int sd = env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4, ad = env == GCBF_ENV_SIMPLE_DRONE ? 3 : 2, pd = env == GCBF_ENV_SIMPLE_DRONE ? 3 : 2;
  const int64_t total = (int64_t)num_graphs * N;
  for (int64_t node = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; node < total; node += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(node / N), l = (int)(node % N);
    const bool is_agent = l < n;
    float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, uc[3] = {0.f, 0.f, 0.f}, xd[6];
    for (int k = 0; k < sd; ++k) s[k] = states[node * ld + k];
    bool frozen = false, pass[3];
    if (is_agent) {
      const int64_t a = (int64_t)g * n + l;
      const float* goal_row = (freeze && env != GCBF_ENV_SIMPLE_CAR) ? goal + ((int64_t)g * goal_gstride + l) * ld_goal : nullptr;
      frozen = jvp::agent_inputs(ad, pd, s, action + a * ad, u_ref + a * ad, goal_row, action_lim, dist2goal, uc, pass);
    }
    jvp::state_dot(env, is_agent, s, uc, speed_limit, frozen, xd);
    for (int k = 0; k < sd; ++k) out[node * ld_out + k] = xd[k];
  }
}

__global__ void edge_attr_tangent_kernel(int env, const float* __restrict__ states, int ld, const float* __restrict__ sdot, int ld_sd,
                                         const int64_t* __restrict__ ei, int64_t E, float* __restrict__ out) {
  const int sd = env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4, ed = env == GCBF_ENV_SIMPLE_CAR ? 4 : (env == GCBF_ENV_DUBINS_CAR ? 5 : 6);
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < E; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t j = ei[e], i = ei[E + e];                // source j, target i: edge_attr = g(s_j) - g(s_i)
    float sj[6], dj[6], si[6], di[6], gj[6], gi[6];
    for (int k = 0; k < sd; ++k) {
      sj[k] = states[j * ld + k]; dj[k] = sdot[j * ld_sd + k];
      si[k] = states[i * ld + k]; di[k] = sdot[i * ld_sd + k];
    }
    jvp::feature_dot(env, sj, dj, gj);
    jvp::feature_dot(env, si, di, gi);
    for (int k = 0; k < ed; ++k) out[e * ed + k] = gj[k] - gi[k];
  }
}

// thread per (target, channel), channel fastest
__global__ void attn_tangent_kernel(const float* __restrict__ msg, int ld_msg, const float* __restrict__ t_msg, int ld_tmsg,
                                    const float* __restrict__ att, const float* __restrict__ t_gate, const int32_t* __restrict__ rowptr,
                                    int num_nodes, int C, float* __restrict__ out, int ld_out) {
  const int64_t total = (int64_t)num_nodes * C;
  for (int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; idx < total; idx += (int64_t)gridDim.x * blockDim.x) {
    const int i = (int)(idx / C), c = (int)(idx % C);
    out[(int64_t)i * ld_out + c] = jvp::attn_tangent_cell(msg, ld_msg, t_msg, ld_tmsg, att, t_gate, rowptr[i], rowptr[i + 1], c);
  }
}

// ---- backward of the tangent pass ---------------------------------------------------------------------------------------------------

// dL/d action from dL/d x_dot (d_sdot [num_graphs * N, >= state_dim]): the VJP of state_dot_kernel through the clamp and the reach-freeze;
// agents only (obstacle rows have no action).  accumulate: add onto d_action instead of overwriting it.
__global__ void state_dot_bwd_kernel(int env, int num_graphs, int N, int n, const float* __restrict__ states, int ld,
                                     const float* __restrict__ action, const float* __restrict__ u_ref, const float* __restrict__ goal, int ld_goal,
                                     int goal_gstride, float action_lim, float dist2goal, int freeze, const float* __restrict__ d_sdot, int ld_dsd,
                                     float* __restrict__ d_action, int accumulate) {
  const int sd = env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4, ad = env == GCBF_ENV_SIMPLE_DRONE ? 3 : 2, pd = env == GCBF_ENV_SIMPLE_DRONE ? 3 : 2;
  const int64_t total = (int64_t)num_graphs * n;
  for (int64_t a = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; a < total; a += (int64_t)gridDim.x * blockDim.x) {
    const int g = (int)(a / n), l = (int)(a % n);
    const int64_t node = (int64_t)g * N + l;
    float s[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, uc[3], dx[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, du[3];
    bool pass[3];
    for (int k = 0; k < sd; ++k) { s[k] = states[node * ld + k]; dx[k] = d_sdot[node * ld_dsd + k]; }
    const float* goal_row = (freeze && env != GCBF_ENV_SIMPLE_CAR) ? goal + ((int64_t)g * goal_gstride + l) * ld_goal : nullptr;
    const bool frozen = jvp::agent_inputs(ad, pd, s, action + a * ad, u_ref + a * ad, goal_row, action_lim, dist2goal, uc, pass);
    jvp::state_dot_vjp(env, true, frozen, dx, du);
    for (int k = 0; k < ad; ++k) {
      const float v = pass[k] ? du[k] : 0.f;
      d_action[a * ad + k] = accumulate ? d_action[a * ad + k] + v : v;
    }
  }
}

// element-wise: (dZ, dTZ) of an activation and its tangent (jvp::act_tangent_vjp); TZ (the pre-activation tangent) is read for tanh only
__global__ void act_tangent_bwd_kernel(const float* __restrict__ dY, const float* __restrict__ dTY, const float* __restrict__ Y,
                                       const float* __restrict__ TZ, int64_t count, int act, float* __restrict__ dZ, float* __restrict__ dTZ) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x) {
    float dz, dtz;
    jvp::act_tangent_vjp(act, dY[i], dTY[i], Y[i], act == 2 ? TZ[i] : 0.f, &dz, &dtz);
    dZ[i] = dz;
    dTZ[i] = dtz;
  }
}

#if defined(__CUDACC__)
// VJP of attn_tangent_kernel (jvp::attn_tangent_vjp_*): one warp per target over its CSR range, lanes stride the channels, the edge dot
// products p_e = m_e . tau and q_e = m_dot_e . tau are xor-shuffle sums (the same on every lane, fixed order: deterministic, no atomics).
// Pass 1 forms the target's sums P, Q, GP; pass 2 recomputes p_e, q_e and writes.  Warp intrinsics: not part of the host emulation.
__global__ void __launch_bounds__(256) attn_tangent_bwd_kernel(
    const float* __restrict__ msg, int ld_msg, const float* __restrict__ t_msg, int ld_tmsg, const float* __restrict__ att,
    const float* __restrict__ t_gate, const int32_t* __restrict__ rowptr, int num_nodes, int C, const float* __restrict__ d_t_aggr, int ld_dta,
    float* __restrict__ d_t_msg, int ld_dtm, float* __restrict__ d_t_gate, float* __restrict__ d_msg, int ld_dmsg, float* __restrict__ d_gate,
    int accumulate) {
  const int lane = threadIdx.x & 31;
  const int64_t warps = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < num_nodes; i += warps) {
    const int beg = rowptr[i], end = rowptr[i + 1];
    if (end <= beg) continue;
    const float* tau = d_t_aggr + i * ld_dta;
    float gbar = 0.f;
    for (int e = beg; e < end; ++e) gbar = fmaf(att[e], t_gate[e], gbar);
    float P = 0.f, Q = 0.f, GP = 0.f;
    for (int e = beg; e < end; ++e) {
      float p = 0.f, q = 0.f;
      for (int c = lane; c < C; c += 32) {
        p = fmaf(msg[(int64_t)e * ld_msg + c], tau[c], p);
        q = fmaf(t_msg[(int64_t)e * ld_tmsg + c], tau[c], q);
      }
      for (int o = 16; o > 0; o >>= 1) { p += __shfl_xor_sync(0xffffffffu, p, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
      const float a = att[e];
      P = fmaf(a, p, P);
      Q = fmaf(a, q, Q);
      GP = fmaf(a * t_gate[e], p, GP);
    }
    const float R = jvp::attn_tangent_vjp_R(Q, GP, gbar, P);
    for (int e = beg; e < end; ++e) {
      const float a = att[e], gd = t_gate[e];
      float p = 0.f, q = 0.f;
      for (int c = lane; c < C; c += 32) {
        const float tc = tau[c];
        p = fmaf(msg[(int64_t)e * ld_msg + c], tc, p);
        q = fmaf(t_msg[(int64_t)e * ld_tmsg + c], tc, q);
        float dtm, dm;
        jvp::attn_tangent_vjp_cell(a, gd, gbar, tc, &dtm, &dm);
        d_t_msg[(int64_t)e * ld_dtm + c] = dtm;
        float* dmp = d_msg + (int64_t)e * ld_dmsg + c;
        *dmp = accumulate ? *dmp + dm : dm;
      }
      for (int o = 16; o > 0; o >>= 1) { p += __shfl_xor_sync(0xffffffffu, p, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
      if (lane == 0) {
        float dtg, dg;
        jvp::attn_tangent_vjp_edge(a, gd, gbar, p, q, P, R, &dtg, &dg);
        d_t_gate[e] = dtg;
        d_gate[e] = accumulate ? d_gate[e] + dg : dg;
      }
    }
  }
}
#endif

}  // namespace gcbf
