// Per-element arithmetic of the analytic h_dot pass (SURVEY 8f-3), written once for device and host (see macbf_core.h for the
// pattern: the kernels in jvp.cu are grid-stride loops around these functions, tests/host_driver/jvp_host.cpp compiles the same
// functions with g++ for the CPU test-suite).
//
// h_dot_i = sum_k (dh_i / ds_k) . f(s_k, u_k): the directional derivative of the CBF along the closed-loop vector field with the
// graph's edges held fixed -- what the reference approximates by the finite difference (h(x + dt f) - h(x)) / dt at
// gcbf/algo/gcbf.py:193-207.  It is a forward-mode (tangent) pass through forward_graph's pieces:
//   state_dot      f(x, clamp(u + u_ref(x)))          simple_car.py:78-89, dubins_car.py:110-132, simple_drone.py:103-120
//   edge tangent   d/dt [g(s_j) - g(s_i)]             simple_car.py:246-247, dubins_car.py:724-728, simple_drone.py:313-314
//   attention      d/dt sum_e softmax(gate)_e m_e     gcbf/nn/gnn.py:17-19 (AttentionalAggregation)
// and the linear layers / activations of the MLPs, which reuse the forward GEMM kernels and gcbf_act_bwd on the tangent.
#pragma once
#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define GCBF_JHD __host__ __device__ __forceinline__
#else
#define GCBF_JHD inline
#endif

namespace gcbf {
namespace jvp {

// IEEE round-to-nearest arithmetic that the device compiler may not contract or approximate (the host build uses -ffp-contract=off)
#if defined(__CUDA_ARCH__)
GCBF_JHD float add_rn(float a, float b) { return __fadd_rn(a, b); }
GCBF_JHD float sub_rn(float a, float b) { return __fsub_rn(a, b); }
GCBF_JHD float fma_rn(float a, float b, float c) { return __fmaf_rn(a, b, c); }
GCBF_JHD float sqrt_rn(float a) { return __fsqrt_rn(a); }
#else
GCBF_JHD float add_rn(float a, float b) { return a + b; }
GCBF_JHD float sub_rn(float a, float b) { return a - b; }
GCBF_JHD float fma_rn(float a, float b, float c) { return fmaf(a, b, c); }
GCBF_JHD float sqrt_rn(float a) { return sqrtf(a); }
#endif

// The per-agent inputs of the closed-loop vector field: uc = clamp(action + u_ref, -lim, lim), pass[k] = the clamp lets the gradient
// through (torch.clamp: -lim <= raw <= lim), and the return value: the single-graph reach-freeze (|pos - goal| < dist2goal; goal_row ==
// nullptr: no freeze).  Shared by the state derivative and its VJP.
GCBF_JHD bool agent_inputs(int ad, int pd, const float* s, const float* action, const float* u_ref, const float* goal_row, float action_lim,
                           float dist2goal, float* uc, bool* pass) {
  for (int k = 0; k < ad; ++k) {
    const float raw = add_rn(action[k], u_ref[k]);
    uc[k] = fminf(fmaxf(raw, -action_lim), action_lim);
    pass[k] = raw >= -action_lim && raw <= action_lim;
  }
  if (goal_row == nullptr) return false;
  float acc = 0.f;
  for (int k = 0; k < pd; ++k) {
    const float d = sub_rn(s[k], goal_row[k]);
    acc = fma_rn(d, d, acc);
  }
  return sqrt_rn(acc) < dist2goal;
}

// x_dot of one node.  s: state row; uc: the node's TOTAL clamped action (agents only; ignored for obstacles); frozen: the
// single-graph reach-freeze of dynamics() (dubins_car.py:126-130, simple_drone.py:113-117).  env: 0 SimpleCar, 1 DubinsCar, 2 SimpleDrone.
GCBF_JHD void state_dot(int env, bool is_agent, const float* s, const float* uc, float speed_limit, bool frozen, float* xdot) {
  for (int k = 0; k < 6; ++k) xdot[k] = 0.f;
  if (env == 0) {
    xdot[0] = s[2]; xdot[1] = s[3]; xdot[2] = uc[0]; xdot[3] = uc[1];
  } else if (env == 1) {                               // obstacles move too (their action is zero)
    const float vc = fminf(s[3], speed_limit);
    xdot[0] = vc * cosf(s[2]);
    xdot[1] = vc * sinf(s[2]);
    if (is_agent) { xdot[2] = uc[0] * 10.f; xdot[3] = uc[1]; }
  } else if (is_agent) {                                // drone obstacles are static
    xdot[0] = s[3]; xdot[1] = s[4]; xdot[2] = s[5];
    xdot[3] = -1.1f * s[3] + 1.1f * uc[0];
    xdot[4] = -1.1f * s[4] + 1.1f * uc[1];
    xdot[5] = -6.f * s[5] + 6.f * uc[2];
  }
  if (frozen)
    for (int k = 0; k < 6; ++k) xdot[k] = 0.f;
}

// VJP of state_dot with respect to the clamped action: d_uc = (d x_dot / d uc)^T d_xdot (zero for obstacles and frozen agents; the state
// derivative is linear in uc, so this is exact).
GCBF_JHD void state_dot_vjp(int env, bool is_agent, bool frozen, const float* d_xdot, float* d_uc) {
  d_uc[0] = d_uc[1] = d_uc[2] = 0.f;
  if (!is_agent || frozen) return;
  if (env == 0) {
    d_uc[0] = d_xdot[2]; d_uc[1] = d_xdot[3];
  } else if (env == 1) {
    d_uc[0] = d_xdot[2] * 10.f; d_uc[1] = d_xdot[3];
  } else {
    d_uc[0] = 1.1f * d_xdot[3]; d_uc[1] = 1.1f * d_xdot[4]; d_uc[2] = 6.f * d_xdot[5];
  }
}

// d/dt g(s) given s and s_dot.  g = identity (SimpleCar: 4, SimpleDrone: 6); DubinsCar g = [x, y, theta, v cos theta, v sin theta]
GCBF_JHD void feature_dot(int env, const float* s, const float* sd, float* gd) {
  if (env == 1) {
    const float c = cosf(s[2]), sn = sinf(s[2]);
    gd[0] = sd[0]; gd[1] = sd[1]; gd[2] = sd[2];
    gd[3] = sd[3] * c - s[3] * sn * sd[2];
    gd[4] = sd[3] * sn + s[3] * c * sd[2];
  } else {
    const int d = env == 0 ? 4 : 6;
    for (int k = 0; k < d; ++k) gd[k] = sd[k];
  }
}

// tangent of the attention aggregation of ONE (target, channel) cell over the target's CSR range [beg, end):
//   aggr = sum_e a_e m_e,  a = softmax(gate)  =>  d aggr = sum_e a_e (dm_e + m_e (dg_e - sum_k a_k dg_k))
GCBF_JHD float attn_tangent_cell(const float* msg, int ld_msg, const float* t_msg, int ld_tmsg, const float* att, const float* t_gate,
                                 int beg, int end, int c) {
  float mean_tg = 0.f;
  for (int e = beg; e < end; ++e) mean_tg += att[e] * t_gate[e];
  float acc = 0.f;
  for (int e = beg; e < end; ++e)
    acc += att[e] * (t_msg[(int64_t)e * ld_tmsg + c] + msg[(int64_t)e * ld_msg + c] * (t_gate[e] - mean_tg));
  return acc;
}

// ---- backward of the tangent pass (the analytic-h_dot training loss) --------------------------------------------------------------------
// Activation y = act(z) with tangent y_dot = act'(z) z_dot; given dY = dL/dy and dTY = dL/dy_dot, the gradients of the pre-activation and of
// its tangent.  ReLU: no second-order term (almost everywhere).  tanh: y_dot = (1 - y^2) z_dot, so dL/dz also carries
// d(1 - y^2)/dz z_dot dTY = -2 y (1 - y^2) z_dot dTY.  act 0 (none): identity.
GCBF_JHD void act_tangent_vjp(int act, float dy, float dty, float y, float tz, float* dz, float* dtz) {
  if (act == 1) {
    const bool on = y > 0.f;
    *dz = on ? dy : 0.f;
    *dtz = on ? dty : 0.f;
  } else if (act == 2) {
    const float s = 1.f - y * y;
    *dtz = s * dty;
    *dz = s * (dy - 2.f * y * tz * dty);
  } else {
    *dz = dy;
    *dtz = dty;
  }
}

// Attention tangent t_i = sum_e a_e (m_dot_e + m_e (g_dot_e - gbar_i)), gbar_i = sum_k a_k g_dot_k, a = softmax(g) over the target's
// in-edges.  With tau = dL/dt_i, p_e = m_e . tau, q_e = m_dot_e . tau, P = sum_k a_k p_k and R = sum_k a_k r_k (r_e below):
//   dL/dm_dot_e = a_e tau                      dL/dg_dot_e = a_e (p_e - P)
//   dL/dm_e    += a_e (g_dot_e - gbar) tau      dL/dg_e    += a_e (r_e - R),  r_e = q_e + g_dot_e (p_e - P) - gbar p_e
// (the last two are the second-order terms added onto the primal aggregation's gradients).  Per channel of one edge:
GCBF_JHD void attn_tangent_vjp_cell(float a, float gdot, float gbar, float tau, float* d_tmsg, float* d_msg_add) {
  *d_tmsg = a * tau;
  *d_msg_add = a * (gdot - gbar) * tau;
}

// per edge, given its dot products p, q and the target's sums P, R:
GCBF_JHD void attn_tangent_vjp_edge(float a, float gdot, float gbar, float p, float q, float P, float R, float* d_tgate, float* d_gate_add) {
  *d_tgate = a * (p - P);
  const float r = q + gdot * (p - P) - gbar * p;
  *d_gate_add = a * (r - R);
}

// R from the target's sums: sum_k a_k r_k = Q + GP - 2 gbar P with Q = sum_k a_k q_k, GP = sum_k a_k g_dot_k p_k
GCBF_JHD float attn_tangent_vjp_R(float Q, float GP, float gbar, float P) { return Q + GP - 2.f * gbar * P; }

}  // namespace jvp
}  // namespace gcbf
