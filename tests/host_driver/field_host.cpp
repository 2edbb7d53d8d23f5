// TEST INFRASTRUCTURE ONLY: the per-element functions of the CBF-field probe graphs (csrc/field_core.h, csrc/graph_core.h) built for
// the host.  Compiled by tests/test_cbf_field_cpu.py with g++ -ffp-contract=off.
#include "field_core.h"

using namespace gcbf;

extern "C" {

void host_probe_state(const float* s, int state_dim, int x_dim, float vx, int y_dim, float vy, float* out) {
  field::probe_state(s, state_dim, x_dim, vx, y_dim, vy, out);
}

int host_pair_hit(const float* pi, const float* pj, int pos_dim, float r, int metric) {
  return graph::pair_hit(pi, pj, pos_dim, r, graph::mul_rn(r, r), metric) ? 1 : 0;
}

// g(s_src) - g(s_probe)
void host_probe_edge_attr(int env, const float* s_src, const float* s_probe, float* out) {
  float gp[6];
  switch (env) {
    case GCBF_ENV_SIMPLE_CAR: graph::edge_feat<GCBF_ENV_SIMPLE_CAR>(s_probe, gp); field::probe_edge_attr<GCBF_ENV_SIMPLE_CAR>(s_src, gp, out); break;
    case GCBF_ENV_DUBINS_CAR: graph::edge_feat<GCBF_ENV_DUBINS_CAR>(s_probe, gp); field::probe_edge_attr<GCBF_ENV_DUBINS_CAR>(s_src, gp, out); break;
    default: graph::edge_feat<GCBF_ENV_SIMPLE_DRONE>(s_probe, gp); field::probe_edge_attr<GCBF_ENV_SIMPLE_DRONE>(s_src, gp, out); break;
  }
}

void host_probe_index(int64_t t, int num_probe_agents, int nx, int ny, int64_t* out) {
  const field::ProbeIdx p = field::probe_index(t, num_probe_agents, nx, ny);
  out[0] = p.b; out[1] = p.ai; out[2] = p.iy; out[3] = p.ix;
}

}  // extern "C"
