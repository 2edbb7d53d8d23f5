// Analytic h_dot (SURVEY 8f-3): the three kernels a tangent pass through forward_graph + CBFGNN needs beyond the forward GEMMs --
// closed-loop state derivative, edge-feature tangent, attention-aggregation tangent.  The kernels live in jvp_kernels.cuh (shared with the
// host emulation of the CPU test-suite); this file holds the C-ABI entry points that launch them.
#include "common.cuh"
#include "jvp_kernels.cuh"



using namespace gcbf;

extern "C" int gcbf_state_dot(const gcbf_env_cfg* cfg, const float* states, int ld_state, const float* action, const float* u_ref,
                              const float* goal, int ld_goal, int goal_per_graph, int freeze, float* state_dot, int ld_out, void* stream) {
  GCBF_REQUIRE(cfg != nullptr, "gcbf_state_dot: null cfg");
  GCBF_REQUIRE(cfg->env >= 0 && cfg->env <= 2, "gcbf_state_dot: unknown env %d", cfg->env);
  GCBF_REQUIRE(cfg->num_graphs >= 0 && cfg->num_agents >= 0 && cfg->nodes_per_graph >= cfg->num_agents, "gcbf_state_dot: bad sizes");
  const int sd = cfg->env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4, pd = cfg->env == GCBF_ENV_SIMPLE_DRONE ? 3 : 2;
  GCBF_REQUIRE(ld_state >= sd && ld_out >= sd, "gcbf_state_dot: leading dimensions");
  const int64_t nodes = (int64_t)cfg->num_graphs * cfg->nodes_per_graph;
  GCBF_REQUIRE(nodes < (1ll << 31), "gcbf_state_dot: too many nodes");
  if (nodes == 0) return GCBF_OK;
  GCBF_REQUIRE(states && state_dot && (cfg->num_agents == 0 || (action && u_ref)), "gcbf_state_dot: null pointer");
  GCBF_REQUIRE(!freeze || cfg->env == GCBF_ENV_SIMPLE_CAR || (goal && ld_goal >= pd), "gcbf_state_dot: the reach-freeze needs the goal positions");
  const float action_lim = cfg->env == GCBF_ENV_DUBINS_CAR ? 2.f : 10.f;       // simple_car.py:264-268, dubins_car.py:758-762, simple_drone.py:343-347
  const int grid = (int)imin64(ceil_div(nodes, 256), 8 * kNumSMs);
  state_dot_kernel<<<grid, 256, 0, as_stream(stream)>>>(cfg->env, cfg->num_graphs, cfg->nodes_per_graph, cfg->num_agents, states, ld_state, action,
                                                        u_ref, goal, ld_goal, goal_per_graph ? cfg->num_agents : 0, action_lim,
                                                        (float)cfg->speed_limit, (float)cfg->dist2goal, freeze, state_dot, ld_out);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_edge_attr_tangent(int env, const float* states, int ld_state, const float* state_dot, int ld_sdot, const int64_t* edge_index,
                                      int64_t num_edges, float* t_edge_attr, void* stream) {
  GCBF_REQUIRE(env >= 0 && env <= 2 && num_edges >= 0, "gcbf_edge_attr_tangent: bad arguments");
  const int sd = env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4;
  GCBF_REQUIRE(ld_state >= sd && ld_sdot >= sd, "gcbf_edge_attr_tangent: leading dimensions");
  if (num_edges == 0) return GCBF_OK;
  GCBF_REQUIRE(states && state_dot && edge_index && t_edge_attr, "gcbf_edge_attr_tangent: null pointer");
  const int grid = (int)imin64(ceil_div(num_edges, 256), 8 * kNumSMs);
  edge_attr_tangent_kernel<<<grid, 256, 0, as_stream(stream)>>>(env, states, ld_state, state_dot, ld_sdot, edge_index, num_edges, t_edge_attr);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_attn_aggr_tangent(const float* msg, int ld_msg, const float* t_msg, int ld_tmsg, const float* att, const float* t_gate,
                                      const int32_t* rowptr, int num_nodes, int channels, float* t_aggr, int ld_taggr, void* stream) {
  GCBF_REQUIRE(num_nodes >= 0 && channels >= 1 && ld_msg >= channels && ld_tmsg >= channels && ld_taggr >= channels, "gcbf_attn_aggr_tangent: bad sizes");
  if (num_nodes == 0) return GCBF_OK;
  GCBF_REQUIRE(rowptr && t_aggr, "gcbf_attn_aggr_tangent: null pointer");     // the edge arrays may be null for a graph without edges
  const int64_t total = (int64_t)num_nodes * channels;
  const int grid = (int)imin64(ceil_div(total, 256), 8 * kNumSMs);
  attn_tangent_kernel<<<grid, 256, 0, as_stream(stream)>>>(msg, ld_msg, t_msg, ld_tmsg, att, t_gate, rowptr, num_nodes, channels, t_aggr, ld_taggr);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

// ---- backward of the tangent pass (the analytic-h_dot training loss, GCBF.params['h_dot'] = 'analytic') ------------------------------

extern "C" int gcbf_attn_aggr_tangent_bwd(const float* msg, int ld_msg, const float* t_msg, int ld_tmsg, const float* att, const float* t_gate,
                                          const int32_t* rowptr, int num_nodes, int channels, const float* d_t_aggr, int ld_dtaggr, float* d_t_msg,
                                          int ld_dtmsg, float* d_t_gate, float* d_msg, int ld_dmsg, float* d_gate, int accumulate, void* stream) {
  GCBF_REQUIRE(num_nodes >= 0 && channels >= 1 && ld_msg >= channels && ld_tmsg >= channels && ld_dtaggr >= channels && ld_dtmsg >= channels &&
                   ld_dmsg >= channels, "gcbf_attn_aggr_tangent_bwd: bad sizes");
  if (num_nodes == 0) return GCBF_OK;
  GCBF_REQUIRE(rowptr && d_t_aggr, "gcbf_attn_aggr_tangent_bwd: null pointer");   // the edge arrays may be null for a graph without edges
  const int grid = (int)imin64(ceil_div((int64_t)num_nodes * 32, 256), 16 * kNumSMs);
  attn_tangent_bwd_kernel<<<grid, 256, 0, as_stream(stream)>>>(msg, ld_msg, t_msg, ld_tmsg, att, t_gate, rowptr, num_nodes, channels, d_t_aggr,
                                                               ld_dtaggr, d_t_msg, ld_dtmsg, d_t_gate, d_msg, ld_dmsg, d_gate, accumulate);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_act_tangent_bwd(const float* dY, const float* dTY, const float* Y, const float* TZ, int64_t count, int act, float* dZ,
                                    float* dTZ, void* stream) {
  GCBF_REQUIRE(count >= 0 && act >= 0 && act <= 2, "gcbf_act_tangent_bwd: bad arguments");
  if (count == 0) return GCBF_OK;
  GCBF_REQUIRE(dY && dTY && Y && dZ && dTZ && (act != 2 || TZ), "gcbf_act_tangent_bwd: null pointer");
  const int grid = (int)imin64(ceil_div(count, 256), 8 * kNumSMs);
  act_tangent_bwd_kernel<<<grid, 256, 0, as_stream(stream)>>>(dY, dTY, Y, TZ, count, act, dZ, dTZ);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_state_dot_bwd(const gcbf_env_cfg* cfg, const float* states, int ld_state, const float* action, const float* u_ref,
                                  const float* goal, int ld_goal, int goal_per_graph, int freeze, const float* d_state_dot, int ld_dsdot,
                                  float* d_action, int accumulate, void* stream) {
  GCBF_REQUIRE(cfg != nullptr, "gcbf_state_dot_bwd: null cfg");
  GCBF_REQUIRE(cfg->env >= 0 && cfg->env <= 2, "gcbf_state_dot_bwd: unknown env %d", cfg->env);
  GCBF_REQUIRE(cfg->num_graphs >= 0 && cfg->num_agents >= 0 && cfg->nodes_per_graph >= cfg->num_agents, "gcbf_state_dot_bwd: bad sizes");
  const int sd = cfg->env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4, pd = cfg->env == GCBF_ENV_SIMPLE_DRONE ? 3 : 2;
  GCBF_REQUIRE(ld_state >= sd && ld_dsdot >= sd, "gcbf_state_dot_bwd: leading dimensions");
  const int64_t agents = (int64_t)cfg->num_graphs * cfg->num_agents;
  GCBF_REQUIRE((int64_t)cfg->num_graphs * cfg->nodes_per_graph < (1ll << 31), "gcbf_state_dot_bwd: too many nodes");
  if (agents == 0) return GCBF_OK;
  GCBF_REQUIRE(states && action && u_ref && d_state_dot && d_action, "gcbf_state_dot_bwd: null pointer");
  GCBF_REQUIRE(!freeze || cfg->env == GCBF_ENV_SIMPLE_CAR || (goal && ld_goal >= pd), "gcbf_state_dot_bwd: the reach-freeze needs the goal positions");
  const float action_lim = cfg->env == GCBF_ENV_DUBINS_CAR ? 2.f : 10.f;       // as gcbf_state_dot
  const int grid = (int)imin64(ceil_div(agents, 256), 8 * kNumSMs);
  state_dot_bwd_kernel<<<grid, 256, 0, as_stream(stream)>>>(cfg->env, cfg->num_graphs, cfg->nodes_per_graph, cfg->num_agents, states, ld_state,
                                                            action, u_ref, goal, ld_goal, goal_per_graph ? cfg->num_agents : 0, action_lim,
                                                            (float)cfg->dist2goal, freeze, d_state_dot, ld_dsdot, d_action, accumulate);
  GCBF_LAUNCH_OK();
  return GCBF_OK;
}

extern "C" int gcbf_edge_attr_bwd_ordered(int env, const float* states, int ld_state, const int64_t* edge_index, int64_t num_edges, int num_nodes,
                                          const float* d_edge_attr, float* d_states, void* stream) {
  GCBF_REQUIRE(env >= 0 && env <= 2 && num_edges >= 0 && num_nodes >= 0, "gcbf_edge_attr_bwd_ordered: bad arguments");
  GCBF_REQUIRE(ld_state >= (env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4), "gcbf_edge_attr_bwd_ordered: leading dimension");
  if (num_edges == 0) return GCBF_OK;
  GCBF_REQUIRE(states && edge_index && d_edge_attr && d_states, "gcbf_edge_attr_bwd_ordered: null pointer");
  return edge_attr_bwd_ordered(env, states, ld_state, edge_index, num_edges, num_nodes, d_edge_attr, d_states, as_stream(stream));
}
