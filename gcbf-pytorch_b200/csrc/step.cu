// One inner iteration of GCBF.update (reference gcbf/algo/gcbf.py:158-226) as three C-ABI calls:
//
//   gcbf_step_forward   h = cbf(graphs) [:161], actions = actor(graphs) [:162] on the side stream, safe / unsafe masks [:168,180] in one
//                       launch, graphs_next = forward_graph(graphs, actions) [:193], h_next = cbf(graphs_next) [:194]; the per-graph
//                       single-step + radius re-link of [:195-199] is ONE batched count launch started on the side stream
//   gcbf_step_relink    the step's one host sync (re-linked edge count), h_next_new = cbf(re-linked) [:200-201] value-only on the side
//                       stream, loss partial sums [:169-212]
//   gcbf_step_backward  d loss / d (h, h_next, actions) [:215-218], backward through cbf (h_next -> edge_attr(x+) -> x+ -> clamp ->
//                       actions, then h) and the actor [:222], gradients accumulated straight into the descriptors' gW / gb
//
// Data-parallel callers all-reduce `partial` between relink and backward and the gradient bucket after backward; clip + Adam
// (gcbf_grad_sumsq / gcbf_clip_adam) follow.  The three CBF forwards advance the spectral-norm vectors in program order even though
// the third one runs on the side stream (event chain), exactly like the reference's three self.cbf(...) calls.
#include "chain.h"

namespace gcbf {
namespace chain {

struct StepCtx {
  NetCtx c1, c2, ca;                  // cbf(graphs), cbf(graphs_next), actor(graphs)
  uint8_t* ws_base; size_t ws_cap; size_t off_after_forward;
  float *h, *actions, *h_next, *h_next_new, *hdot, *scalars;
  uint8_t *safe, *unsafe, *coll, *pass_mask;
  double* partial;
  float *states_next, *ea_next, *st_relink;
  int32_t* rowptr_agents;
  int64_t E_new;
  int phase;                          // 1 after forward, 2 after relink
};
static_assert(sizeof(StepCtx) <= sizeof(gcbf_step_ctx), "gcbf_step_ctx too small");

// events + the pinned word the re-linked edge count is copied to (host resources, created once per process / device)
struct HostRes {
  int device = -1;
  cudaEvent_t fork = nullptr, actor_done = nullptr, inputs_ready = nullptr, pi2_done = nullptr, side_done = nullptr, dact_ready = nullptr,
              count_done = nullptr;
  int32_t* e_new_pinned = nullptr;
};
static HostRes g_res;

static int host_res(HostRes** out) {
  int dev = 0;
  GCBF_CUDA_OK(cudaGetDevice(&dev));
  if (g_res.device != dev) {
    cudaEvent_t* evs[] = {&g_res.fork, &g_res.actor_done, &g_res.inputs_ready, &g_res.pi2_done, &g_res.side_done, &g_res.dact_ready, &g_res.count_done};
    for (cudaEvent_t* e : evs) {
      if (*e) cudaEventDestroy(*e);
      GCBF_CUDA_OK(cudaEventCreateWithFlags(e, cudaEventDisableTiming));
    }
    if (!g_res.e_new_pinned) GCBF_CUDA_OK(cudaHostAlloc(&g_res.e_new_pinned, 64, cudaHostAllocDefault));
    g_res.device = dev;
  }
  *out = &g_res;
  return 0;
}

int check_step(const gcbf_step_desc* d, const gcbf_step_batch* b, const char* what) {
  if (!d || !b) { set_error("%s: null descriptor", what); return GCBF_E_INVALID; }
  if (int rc = check_net(&d->cbf)) return rc;
  if (int rc = check_net(&d->actor)) return rc;
  const int M = b->num_agents_total;
  if (d->cbf.n_head == 0 || d->actor.n_head == 0 || d->cbf.head[d->cbf.n_head - 1].N != 1 || d->actor.head[d->actor.n_head - 1].N != d->action_dim ||
      d->actor.head_extra_dim != d->action_dim || d->cbf.head_extra_dim != 0) {
    set_error("%s: cbf must end in a 1-wide head, the actor in an action_dim-wide head over cat[feat, u_ref]", what);
    return GCBF_E_INVALID;
  }
  if (b->num_edges < 0 || b->num_edges >= (1ll << 31) || b->num_nodes <= 0 || M <= 0 || M > b->num_nodes ||
      (long long)d->env.num_graphs * d->env.nodes_per_graph != b->num_nodes || (long long)d->env.num_graphs * d->env.num_agents != M ||
      (!b->row_index && M != b->num_nodes) || b->ld_state != d->state_dim) {
    set_error("%s: batch sizes (nodes %d, agents %d, graphs %d x %d)", what, b->num_nodes, M, d->env.num_graphs, d->env.nodes_per_graph);
    return GCBF_E_INVALID;
  }
  return 0;
}

// ---- forward ---------------------------------------------------------------------------------------------------------------
static int step_forward(Run& R, const gcbf_step_desc& d, const gcbf_step_batch& b, StepCtx* c, cudaStream_t main, cudaStream_t side, HostRes* hr) {
  const int M = b.num_agents_total, Nn = b.num_nodes, E = (int)b.num_edges, a = d.action_dim, s = d.state_dim;
  const int ed = d.cbf.edge_dim;
  // results first (small, read back by the caller)
  c->h = (float*)R.ws.alloc((size_t)M * 4);
  c->actions = (float*)R.ws.alloc((size_t)M * a * 4);
  c->h_next = (float*)R.ws.alloc((size_t)M * 4);
  c->h_next_new = (float*)R.ws.alloc((size_t)M * 4);
  c->hdot = (float*)R.ws.alloc((size_t)M * 4);
  c->scalars = (float*)R.ws.alloc(8 * 4);
  c->partial = (double*)R.ws.alloc(GCBF_LP_SIZE * 8);
  c->safe = (uint8_t*)R.ws.alloc((size_t)3 * M);
  c->unsafe = c->safe + M;
  c->coll = c->safe + 2 * (size_t)M;
  c->pass_mask = (uint8_t*)R.ws.alloc((size_t)M * a);
  c->states_next = (float*)R.ws.alloc((size_t)Nn * s * 4);
  c->ea_next = (float*)R.ws.alloc((size_t)E * ed * 4);
  c->st_relink = (float*)R.ws.alloc((size_t)Nn * s * 4);
  c->rowptr_agents = (int32_t*)R.ws.alloc((size_t)(M + 1) * 4);
  uint8_t* pm_relink = (uint8_t*)R.ws.alloc((size_t)M * a);     // clamp mask of the re-link step (not differentiated)
  gcbf_net_desc cbf_again = d.cbf;                               // weight companions are refreshed by the FIRST pass of a net only
  cbf_again.refresh_weights = 0;
  const bool two = side != nullptr && side != main && !R.dry;
  // h and the actor's actions are independent: the actor's forward runs on the side stream so its kernels fill the CBF net's wave tails
  if (two) { CHAIN_CUDA(cudaEventRecord(hr->fork, main)); CHAIN_CUDA(cudaStreamWaitEvent(side, hr->fork, 0)); }
  R.st = two ? side : main;
  if (int rc = net_forward(R, d.actor, b.x, b.edge_attr, b.edge_index, b.rowptr, E, Nn, b.row_index, M, b.u_ref, c->actions, a, &c->ca)) return rc;   // gcbf.py:162
  if (two) CHAIN_CUDA(cudaEventRecord(hr->actor_done, side));
  R.st = main;
  if (int rc = net_forward(R, d.cbf, b.x, b.edge_attr, b.edge_index, b.rowptr, E, Nn, b.row_index, M, nullptr, c->h, 1, &c->c1)) return rc;           // gcbf.py:161 (power iteration #1)
  if (two) CHAIN_CUDA(cudaStreamWaitEvent(main, hr->actor_done, 0));
  gcbf_env_cfg cfg = d.env;
  if (!R.dry) {
    CHAIN_CALL(gcbf_masks(&cfg, b.states, b.ld_state, c->safe, c->unsafe, c->coll, main));                                                   // gcbf.py:168, 180
    // graphs_next = env.forward_graph(graphs, actions): retained edges, new edge features  (gcbf.py:193).  A batch of exactly one
    // graph satisfies the reference's single-graph discriminator (dubins_car.py:126): reach-freeze branch
    CHAIN_CALL((d.goal_per_graph ? gcbf_step_fwd_multi : gcbf_step_fwd)(&cfg, b.states, b.ld_state, c->actions, d.goal, d.ld_goal, d.lqr_gain,
                                                                      d.env.num_graphs == 1 ? 1 : 0, c->states_next, c->pass_mask, main));
    CHAIN_CALL(gcbf_edge_attr_fwd(d.env.env, c->states_next, s, b.edge_index, E, c->ea_next, main));
    R.launched(E ? 3 : 2);
    if (two) CHAIN_CUDA(cudaEventRecord(hr->inputs_ready, main));
  }
  if (int rc = net_forward(R, cbf_again, b.x, c->ea_next, b.edge_index, b.rowptr, E, Nn, b.row_index, M, nullptr, c->h_next, 1, &c->c2)) return rc;       // gcbf.py:194 (power iteration #2)
  if (!R.dry) {
    if (two) { CHAIN_CUDA(cudaEventRecord(hr->pi2_done, main)); CHAIN_CUDA(cudaStreamWaitEvent(side, hr->inputs_ready, 0)); }
    cudaStream_t rs = two ? side : main;
    // gcbf.py:195-199, batched: every graph is a SINGLE graph there, so the reach-freeze branch applies; then the radius count
    CHAIN_CALL((d.goal_per_graph ? gcbf_step_fwd_multi : gcbf_step_fwd)(&cfg, b.states, b.ld_state, c->actions, d.goal, d.ld_goal, d.lqr_gain, 1,
                                                                      c->st_relink, pm_relink, rs));
    CHAIN_CALL(gcbf_radius_graph_count(c->st_relink, s, d.pos_dim, d.env.num_graphs, d.env.nodes_per_graph, d.env.num_agents, d.comm_radius,
                                       d.graph_metric, c->rowptr_agents, rs));
    CHAIN_CUDA(cudaMemcpyAsync(hr->e_new_pinned, c->rowptr_agents + M, 4, cudaMemcpyDeviceToHost, rs));
    CHAIN_CUDA(cudaEventRecord(hr->count_done, rs));
    R.launched(3);
  }
  return 0;
}

// ---- re-linked value pass + loss partials -------------------------------------------------------------------------------------
static int step_relink(Run& R, const gcbf_step_desc& d, const gcbf_step_batch& b, StepCtx* c, int64_t E_new, gcbf_step_out* out,
                       cudaStream_t main, cudaStream_t side, HostRes* hr) {
  const int M = b.num_agents_total, Nn = b.num_nodes, s = d.state_dim, ed = d.cbf.edge_dim;
  const bool two = side != nullptr && side != main && !R.dry;
  cudaStream_t rs = two ? side : main;
  R.st = rs;
  int64_t* ei = (int64_t*)R.ws.alloc((size_t)2 * E_new * 8);
  int32_t* rowptr = (int32_t*)R.ws.alloc((size_t)(Nn + 1) * 4);
  int32_t* flag = (int32_t*)R.ws.alloc(4);
  float* ea = (float*)R.ws.alloc((size_t)E_new * ed * 4);
  gcbf_net_desc cbf_again = d.cbf;
  cbf_again.refresh_weights = 0;
  if (!R.dry) {
    CHAIN_CALL(gcbf_radius_graph_fill(c->st_relink, s, d.pos_dim, d.env.num_graphs, d.env.nodes_per_graph, d.env.num_agents, d.comm_radius,
                                      d.graph_metric, c->rowptr_agents, E_new ? ei : nullptr, E_new, rs));
    CHAIN_CALL(gcbf_rowptr_from_targets(E_new ? ei + E_new : nullptr, E_new, Nn, rowptr, flag, rs));
    CHAIN_CALL(gcbf_edge_attr_fwd(d.env.env, c->st_relink, s, ei, E_new, ea, rs));
    R.launched(E_new ? 3 : 2);
    if (two) CHAIN_CUDA(cudaStreamWaitEvent(side, hr->pi2_done, 0));       // power iteration #3 stays behind #2 (and its snapshot)
  }
  if (int rc = net_forward(R, cbf_again, b.x, ea, ei, rowptr, E_new, Nn, b.row_index, M, nullptr, c->h_next_new, 1, nullptr)) return rc;   // gcbf.py:200-201, value only
  if (!R.dry) {
    if (two) { CHAIN_CUDA(cudaEventRecord(hr->side_done, side)); CHAIN_CUDA(cudaStreamWaitEvent(main, hr->side_done, 0)); }
    CHAIN_CALL(gcbf_loss_partials(c->h, c->h_next, c->h_next_new, c->actions, d.action_dim, c->safe, c->unsafe, M, d.alpha, d.eps,
                                  (float)d.env.dt, c->partial, c->hdot, main));
    R.launched(1);
    out->edge_index_new = ei;
    out->num_edges_new = E_new;
  }
  return 0;
}

// ---- backward ----------------------------------------------------------------------------------------------------------------
static int step_backward(Run& R, const gcbf_step_desc& d, const gcbf_step_batch& b, StepCtx* c, cudaStream_t main, cudaStream_t side,
                         HostRes* hr, void* const* events) {
  const int M = b.num_agents_total, Nn = b.num_nodes, E = (int)b.num_edges, a = d.action_dim, s = d.state_dim, ed = d.cbf.edge_dim;
  const bool two = side != nullptr && side != main && !R.dry;
  R.st = main;
  float* d_h = (float*)R.ws.alloc((size_t)M * 4);
  float* d_hn = (float*)R.ws.alloc((size_t)M * 4);
  float* d_act = (float*)R.ws.alloc((size_t)M * a * 4);
  float* d_act_dyn = (float*)R.ws.alloc((size_t)M * a * 4);
  float* d_ea = (float*)R.ws.alloc((size_t)E * ed * 4);
  float* d_states = (float*)R.ws.alloc((size_t)Nn * s * 4);
  gcbf_env_cfg cfg = d.env;
  if (!R.dry) {
    CHAIN_CALL(gcbf_loss_grads(c->h, c->h_next, c->h_next_new, c->actions, a, c->safe, c->unsafe, M, d.alpha, d.eps, (float)d.env.dt,
                               d.coef_unsafe, d.coef_safe, d.coef_hdot, d.coef_action, c->partial, d_h, d_hn, d_act, c->scalars, main));
    R.launched(1);
    if (d.grad_bucket) CHAIN_CUDA(cudaMemsetAsync(d.grad_bucket, 0, (size_t)d.grad_bucket_floats * 4, main));                  // gcbf.py:220-221
  }
  // the two CBF passes accumulate into the same gradient buffers: same stream, one after the other; their scratch is shared
  const size_t mark = R.ws.off;
  if (int rc = net_backward(R, d.cbf, c->c2, b.rowptr, b.row_index, d_hn, 1, d_ea, false)) return rc;      // h_next -> cbf params, edge_attr(x+)
  if (!R.dry) {
    // edge_attr(x+) -> x+ -> clamp(u + u_ref) -> actions  (VJP of forward_graph, gcbf.py:193)
    CHAIN_CUDA(cudaMemsetAsync(d_states, 0, (size_t)Nn * s * 4, main));
    CHAIN_CALL(edge_attr_bwd_ordered(d.env.env, c->states_next, s, b.edge_index, E, Nn, d_ea, d_states, main));
    CHAIN_CALL(gcbf_step_bwd(&cfg, d_states, s, c->pass_mask, d_act_dyn, main));
    R.launched(E ? 2 : 1);
  }
  if (int rc = vec_add(R, d_act, d_act_dyn, (int64_t)M * a)) return rc;
  if (two) { CHAIN_CUDA(cudaEventRecord(hr->dact_ready, main)); }
  const size_t after2 = R.ws.off;
  R.ws.off = mark;
  // (events: the gamma + head gradients of a net are final once its LAST pass is through gamma -- callers start that range's
  // all-reduce there, while the E-row phi / gate backward still runs)
  if (int rc = net_backward(R, d.cbf, c->c1, b.rowptr, b.row_index, d_h, 1, nullptr, false, (events && !R.dry) ? (cudaEvent_t)events[0] : nullptr)) return rc;    // h -> cbf params
  if (events && !R.dry) CHAIN_CUDA(cudaEventRecord((cudaEvent_t)events[1], main));
  const size_t after1 = R.ws.off;
  R.ws.off = after1 > after2 ? after1 : after2;
  // the actor's backward only needs d_act: on the side stream it overlaps the second CBF backward
  if (two) { CHAIN_CUDA(cudaStreamWaitEvent(side, hr->dact_ready, 0)); R.st = side; }
  if (int rc = net_backward(R, d.actor, c->ca, b.rowptr, b.row_index, d_act, a, nullptr, false, (events && !R.dry) ? (cudaEvent_t)events[2] : nullptr)) return rc;
  if (events && !R.dry) CHAIN_CUDA(cudaEventRecord((cudaEvent_t)events[3], R.st));
  if (two) { CHAIN_CUDA(cudaEventRecord(hr->side_done, side)); CHAIN_CUDA(cudaStreamWaitEvent(main, hr->side_done, 0)); }
  R.st = main;
  return 0;
}

static void fill_out(const StepCtx& c, gcbf_step_out* out) {
  out->h = c.h; out->actions = c.actions; out->h_next = c.h_next; out->h_next_new = c.h_next_new; out->hdot = c.hdot; out->scalars = c.scalars;
  out->safe = c.safe; out->unsafe = c.unsafe; out->partial = c.partial;
}

}  // namespace chain
}  // namespace gcbf

using namespace gcbf;
using namespace gcbf::chain;

extern "C" size_t gcbf_step_workspace_bytes(const gcbf_step_desc* d, const gcbf_step_batch* b) {
  if (check_step(d, b, "gcbf_step_workspace_bytes")) return 0;
  Run R(nullptr, 0, nullptr, true);
  StepCtx c;
  memset(&c, 0, sizeof(c));
  if (step_forward(R, *d, *b, &c, nullptr, nullptr, nullptr)) return 0;
  if (step_backward(R, *d, *b, &c, nullptr, nullptr, nullptr, nullptr)) return 0;
  return R.ws.off + 4096;
}

extern "C" size_t gcbf_step_relink_workspace_bytes(const gcbf_step_desc* d, const gcbf_step_batch* b, int64_t num_edges_new) {
  if (check_step(d, b, "gcbf_step_relink_workspace_bytes") || num_edges_new < 0) return 0;
  Run R(nullptr, 0, nullptr, true);
  StepCtx c;
  memset(&c, 0, sizeof(c));
  gcbf_step_out o;
  if (step_relink(R, *d, *b, &c, num_edges_new, &o, nullptr, nullptr, nullptr)) return 0;
  return R.ws.off + 4096;
}

extern "C" int gcbf_step_forward(const gcbf_step_desc* d, const gcbf_step_batch* b, void* workspace, size_t workspace_bytes,
                                 gcbf_step_ctx* ctx, gcbf_step_out* out, void* stream, void* side_stream) {
  if (int rc = check_step(d, b, "gcbf_step_forward")) return rc;
  GCBF_REQUIRE(ctx && out && workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "gcbf_step_forward: bad arguments");
  GCBF_REQUIRE(b->states && b->x && b->rowptr && b->u_ref && d->goal && (b->num_edges == 0 || (b->edge_attr && b->edge_index)), "gcbf_step_forward: null pointer");
  const size_t need = gcbf_step_workspace_bytes(d, b);
  if (need > workspace_bytes) { set_error("gcbf_step_forward: workspace too small (%zu needed, %zu given)", need, workspace_bytes); return GCBF_E_WORKSPACE; }
  HostRes* hr;
  if (int rc = host_res(&hr)) return rc;
  StepCtx* c = reinterpret_cast<StepCtx*>(ctx);
  memset(c, 0, sizeof(*c));
  memset(out, 0, sizeof(*out));
  Run R(workspace, workspace_bytes, as_stream(stream), false);
  int rc = step_forward(R, *d, *b, c, as_stream(stream), as_stream(side_stream), hr);
  c->ws_base = static_cast<uint8_t*>(workspace); c->ws_cap = workspace_bytes; c->off_after_forward = R.ws.off;
  c->phase = 1;
  fill_out(*c, out);
  return R.finish(rc, "gcbf_step_forward");
}

extern "C" int gcbf_step_relink(const gcbf_step_desc* d, const gcbf_step_batch* b, gcbf_step_ctx* ctx, void* workspace2,
                                size_t workspace2_bytes, size_t* needed_bytes, gcbf_step_out* out, void* stream, void* side_stream) {
  if (int rc = check_step(d, b, "gcbf_step_relink")) return rc;
  GCBF_REQUIRE(ctx && out && needed_bytes, "gcbf_step_relink: bad arguments");
  StepCtx* c = reinterpret_cast<StepCtx*>(ctx);
  GCBF_REQUIRE(c->phase >= 1, "gcbf_step_relink: call gcbf_step_forward first");
  HostRes* hr;
  if (int rc = host_res(&hr)) return rc;
  if (c->phase == 1) {
    GCBF_CUDA_OK(cudaEventSynchronize(hr->count_done));        // the step's one host sync: the re-linked edge count
    c->E_new = *hr->e_new_pinned;
    c->phase = 2;
  }
  const size_t need = gcbf_step_relink_workspace_bytes(d, b, c->E_new);
  *needed_bytes = need;
  if (need > workspace2_bytes || !workspace2) {
    set_error("gcbf_step_relink: workspace2 too small for %lld re-linked edges (%zu needed, %zu given)", (long long)c->E_new, need, workspace2_bytes);
    return GCBF_E_WORKSPACE;                                   // nothing launched: call again with a larger workspace2
  }
  GCBF_REQUIRE((reinterpret_cast<uintptr_t>(workspace2) & 255) == 0, "gcbf_step_relink: workspace2 must be 256-byte aligned");
  Run R(workspace2, workspace2_bytes, as_stream(stream), false);
  fill_out(*c, out);
  int rc = step_relink(R, *d, *b, c, c->E_new, out, as_stream(stream), as_stream(side_stream), hr);
  c->phase = 3;
  return R.finish(rc, "gcbf_step_relink");
}

extern "C" int gcbf_step_backward(const gcbf_step_desc* d, const gcbf_step_batch* b, gcbf_step_ctx* ctx, gcbf_step_out* out, void* const* events,
                                  void* stream, void* side_stream) {
  if (int rc = check_step(d, b, "gcbf_step_backward")) return rc;
  GCBF_REQUIRE(ctx && out, "gcbf_step_backward: bad arguments");
  StepCtx* c = reinterpret_cast<StepCtx*>(ctx);
  GCBF_REQUIRE(c->phase == 3, "gcbf_step_backward: call gcbf_step_forward and gcbf_step_relink first");
  HostRes* hr;
  if (int rc = host_res(&hr)) return rc;
  Run R(c->ws_base, c->ws_cap, as_stream(stream), false);
  R.ws.off = c->off_after_forward;
  int rc = step_backward(R, *d, *b, c, as_stream(stream), as_stream(side_stream), hr, events);
  c->phase = 4;
  return R.finish(rc, "gcbf_step_backward");
}
