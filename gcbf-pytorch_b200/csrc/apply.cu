// GCBF.apply, the test-time controller (reference gcbf/algo/gcbf.py:260-309), as ONE C-ABI call for B graphs at once:
//
//   h = cbf(graph) [:262], action = actor(graph) [:263], h_next = cbf(forward_graph(graph, 0)) [:264-267]; agents whose nominal (zero)
//   action satisfies the h_dot condition keep it [:271-273]; then up to max_iter + 1 rounds of
//       h_next = cbf(forward_graph(graph, action)) [:288-290], max_val = relu(-h_dot - alpha h) [:291-292],
//       a graph is done when none of its agents violates or the round counter passed max_iter [:294],
//       d mean_g(max_val) / d action through the CBF net's input-gradient path (no weight gradient) [:300],
//       one Adam(lr) step per VIOLATING agent (its own step count) [:298-302] + the gradient-proportional noise [:305].
//
// Every piece of the loop's state is per agent (action, Adam moments, step count) or per graph (done flag, round count), and the GNN
// passes are block-diagonal, so graph g of a batch computes exactly what a call on graph g alone computes: a done graph keeps its
// action, gets no Adam step and is not re-evaluated, while the other graphs go on.  The reference keeps one torch.optim.Adam per
// agent; here the per-agent optimiser state is three small arrays (m, v, step count) and one kernel updates every violating agent.
// Each round costs one host sync (the number of graphs still refining decides whether the backward is launched at all), like the
// reference's `if loss_h_dot <= 0` [:294].  Every CBF pass advances the spectral-norm vectors (the reference never calls .eval(),
// SURVEY 3.5); a batch makes the passes of its slowest graph, in the same order.  gcbf_apply is the one-graph case.
#include <cstdlib>

#include "chain.h"

namespace gcbf {
namespace chain {

// keep the actor's action only where the nominal action violates the condition; zero the optimiser state
__global__ void apply_init_kernel(const float* __restrict__ h, const float* __restrict__ hn, const float* __restrict__ actor_action,
                                  float* __restrict__ act, float* __restrict__ m, float* __restrict__ v, float* __restrict__ t, int M,
                                  int a, float dt, float alpha) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M * a) return;
  const int r = i / a;
  const float hd = __fdiv_rn(__fsub_rn(hn[r], h[r]), dt);
  const float viol = fmaxf(__fsub_rn(-hd, __fmul_rn(alpha, h[r])), 0.f);
  act[i] = viol <= 0.f ? 0.f : actor_action[i];
  m[i] = 0.f;
  v[i] = 0.f;
  if (i % a == 0) t[r] = 0.f;
}

// max_val = relu(-h_dot - alpha h) of the graphs still refining (0 for done graphs), d mean_g(max_val) / d h_next (n = agents per graph),
// violating agents per graph.  Integer atomics: the counts do not depend on the order (warps straddle graphs when n < 32)
__global__ void apply_viol_kernel(const float* __restrict__ h, const float* __restrict__ hn, const int* __restrict__ done,
                                  float* __restrict__ max_val, float* __restrict__ d_hn, int* __restrict__ graph_count, int M, int n,
                                  float dt, float alpha) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const int g = i / n;
  float mv = 0.f;
  if (!done[g]) {
    const float hd = __fdiv_rn(__fsub_rn(hn[i], h[i]), dt);
    mv = fmaxf(__fsub_rn(-hd, __fmul_rn(alpha, h[i])), 0.f);
  }
  max_val[i] = mv;
  const bool on = mv > 0.f;
  d_hn[i] = on ? -1.f / (dt * (float)n) : 0.f;
  if (on) atomicAdd(graph_count + g, 1);
}

// after round `count[1]` was evaluated: a graph with no violating agent, or any graph once the round counter passed max_iter, is done
// (rounds[g] = the Adam rounds it did); count[0] = graphs still refining (what the host reads), count[1] += 1 (the Adam kernel of this
// round reads noise slice count[1] - 1).  One block; the per-graph counts are cleared for the next round.
__global__ void apply_done_kernel(int* __restrict__ done, int* __restrict__ graph_count, int32_t* __restrict__ rounds,
                                  int* __restrict__ count, int G, int max_iter) {
  __shared__ int active;
  if (threadIdx.x == 0) active = 0;
  __syncthreads();
  const int it = count[1];
  int mine = 0;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    if (!done[g]) {
      if (graph_count[g] == 0 || it > max_iter) {
        done[g] = 1;
        rounds[g] = it;
      } else {
        ++mine;
      }
    }
    graph_count[g] = 0;
  }
  if (mine) atomicAdd(&active, mine);
  __syncthreads();
  if (threadIdx.x == 0) {
    count[0] = active;
    count[1] = it + 1;
  }
}

// torch.optim.Adam(lr, betas (0.9, 0.999), eps 1e-8) on the rows with max_val != 0, each with its own step count, then
// action -= rand * lr * noise * grad  (gcbf.py:301-305)
__global__ void agent_adam_kernel(float* __restrict__ act, float* __restrict__ m, float* __restrict__ v, float* __restrict__ t,
                                  const float* __restrict__ g, const float* __restrict__ max_val, const float* __restrict__ noise_all,
                                  const int* __restrict__ rounds, int M, int a, float lr, float rand) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;      // one thread per agent (= per reference optimiser)
  if (r >= M || max_val[r] == 0.f) return;
  // this round's slice of the noise: the round index lives on the device so that the launch is identical every round (CUDA graph)
  const float* noise = noise_all ? noise_all + (size_t)(rounds[1] - 1) * M * a : nullptr;
  const float step = t[r] + 1.f;
  t[r] = step;
  const double bc1 = 1.0 - pow(0.9, (double)step), bc2 = 1.0 - pow(0.999, (double)step);
  const float step_size = (float)((double)lr / bc1), bc2_sqrt = (float)sqrt(bc2);
  for (int k = 0; k < a; ++k) {
    const int i = r * a + k;
    const float gi = g[i];
    const float mi = m[i] + (gi - m[i]) * (1.f - 0.9f);                      // exp_avg.lerp_(grad, 1 - beta1)
    const float vi = v[i] * 0.999f + (1.f - 0.999f) * gi * gi;               // exp_avg_sq.mul_(beta2).addcmul_(grad, grad, 1 - beta2)
    float p = act[i] - step_size * (mi / (sqrtf(vi) / bc2_sqrt + 1e-8f));     // param.addcdiv_(exp_avg, denom, -step_size)
    if (noise) p -= rand * lr * noise[i] * gi;                               // gcbf.py:305
    act[i] = p;
    m[i] = mi;
    v[i] = vi;
  }
}

struct ApplyBufs {
  float *h, *actor_action, *hn, *act, *m, *v, *t, *max_val, *d_hn, *zero_action, *states_next, *ea_next, *g, *d_ea, *d_states;
  uint8_t* pass_mask;
  int* count;                     // [0] graphs still refining after the round, [1] rounds evaluated
  int *done, *graph_count;        // per graph
  int32_t* rounds;                // per graph: the caller's array, or workspace for gcbf_apply
};

static int* g_pinned_count = nullptr;

// one forward_graph + CBF pass for the current `action`
static int apply_forward(Run& R, const gcbf_step_desc& d, const gcbf_step_batch& b, const gcbf_net_desc& cbf, const ApplyBufs& B,
                         const float* action, NetCtx* ctx) {
  const int M = b.num_agents_total, Nn = b.num_nodes, E = (int)b.num_edges, s = d.state_dim;
  gcbf_env_cfg cfg = d.env;
  if (!R.dry) {
    // every graph is a single graph of the reference: the reach-freeze branch of forward_graph (dubins_car.py:126), per graph
    CHAIN_CALL((d.goal_per_graph ? gcbf_step_fwd_multi : gcbf_step_fwd)(&cfg, b.states, b.ld_state, action, d.goal, d.ld_goal, d.lqr_gain, 1,
                                                                        B.states_next, B.pass_mask, R.st));
    CHAIN_CALL(gcbf_edge_attr_fwd(d.env.env, B.states_next, s, b.edge_index, E, B.ea_next, R.st));
    R.launched(E ? 2 : 1);
  }
  return net_forward(R, cbf, b.x, B.ea_next, b.edge_index, b.rowptr, E, Nn, b.row_index, M, nullptr, B.hn, 1, ctx);
}

// rounds: device int32[num_graphs] or NULL (workspace); *iterations (optional): rounds of the slowest graph
static int apply_run(Run& R, const gcbf_step_desc& d, const gcbf_step_batch& b, float lr, float rand, const float* noise, int max_iter,
                     float* action_out, int ld_action, int32_t* rounds, int* iterations, const char* what) {
  const int M = b.num_agents_total, Nn = b.num_nodes, E = (int)b.num_edges, a = d.action_dim, s = d.state_dim, ed = d.cbf.edge_dim;
  const int G = d.env.num_graphs, n = d.env.num_agents;
  const float dt = (float)d.env.dt;
  ApplyBufs B;
  B.h = (float*)R.ws.alloc((size_t)M * 4);
  B.hn = (float*)R.ws.alloc((size_t)M * 4);
  B.max_val = (float*)R.ws.alloc((size_t)M * 4);
  B.d_hn = (float*)R.ws.alloc((size_t)M * 4);
  B.t = (float*)R.ws.alloc((size_t)M * 4);
  B.actor_action = (float*)R.ws.alloc((size_t)M * a * 4);
  B.act = (float*)R.ws.alloc((size_t)M * a * 4);
  B.m = (float*)R.ws.alloc((size_t)M * a * 4);
  B.v = (float*)R.ws.alloc((size_t)M * a * 4);
  B.g = (float*)R.ws.alloc((size_t)M * a * 4);
  B.zero_action = (float*)R.ws.alloc((size_t)M * a * 4);
  B.pass_mask = (uint8_t*)R.ws.alloc((size_t)M * a);
  B.count = (int*)R.ws.alloc(256);
  B.done = (int*)R.ws.alloc((size_t)G * 4 * 2);
  B.graph_count = B.done + G;
  B.rounds = (int32_t*)R.ws.alloc((size_t)G * 4);
  if (rounds) B.rounds = rounds;
  B.states_next = (float*)R.ws.alloc((size_t)Nn * s * 4);
  B.d_states = (float*)R.ws.alloc((size_t)Nn * s * 4);
  B.ea_next = (float*)R.ws.alloc((size_t)E * ed * 4);
  B.d_ea = (float*)R.ws.alloc((size_t)E * ed * 4);
  gcbf_net_desc cbf_again = d.cbf;
  cbf_again.refresh_weights = 0;
  gcbf_env_cfg cfg = d.env;
  const int grid_ma = ceil_div(M * a, 256), grid_m = ceil_div(M, 256), block_g = G < 256 ? 32 * ceil_div(G, 32) : 256;
  const size_t mark0 = R.ws.off;
  if (int rc = net_forward(R, d.cbf, b.x, b.edge_attr, b.edge_index, b.rowptr, E, Nn, b.row_index, M, nullptr, B.h, 1, nullptr)) return rc;            // :262
  size_t peak = R.ws.off;
  R.ws.off = mark0;
  if (int rc = net_forward(R, d.actor, b.x, b.edge_attr, b.edge_index, b.rowptr, E, Nn, b.row_index, M, b.u_ref, B.actor_action, a, nullptr)) return rc;   // :263
  peak = peak > R.ws.off ? peak : R.ws.off;
  R.ws.off = mark0;
  if (!R.dry) CHAIN_CUDA(cudaMemsetAsync(B.zero_action, 0, (size_t)M * a * 4, R.st));
  if (int rc = apply_forward(R, d, b, cbf_again, B, B.zero_action, nullptr)) return rc;                                                                // :264-267
  peak = peak > R.ws.off ? peak : R.ws.off;
  R.ws.off = mark0;
  if (!R.dry) {
    apply_init_kernel<<<grid_ma, 256, 0, R.st>>>(B.h, B.hn, B.actor_action, B.act, B.m, B.v, B.t, M, a, dt, d.alpha);                                    // :268-273
    GCBF_LAUNCH_OK();
    R.launched(2);
  }
  // One round = two launch sequences around the host's look at the number of graphs still refining.  Every round of a call launches exactly the
  // same kernels on the same pointers (the workspace is rewound, the noise slice is picked on the device), so round 1 is captured into
  // two CUDA graphs that rounds 2.. replay: ~75 dependent launches of a few microseconds each become two graph launches.  Round 0 runs
  // eagerly (one-time attribute / descriptor set-up happens there); GCBF_APPLY_GRAPH=0, per-launch timing or a failed capture keep the
  // eager path.
  NetCtx ctx;
  auto round_fwd = [&]() -> int {
    if (int rc = apply_forward(R, d, b, cbf_again, B, B.act, &ctx)) return rc;                                                                          // :288-290
    if (!R.dry) {
      apply_viol_kernel<<<grid_m, 256, 0, R.st>>>(B.h, B.hn, B.done, B.max_val, B.d_hn, B.graph_count, M, n, dt, d.alpha);                              // :291-293
      GCBF_LAUNCH_OK();
      apply_done_kernel<<<1, block_g, 0, R.st>>>(B.done, B.graph_count, B.rounds, B.count, G, max_iter);                                                // :294
      GCBF_LAUNCH_OK();
      CHAIN_CUDA(cudaMemcpyAsync(g_pinned_count, B.count, 4, cudaMemcpyDeviceToHost, R.st));
      R.launched(3);
    }
    return 0;
  };
  auto round_bwd = [&]() -> int {
    if (int rc = net_backward(R, cbf_again, ctx, b.rowptr, b.row_index, B.d_hn, 1, B.d_ea, true)) return rc;                                            // :300 (no weight gradient)
    peak = peak > R.ws.off ? peak : R.ws.off;
    R.ws.off = mark0;
    if (R.dry) return 0;
    CHAIN_CUDA(cudaMemsetAsync(B.d_states, 0, (size_t)Nn * s * 4, R.st));
    CHAIN_CALL(edge_attr_bwd_ordered(d.env.env, B.states_next, s, b.edge_index, E, Nn, B.d_ea, B.d_states, R.st));
    CHAIN_CALL(gcbf_step_bwd(&cfg, B.d_states, s, B.pass_mask, B.g, R.st));
    agent_adam_kernel<<<grid_m, 256, 0, R.st>>>(B.act, B.m, B.v, B.t, B.g, B.max_val, noise, B.count, M, a, lr, rand);                                  // :301-305
    GCBF_LAUNCH_OK();
    R.launched(E ? 4 : 3);
    return 0;
  };
  struct Captured { cudaGraphExec_t exec = nullptr; long long launches = 0; } gf, gb;
  bool graphs = !R.dry && !timing_on() && max_iter >= 3;
  if (graphs) { const char* e = getenv("GCBF_APPLY_GRAPH"); graphs = !(e && e[0] == '0'); }
  // runs `body` under stream capture, instantiates and launches the result; on any capture problem falls back to running it eagerly
  auto capture_and_launch = [&](Captured& c, auto& body) -> int {
    const long long before = g_launches.load(std::memory_order_relaxed);
    const size_t off_before = R.ws.off;
    bool ok = cudaStreamBeginCapture(R.st, cudaStreamCaptureModeRelaxed) == cudaSuccess;
    int rc = 0;
    if (ok) {
      rc = body();
      cudaGraph_t graph = nullptr;
      ok = (cudaStreamEndCapture(R.st, &graph) == cudaSuccess) && rc == 0 && graph != nullptr;
      if (ok) ok = cudaGraphInstantiate(&c.exec, graph, 0) == cudaSuccess;
      if (graph) cudaGraphDestroy(graph);
      c.launches = g_launches.load(std::memory_order_relaxed) - before;
    }
    if (!ok) {
      (void)cudaGetLastError();
      if (c.exec) { cudaGraphExecDestroy(c.exec); c.exec = nullptr; }
      graphs = false;
      g_launches.store(before, std::memory_order_relaxed);
      R.ws.off = off_before;
      return body();                       // nothing of the captured sequence has run: run it now
    }
    CHAIN_CUDA(cudaGraphLaunch(c.exec, R.st));
    return 0;
  };
  auto cleanup = [&]() {
    if (gf.exec) cudaGraphExecDestroy(gf.exec);
    if (gb.exec) cudaGraphExecDestroy(gb.exec);
  };
  if (!R.dry) {
    CHAIN_CUDA(cudaMemsetAsync(B.count, 0, 8, R.st));                  // [0] graphs still refining, [1] rounds evaluated
    CHAIN_CUDA(cudaMemsetAsync(B.done, 0, (size_t)G * 4 * 2, R.st));   // done flags, per-graph violating counts
  }
  int it = 0;
  for (;; ++it) {
    int rc = 0;
    if (graphs && gf.exec) { rc = cudaGraphLaunch(gf.exec, R.st) == cudaSuccess ? 0 : GCBF_E_CUDA; R.launched((int)gf.launches); }
    else if (graphs && it == 1) rc = capture_and_launch(gf, round_fwd);
    else rc = round_fwd();
    if (rc) { cleanup(); return rc; }
    if (!R.dry) {
      if (cudaStreamSynchronize(R.st) != cudaSuccess) { cleanup(); set_error("%s: %s", what, cudaGetErrorString(cudaGetLastError())); return GCBF_E_CUDA; }
      if (*g_pinned_count == 0 || it > max_iter) break;                // every graph done (past max_iter all of them are)    :294
    }
    if (graphs && gb.exec) { rc = cudaGraphLaunch(gb.exec, R.st) == cudaSuccess ? 0 : GCBF_E_CUDA; R.launched((int)gb.launches); }
    else if (graphs && it == 1) rc = capture_and_launch(gb, round_bwd);
    else rc = round_bwd();
    if (rc) { cleanup(); return rc; }
    if (R.dry) break;
  }
  cleanup();
  R.ws.off = peak;
  if (!R.dry) {
    CHAIN_CUDA(cudaMemcpy2DAsync(action_out, (size_t)ld_action * 4, B.act, (size_t)a * 4, (size_t)a * 4, M, cudaMemcpyDeviceToDevice, R.st));
    if (iterations) *iterations = it;
  }
  return 0;
}

}  // namespace chain
}  // namespace gcbf

using namespace gcbf;
using namespace gcbf::chain;

static size_t apply_workspace(const gcbf_step_desc* d, const gcbf_step_batch* g, const char* what) {
  if (check_step(d, g, what)) return 0;
  Run R(nullptr, 0, nullptr, true);
  if (apply_run(R, *d, *g, 0.f, 0.f, nullptr, 0, nullptr, 0, nullptr, nullptr, what)) return 0;
  return R.ws.off + 4096;
}

// the checks both entry points make before any CUDA call
static int apply_check(const gcbf_step_desc* d, const gcbf_step_batch* g, float lr, float rand, const float* noise, int max_iter,
                       const float* action, int ld_action, void* workspace, size_t workspace_bytes, const char* what) {
  GCBF_REQUIRE(action && ld_action >= d->action_dim && max_iter >= 0 && lr > 0.f && workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0,
               "%s: bad arguments", what);
  GCBF_REQUIRE(rand == 0.f || noise, "%s: rand != 0 needs the noise array [(max_iter + 1), num_agents, action_dim]", what);
  GCBF_REQUIRE(g->states && g->x && g->rowptr && g->u_ref && d->goal && (g->num_edges == 0 || (g->edge_attr && g->edge_index)), "%s: null pointer", what);
  const size_t need = apply_workspace(d, g, what);
  if (need == 0) return GCBF_E_INVALID;
  if (need > workspace_bytes) { set_error("%s: workspace too small (%zu needed, %zu given)", what, need, workspace_bytes); return GCBF_E_WORKSPACE; }
  if (!g_pinned_count) GCBF_CUDA_OK(cudaHostAlloc(&g_pinned_count, 64, cudaHostAllocDefault));
  return 0;
}

extern "C" size_t gcbf_apply_workspace_bytes(const gcbf_step_desc* d, const gcbf_step_batch* g) {
  return apply_workspace(d, g, "gcbf_apply_workspace_bytes");
}

extern "C" int gcbf_apply(const gcbf_step_desc* d, const gcbf_step_batch* g, float lr, float rand, const float* noise, int max_iter,
                          float* action, int ld_action, int* iterations, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_step(d, g, "gcbf_apply")) return rc;
  GCBF_REQUIRE(d->env.num_graphs == 1 && !d->goal_per_graph, "gcbf_apply: one graph per call (gcbf.py:260 takes a single Data)");
  if (int rc = apply_check(d, g, lr, rand, noise, max_iter, action, ld_action, workspace, workspace_bytes, "gcbf_apply")) return rc;
  Run R(workspace, workspace_bytes, as_stream(stream), false);
  int rc = apply_run(R, *d, *g, lr, rand, rand != 0.f ? noise : nullptr, max_iter, action, ld_action, nullptr, iterations, "gcbf_apply");
  return R.finish(rc, "gcbf_apply");
}

extern "C" size_t gcbf_apply_batch_workspace_bytes(const gcbf_step_desc* d, const gcbf_step_batch* batch) {
  return apply_workspace(d, batch, "gcbf_apply_batch_workspace_bytes");
}

extern "C" int gcbf_apply_batch(const gcbf_step_desc* d, const gcbf_step_batch* batch, float lr, float rand, const float* noise, int max_iter,
                                float* action, int ld_action, int32_t* rounds, int* iterations, void* workspace, size_t workspace_bytes,
                                void* stream) {
  if (int rc = check_step(d, batch, "gcbf_apply_batch")) return rc;      // num_agents_total / num_nodes against num_graphs x the per-graph sizes
  GCBF_REQUIRE(rounds, "gcbf_apply_batch: rounds (device int32[num_graphs]) is required");
  if (int rc = apply_check(d, batch, lr, rand, noise, max_iter, action, ld_action, workspace, workspace_bytes, "gcbf_apply_batch")) return rc;
  Run R(workspace, workspace_bytes, as_stream(stream), false);
  int rc = apply_run(R, *d, *batch, lr, rand, rand != 0.f ? noise : nullptr, max_iter, action, ld_action, rounds, iterations, "gcbf_apply_batch");
  return R.finish(rc, "gcbf_apply_batch");
}
