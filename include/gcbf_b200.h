/*
 * gcbf_b200.h -- C ABI of libgcbf_b200.so: the H100 (sm_90a) hot path of MIT-REALM/gcbf-pytorch.
 *
 * The reference has no FFI of its own (it is pure Python on torch / torch_geometric); the boundary a
 * maintainer binds is therefore the set of tensor operations its Python classes perform.  Every entry
 * below names the reference site (file:line, relative to the reference checkout) it replaces.
 *
 * Conventions
 *   - plain pointers and sizes only; all pointers are DEVICE pointers unless the name ends in `_host`;
 *   - all matrices are dense row-major fp32 with an explicit leading dimension (`ld*`, in elements);
 *     edge_index is int64 [2, E] (row 0 = source j, row 1 = target i), masks are uint8;
 *   - nothing here synchronises, and outputs / workspaces are caller-provided; every launch goes to `stream` (a cudaStream_t
 *     passed as void*).  Reductions over many blocks (split-K weight gradients, column sums, the train step's edge-feature VJP)
 *     write per-block partials to short-lived scratch taken from the library's own stream-ordered memory pool (cudaMallocAsync
 *     semantics, freed on `stream`, cached in the pool) and sum them in a fixed order, so results are run-to-run reproducible.
 *     That scratch (up to a few tens of MB at the largest configurations) is NOT counted by the *_workspace_bytes queries;
 *     an allocation failure is reported as GCBF_E_CUDA;
 *   - return value: 0 on success, negative GCBF_E_* on failure; gcbf_last_error() gives the text;
 *   - per-kernel entry points are thread-compatible (no global mutable state except the per-thread last-error string); the
 *     chain-level entry points of ABI v3 keep per-process state (seven CUDA events and one pinned word per device for the train
 *     step's streams, the instrumentation records, the gemm-implementation switch) and must be driven from one host thread per
 *     process -- the deployment model is one process per GPU.
 */
#ifndef GCBF_B200_H
#define GCBF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define GCBF_OK 0
#define GCBF_E_INVALID (-1) /* bad argument (null pointer, negative size, unsupported enum) */
#define GCBF_E_CUDA (-2)    /* a CUDA runtime call / launch failed */
#define GCBF_E_UNSUPPORTED (-3)

/* environment kinds: gcbf/env/__init__.py:11-26 */
#define GCBF_ENV_SIMPLE_CAR 0   /* gcbf/env/simple_car.py  : state [x,y,vx,vy],       edge_dim 4, action 2 */
#define GCBF_ENV_DUBINS_CAR 1   /* gcbf/env/dubins_car.py  : state [x,y,theta,v],     edge_dim 5, action 2 */
#define GCBF_ENV_SIMPLE_DRONE 2 /* gcbf/env/simple_drone.py: state [x,y,z,vx,vy,vz], edge_dim 6, action 3 */

/* activation codes for the linear epilogue: gcbf/nn/mlp.py:44-47 (ReLU hidden), gcbf/algo/gcbf.py:34 (Tanh) */
#define GCBF_ACT_NONE 0
#define GCBF_ACT_RELU 1
#define GCBF_ACT_TANH 2

const char* gcbf_last_error(void);
int gcbf_abi_version(void);
/* sizeof() of ABI structure number `which` as the library was compiled (0 gcbf_env_cfg, 1 gcbf_linear_desc, 2 gcbf_net_desc,
 * 3 gcbf_step_desc, 4 gcbf_step_batch, 5 gcbf_step_out, 6 gcbf_net_ctx, 7 gcbf_mlp_ctx, 8 gcbf_step_ctx, 9 gcbf_time_rec,
 * 10 gcbf_sn_layer, 11 gcbf_split_desc, 12 gcbf_h16, 13 gcbf_field_desc, 14 gcbf_reset_desc; 0 for unknown): bindings check their
 * mirrors against it */
size_t gcbf_abi_struct_size(int which);
/* 1 if the library was built with the wgmma (3xFP16) GEMM path compiled in, else 0 (ABI v5: was gcbf_has_tcgen05) */
int gcbf_has_wgmma(void);
/* which kernel the most recent gcbf_linear_* call on this thread launched: 1 = fp32 SIMT tile GEMM,
 * 3 = fp32 skinny-K stream kernel (in-features <= 16), 4 = row-streaming kernel (out-features <= 32), 5 = few-rows kernels
 * (M <= 64: rollout-time single-graph passes stream the weights instead of tiling the output).  (The wgmma path
 * has its own entry points, gcbf_linear_*_h.) */
int gcbf_last_gemm_impl(void);

/* ---------------------------------------------------------------------------------------------------
 * K1  radius graph.  Replaces SimpleCar.add_communication_links -> torch_cluster.radius_graph
 * (gcbf/env/simple_car.py:32-33, 249-252; metric 0: sum_d (dx_d)^2 < r*r, unfused) and the dense
 * torch.norm / nonzero build of DubinsCar / SimpleDrone (gcbf/env/dubins_car.py:730-746,
 * gcbf/env/simple_drone.py:316-333; metric 1: sqrt(fma-chain) < r, matching torch.norm on CPU).
 * A batch is `num_graphs` graphs of `nodes_per_graph` rows each, agents first; targets are the first
 * `num_agents` rows of every graph, sources all rows (SimpleCar: pass nodes_per_graph == num_agents).
 * `count` writes rowptr[num_graphs*num_agents + 1] (int32 exclusive scan, agent-major); rowptr[last]
 * is E.  `fill` writes edge_index[2,E] int64 sorted (target asc, source asc) with batch node offsets
 * (what Batch.from_data_list produces, gcbf/algo/gcbf.py:159,200).
 * ------------------------------------------------------------------------------------------------- */
int gcbf_radius_graph_count(const float* states, int ld_state, int pos_dim, int num_graphs,
                            int nodes_per_graph, int num_agents, float radius, int metric,
                            int32_t* rowptr, void* stream);
int gcbf_radius_graph_fill(const float* states, int ld_state, int pos_dim, int num_graphs,
                           int nodes_per_graph, int num_agents, float radius, int metric,
                           const int32_t* rowptr, int64_t* edge_index, int64_t num_edges, void* stream);
/* CSR row pointer over ALL nodes from a target-sorted edge_index row (the `index` PyG's
 * MessagePassing hands to the aggregation, gcbf/nn/gnn.py:28).  unsorted_flag (device int32) is cleared,
 * then set to 1 if targets are out of range or not non-decreasing (caller must then sort).  rowptr has
 * num_nodes+1 int32 entries. */
int gcbf_rowptr_from_targets(const int64_t* edge_dst, int64_t num_edges, int num_nodes, int32_t* rowptr,
                             int32_t* unsorted_flag, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * K2  edge features.  edge_attr = g(s[src]) - g(s[dst]); g = identity (SimpleCar, SimpleDrone:
 * simple_car.py:246-247, simple_drone.py:313-314) or [x,y,theta,v cos,v sin] (dubins_car.py:724-728).
 * bwd accumulates (atomicAdd, so the summation order varies between runs) into d_states, which the caller zero-initialises;
 * the chain-level train step and gcbf_apply use an ordered per-node sum instead.
 * edge_input builds cat([x_i, x_j, edge_attr]) (gnn.py:31, :68) into rows of leading dim ld_out,
 * zero-filling the columns past 2*node_dim+edge_dim.
 * ------------------------------------------------------------------------------------------------- */
int gcbf_edge_attr_fwd(int env, const float* states, int ld_state, const int64_t* edge_index,
                       int64_t num_edges, float* edge_attr, void* stream);
int gcbf_edge_attr_bwd(int env, const float* states, int ld_state, const int64_t* edge_index,
                       int64_t num_edges, const float* d_edge_attr, float* d_states, void* stream);
int gcbf_edge_input_fwd(const float* x, int node_dim, const float* edge_attr, int edge_dim,
                        const int64_t* edge_index, int64_t num_edges, float* out, int ld_out, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * K3  linear layers of gcbf.nn.MLP (gcbf/nn/mlp.py:44-47).  inv_sigma is a device scalar (1/sigma of
 * the spectral-normalised layer, mlp.py:21,33) or NULL for 1.
 *   fwd       : Y[M,N]  = act(inv_sigma * X[M,K] W[N,K]^T + bias[N])
 *   bwd_data  : dX[M,K] (+)= inv_sigma * dZ[M,N] W[N,K]   (* (relu_src[M,K] > 0) if relu_src != NULL)
 *   bwd_weight: dW[N,K] (+)= inv_sigma * dZ[M,N]^T X[M,K] ; db[N] (+)= colsum(dZ)   (db may be NULL)
 *               accumulate != 0 adds into dW/db, otherwise they are overwritten.
 * impl: 0 = auto (skinny-K stream kernels when in-features <= 16, row-streaming kernels when out-features <= 32,
 * else the SIMT tile kernel), 1 = fp32 SIMT tile kernel.  fwd's out_amax (optional device uint32) receives the float bits
 * of max|Y| (for the fp16 split when the next layer runs on the tensor cores).
 * ------------------------------------------------------------------------------------------------- */
int gcbf_linear_fwd(const float* X, int ldx, const float* W, int ldw, const float* bias,
                    const float* inv_sigma, float* Y, int ldy, int M, int N, int K, int act, int impl,
                    void* out_amax, void* stream);
int gcbf_linear_bwd_data(const float* dZ, int lddz, const float* W, int ldw, const float* inv_sigma,
                         const float* relu_src, int ld_relu, float* dX, int lddx, int M, int N, int K,
                         int accumulate, int impl, void* stream);
int gcbf_linear_bwd_weight(const float* dZ, int lddz, const float* X, int ldx, const float* inv_sigma,
                           float* dW, int lddw, float* db, int M, int N, int K, int accumulate, int impl,
                           void* stream);
/* ---------------------------------------------------------------------------------------------------
 * K3 on the tensor cores (wgmma + TMA + mbarrier, csrc/gemm_wgmma_f16.cu): the same three products with
 * error-compensated 3xFP16 arithmetic (fp32-grade: 22 significand bits per operand, fp32 accumulation).
 * Operands are "companions": for an fp32 matrix X[rows, cols] the caller provides a device buffer of
 * 2*rows*ld_h halves (ld_h a multiple of 8, 16-byte aligned) that gcbf_split_f16 fills with the planes
 * hi = fp16(X*s), lo = fp16(X*s - hi) in X's own row-major layout; s is the power of two that puts
 * max|X| (device uint32 slot holding its float bits, from gcbf_amax_f32 or a producer's out_amax) into
 * [2^14, 2^15).  One companion serves every product the matrix is in (the tensor core reads it K-major
 * or MN-major), so nothing is transposed or padded:
 *   fwd_h       : Y  = act(inv_sigma * X W^T + bias)        X[M,K], W[N,K] companions
 *   bwd_data_h  : dX (+)= inv_sigma * dZ W (* relu mask)    dZ[M,N], W[N,K] companions
 *   bwd_weight_h: dW (+)= inv_sigma * dZ^T X                dZ[M,N], X[M,K] companions
 * out_amax (optional, may be NULL): the epilogue atomically maxes |output| into it (zeroed first), which
 * saves the amax pass when the output feeds the next layer's split.  gcbf_split_f16's `colsum`
 * (optional) receives the column sums of the source = the bias gradient when the source is dZ
 * (colsum_accumulate != 0: added to what is there, e.g. the bias's .grad; else overwritten).
 * ------------------------------------------------------------------------------------------------- */
int gcbf_amax_f32(const float* src, int ld, int rows, int cols, void* amax_slot, int accumulate, void* stream);
int gcbf_split_f16(const float* src, int ld, int rows, int cols, const void* amax_slot, void* dst, int ld_h,
                   float* colsum, int colsum_accumulate, void* stream);
/* amax + split of `count` matrices (HOST array of descriptors, device pointers inside) in two launches per 16 matrices:
 * the weights of a net after an optimizer step.  Bit-identical to gcbf_amax_f32 + gcbf_split_f16 per matrix. */
typedef struct gcbf_split_desc {
  const float* src; int32_t ld; int32_t rows; int32_t cols; int32_t ld_h; void* amax_slot; void* dst;
} gcbf_split_desc;
int gcbf_amax_split_batched(const gcbf_split_desc* descs, int count, void* stream);
int gcbf_linear_h_supported(int M, int N, int K);
int gcbf_linear_fwd_h(const void* Xh, int ldxh, const void* x_amax, const void* Wh, int ldwh, const void* w_amax,
                      const float* bias, const float* inv_sigma, float* Y, int ldy, int M, int N, int K, int act,
                      void* out_amax, void* stream);
int gcbf_linear_bwd_data_h(const void* dZh, int lddzh, const void* dz_amax, const void* Wh, int ldwh,
                           const void* w_amax, const float* inv_sigma, const float* relu_src, int ld_relu,
                           float* dX, int lddx, int M, int N, int K, int accumulate, void* out_amax, void* stream);
int gcbf_linear_bwd_weight_h(const void* dZh, int lddzh, const void* dz_amax, const void* Xh, int ldxh,
                             const void* x_amax, const float* inv_sigma, float* dW, int lddw, int M, int N, int K,
                             int accumulate, void* stream);
/* The general form of the three products (ABI v3): operands are `gcbf_h16` descriptors whose scale is either one word per tensor
 * (amax strides 0, what gcbf_split_f16 makes) or one word per (128-row, 256-column) tile of the matrix (amax[rb * amax_row_stride +
 * ct * amax_col_stride]) -- the format the EPILOGUES emit: a forward / data-grad launch can write its output directly as a tile-
 * scaled companion (Yh / dXh, output width > 128), because every CTA knows the exact maximum of its own 128 x 256 tile.  That
 * removes the amax + split passes (and the fp32 round trip through HBM) for every hidden activation / gradient between two
 * tensor-core layers.  Y / dX may be NULL when only the companion is wanted.  data-grad extras: the ReLU mask can be read from
 * the hi plane of the layer output's companion (relu_h; y > 0 <=> hi > 0), and `colsum` (optional) accumulates (per-row-tile partials summed in a fixed order) the
 * column sums of the masked output (= the bias gradient of the layer below).  Weight companions stay per-tensor. */
typedef struct gcbf_h16 {
  void* buf;                /* hi plane [rows][ld] halves, lo plane at buf + rows * ld halves */
  void* amax;               /* uint32 float bits of max|x|: per tensor, or per tile */
  int32_t ld, rows, cols;
  int32_t amax_row_stride;  /* words between the rows of the tile-maxima array (0: per-tensor) */
  int32_t amax_col_stride;  /* 1 for a tile-scaled companion, 0 per-tensor */
  int32_t pad_;
} gcbf_h16;
int gcbf_linear_fwd_t(const gcbf_h16* X, const gcbf_h16* W, const float* bias, const float* inv_sigma, int act, float* Y, int ldy,
                      const gcbf_h16* Yh, void* out_amax, int M, int N, int K, void* stream);
int gcbf_linear_bwd_data_t(const gcbf_h16* dZ, const gcbf_h16* W, const float* inv_sigma, const float* relu_src, int ld_relu,
                           const gcbf_h16* relu_h, float* dX, int lddx, int accumulate, const gcbf_h16* dXh, float* colsum,
                           void* out_amax, int M, int N, int K, void* stream);
int gcbf_linear_bwd_weight_t(const gcbf_h16* dZ, const gcbf_h16* X, const float* inv_sigma, float* dW, int lddw, int accumulate,
                             int M, int N, int K, void* stream);
/* the skinny-K fp32 forward (in-features <= 16: the first phi layer, gnn.py:31) writing ONLY the tile-scaled companion of its output
 * (each 128 x 256 tile is computed twice: once for its exact maximum, once to convert and store) */
int gcbf_linear_fwd_emit(const float* X, int ldx, const float* W, int ldw, const float* bias, const float* inv_sigma, int act,
                         const gcbf_h16* Yh, int M, int N, int K, void* stream);
/* dZ = dY * act'(Y) for the output activation (tanh: 1 - Y^2; relu: Y > 0).  In place allowed. */
int gcbf_act_bwd(const float* dY, const float* Y, float* dZ, int64_t count, int act, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * K4  attention aggregation = torch_geometric AttentionalAggregation as used at gcbf/nn/gnn.py:17-19,
 * 59-60: att = softmax over the in-edges of each target (max-shifted, denominator + 1e-16),
 * aggr_i = sum_e att_e * msg_e (zero for nodes without in-edges).  Edges of node i are the contiguous
 * range rowptr[i]..rowptr[i+1]; one warp per node, shuffle reductions, no atomics.
 *   fwd: msg[E,C], gate[E] -> att[E], aggr rows (leading dim ld_aggr, C columns written)
 *   bwd: d_aggr -> d_msg[E,C] (overwritten, or added to if accumulate != 0), d_gate[E]
 * ------------------------------------------------------------------------------------------------- */
int gcbf_attn_aggr_fwd(const float* msg, int ld_msg, const float* gate, const int32_t* rowptr,
                       int num_nodes, int channels, float* att, float* aggr, int ld_aggr, void* stream);
int gcbf_attn_aggr_bwd(const float* msg, int ld_msg, const float* att, const int32_t* rowptr,
                       int num_nodes, int channels, const float* d_aggr, int ld_daggr, float* d_msg,
                       int ld_dmsg, float* d_gate, int accumulate, void* stream);
/* row gather / scatter by index: the `x[data.agent_mask]` selection of gcbf/algo/gcbf.py:52-53 and
 * gcbf/controller/gnn_controller.py:44-45 (idx = nonzero(agent_mask), int64).
 *   gather : dst[r, 0:cols] = src[idx[r], 0:cols]         r < rows
 *   scatter: dst[idx[r], 0:cols] = src[r, 0:cols]          (adjoint; caller zero-fills dst, idx unique) */
int gcbf_rows_gather(const float* src, int ld_src, const int64_t* idx, float* dst, int ld_dst, int64_t rows,
                     int cols, void* stream);
int gcbf_rows_scatter(const float* src, int ld_src, const int64_t* idx, float* dst, int ld_dst, int64_t rows,
                      int cols, void* stream);
/* strided 2-D copy dst[r, 0:cols] = src[r, 0:cols] (concats such as cat([aggr, x]), cat([feat, u_ref])) */
int gcbf_copy2d(const float* src, int ld_src, float* dst, int ld_dst, int64_t rows, int cols, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * K5  nominal controller + one finite-difference step.
 *   u_ref : simple_car.py:270-304 (LQR + over-speed penalty), dubins_car.py:764-816 (PID),
 *           simple_drone.py:349-377.  goal is [num_agents, goal_dim] shared by all graphs; K is the
 *           LQR gain [action_dim, state_dim] (NULL for DubinsCar).
 *   step  : forward_graph + MultiAgentEnv.forward + dynamics: x+ = x + dt f(x, clamp(u + u_ref(x)))
 *           (simple_car.py:178-194,78-89; dubins_car.py:617-635,110-132; simple_drone.py:236-253,103-120;
 *           gcbf/env/base.py:381-398).  `freeze` != 0 reproduces the single-graph reach-freeze branch.
 *           pass_mask[num_agents_total, action_dim] (uint8) records where the clamp passes gradient
 *           (and is 0 for agents frozen by the reach test).
 *   step_bwd: d_action = (d x+ / d u)^T d_states_next, masked by pass_mask.
 * ------------------------------------------------------------------------------------------------- */
/* Environment description shared by K5/K6.  The doubles are the reference's python-float parameters
 * (`default_params`, simple_car.py:67-76, dubins_car.py:88-100, simple_drone.py:71-82); thresholds such as
 * 4*car_radius are formed in double and then rounded to fp32 exactly as torch does with python scalars. */
typedef struct gcbf_env_cfg {
  int32_t env;             /* GCBF_ENV_* */
  int32_t num_graphs;      /* B */
  int32_t nodes_per_graph; /* N = agents + obstacles (agents first) */
  int32_t num_agents;      /* n */
  double agent_radius;     /* car_radius / drone_radius */
  double speed_limit;
  double dist2goal;
  double dt;
} gcbf_env_cfg;

int gcbf_u_ref(const gcbf_env_cfg* cfg, const float* states, int ld_state, const float* goal, int ld_goal,
               const float* K, float* u_ref, void* stream);
int gcbf_step_fwd(const gcbf_env_cfg* cfg, const float* states, int ld_state, const float* action,
                  const float* goal, int ld_goal, const float* K, int freeze, float* states_next,
                  uint8_t* pass_mask, void* stream);
int gcbf_step_bwd(const gcbf_env_cfg* cfg, const float* d_states_next, int ld_state,
                  const uint8_t* pass_mask, float* d_action, void* stream);
/* the same two with ONE GOAL SET PER GRAPH, goal [num_graphs * num_agents, ld_goal]: many independent environments (each with
 * its own goals) stepped as one batch -- the vectorised rollout of gcbf/trainer/trainer.py:60-70 + gcbf/algo/gcbf.py:128-139 */
int gcbf_u_ref_multi(const gcbf_env_cfg* cfg, const float* states, int ld_state, const float* goal, int ld_goal,
                     const float* K, float* u_ref, void* stream);
int gcbf_step_fwd_multi(const gcbf_env_cfg* cfg, const float* states, int ld_state, const float* action,
                        const float* goal, int ld_goal, const float* K, int freeze, float* states_next,
                        uint8_t* pass_mask, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * K6  safe / unsafe masks and the CBF losses.
 *   masks: simple_car.py:306-370, dubins_car.py:818-882, simple_drone.py:379-444 (per-env constants kept).
 *   loss_partials: local sums for gcbf/algo/gcbf.py:168-212 -> partial[16] (see GCBF_LP_* indices);
 *                  hdot_out (optional) receives the h_dot values of gcbf.py:202-205.
 *   loss_grads   : with (possibly all-reduced) partials, d loss / d h, d h_next, d actions of
 *                  gcbf.py:215-218, and the four loss values + accuracies -> scalars[8].
 *   pair_count   : number of (i, j) with hdot[j] + alpha*h[i] >= 0 -- the M x M broadcast of gcbf.py:209.
 * ------------------------------------------------------------------------------------------------- */
int gcbf_masks(const gcbf_env_cfg* cfg, const float* states, int ld_state, uint8_t* safe, uint8_t* unsafe,
               uint8_t* collision /* optional: collision_mask, simple_car.py:372-387 */, void* stream);
#define GCBF_LP_SUM_UNSAFE 0
#define GCBF_LP_CNT_UNSAFE 1
#define GCBF_LP_OK_UNSAFE 2
#define GCBF_LP_SUM_SAFE 3
#define GCBF_LP_CNT_SAFE 4
#define GCBF_LP_OK_SAFE 5
#define GCBF_LP_SUM_HDOT 6
#define GCBF_LP_CNT_ALL 7
#define GCBF_LP_SUM_ACT 8
#define GCBF_LP_SIZE 16
int gcbf_loss_partials(const float* h, const float* h_next, const float* h_next_new, const float* action,
                       int action_dim, const uint8_t* safe, const uint8_t* unsafe, int64_t num_agents_total,
                       float alpha, float eps, float dt, double* partial, float* hdot_out, void* stream);
int gcbf_loss_grads(const float* h, const float* h_next, const float* h_next_new, const float* action,
                    int action_dim, const uint8_t* safe, const uint8_t* unsafe, int64_t num_agents_total,
                    float alpha, float eps, float dt, float coef_unsafe, float coef_safe, float coef_hdot,
                    float coef_action, const double* partial, float* d_h, float* d_h_next, float* d_action,
                    float* scalars, void* stream);
int gcbf_pair_count(const float* hdot, int64_t m_cols, const float* h, int64_t m_rows, float alpha,
                    unsigned long long* count, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * K7  spectral norm (old-style torch.nn.utils.spectral_norm, training mode, 1 power iteration,
 * eps 1e-12; reached from gcbf/nn/mlp.py:21,33 on EVERY forward): v <- normalize(W^T u),
 * u <- normalize(W v), inv_sigma <- 1 / (u . W v).  u, v updated in place.  workspace: >= (rows_split*K
 * + N + 8) floats, see gcbf_sn_workspace_floats.
 *   sn_grad_fixup: given dW = dL/d(W/sigma) / sigma (what bwd_weight produced with inv_sigma), subtract
 *   the term through sigma: dW -= <dW, W> * inv_sigma * u v^T.
 * ------------------------------------------------------------------------------------------------- */
size_t gcbf_sn_workspace_floats(int N, int K);
int gcbf_sn_power_iter(const float* W, int ldw, int N, int K, float* u, float* v, float* inv_sigma,
                       float* workspace, void* stream);
/* every spectral-normalised layer of a net in four launches: same arithmetic per layer as gcbf_sn_power_iter
 * (bit-identical u, v, 1/sigma).  `layers` is a HOST array of `count` descriptors (device pointers inside);
 * workspace_floats >= sum of gcbf_sn_workspace_floats(N, K) over the layers. */
typedef struct gcbf_sn_layer {
  const float* W; int32_t ldw; int32_t N; int32_t K; int32_t pad_; float* u; float* v; float* inv_sigma;
} gcbf_sn_layer;
int gcbf_sn_power_iter_batched(const gcbf_sn_layer* layers, int count, float* workspace, size_t workspace_floats,
                               void* stream);
/* acc == NULL: dW is corrected in place; otherwise the corrected gradient is added to acc[N, K] (pitch ldacc, e.g. the
 * parameter's .grad view) and dW is left untouched. */
int gcbf_sn_grad_fixup(float* dW, int lddw, const float* W, int ldw, int N, int K, const float* u,
                       const float* v, const float* inv_sigma, float* workspace, float* acc, int ldacc, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * K8  clip_grad_norm_(max_norm) + Adam on one flat parameter bucket (gcbf/algo/gcbf.py:102-103,
 * 220-226): sumsq[0] += sum g^2 (double);  then p, m, v updated with g * min(1, max_norm/(sqrt(sumsq)+1e-6)).
 * ------------------------------------------------------------------------------------------------- */
int gcbf_grad_sumsq(const float* g, int64_t count, double* sumsq, void* stream);
int gcbf_clip_adam(float* p, const float* g, float* m, float* v, int64_t count, const double* sumsq,
                   double max_norm, double lr, double beta1, double beta2, double eps, int step, void* stream);


/* ===================================================================================================
 * Chain-level entry points (ABI v3): ONE call per GNN pass / per phase of the train step instead of one per kernel.
 * The host-side sequencing that gcbf/nn/gnn.py:27-36, gcbf/nn/mlp.py:44-47 and gcbf/algo/gcbf.py:158-226 do with ~250 ATen
 * calls per forward lives in the library (csrc/net.cu, csrc/step.cu); the caller still owns every byte: it passes ONE
 * workspace per call (size from the matching *_workspace_bytes query), the library bump-allocates activations, companions
 * and gradients inside it and never allocates device memory itself.
 * =================================================================================================== */
#define GCBF_E_WORKSPACE (-4) /* workspace too small: the needed size is returned through the call's out-parameter */

/* one nn.Linear of a gcbf.nn.MLP (gcbf/nn/mlp.py:17-41) */
typedef struct gcbf_linear_desc {
  const float* W; const float* b;   /* weight [N, K] (weight_orig when spectral-normalised), pitch ldw; bias [N] */
  float* u; float* v;               /* spectral-norm buffers weight_u [N], weight_v [K] (updated in place by every forward) or NULL */
  float* gW; float* gb;             /* where the backward ACCUMULATES dL/dW (pitch ldgw) and dL/db; NULL = no weight gradient */
  void* Wh; void* w_amax;           /* persistent fp16 [hi|lo] companion of W (2*N*ldwh halves) + its amax word; NULL = never on tensor cores */
  int32_t ldw, ldgw, ldwh;
  int32_t N, K, act;                /* out-features, in-features, GCBF_ACT_* applied to this layer's output */
} gcbf_linear_desc;

#define GCBF_MAX_MLP_LAYERS 4
/* CBFGNNLayer / ControllerGNNLayer (gcbf/nn/gnn.py:14-36, 56-73) + optional row selection + head MLP
 * (CBFGNN.forward gcbf/algo/gcbf.py:37-55, GNNController.forward gcbf/controller/gnn_controller.py:29-48) */
typedef struct gcbf_net_desc {
  gcbf_linear_desc phi[GCBF_MAX_MLP_LAYERS], gate[GCBF_MAX_MLP_LAYERS], gamma[GCBF_MAX_MLP_LAYERS], head[GCBF_MAX_MLP_LAYERS];
  int32_t n_phi, n_gate, n_gamma, n_head;   /* n_head == 0: the pass ends with gamma's output */
  int32_t node_dim, edge_dim, phi_dim;
  int32_t head_extra_dim;                   /* columns concatenated to gamma's output before the head (u_ref: action_dim), or 0 */
  int32_t refresh_weights;                  /* != 0: the weights changed since the companions were made -> re-split them first */
  int32_t pad_;
} gcbf_net_desc;

/* what a forward saves for its backward: pointers into the forward's workspace (which must stay alive and untouched) */
typedef struct gcbf_net_ctx { uint64_t opaque[208]; } gcbf_net_ctx;

/* bytes a forward (save_ctx != 0: everything the backward reads is kept) / a backward needs for E edges, num_nodes nodes,
 * `rows` gamma rows (= num_nodes without row selection) */
size_t gcbf_net_forward_workspace_bytes(const gcbf_net_desc* net, int64_t num_edges, int num_nodes, int rows, int save_ctx);
size_t gcbf_net_backward_workspace_bytes(const gcbf_net_desc* net, int64_t num_edges, int num_nodes, int rows, int need_d_edge_attr);
/* out[rows, out_dim] (pitch ld_out) = head(gamma(cat[aggr, x])[row_index] ++ head_extra); row_index (int64[rows]) NULL = all nodes.
 * ctx NULL = inference (nothing kept).  Advances the spectral-norm buffers by one power iteration (the reference never calls
 * .eval(), SURVEY 3.5). */
int gcbf_net_forward(const gcbf_net_desc* net, const float* x, const float* edge_attr, const int64_t* edge_index,
                     const int32_t* rowptr, int64_t num_edges, int num_nodes, const int64_t* row_index, int rows,
                     const float* head_extra, float* out, int ld_out, void* workspace, size_t workspace_bytes,
                     gcbf_net_ctx* ctx, void* stream);
/* accumulates weight / bias gradients into the descriptors' gW / gb (skipped where NULL or when skip_wgrad != 0) and writes
 * d_edge_attr [E, edge_dim] if it is not NULL */
int gcbf_net_backward(const gcbf_net_desc* net, const gcbf_net_ctx* ctx, const float* d_out, int ld_dout, float* d_edge_attr,
                      int skip_wgrad, void* workspace, size_t workspace_bytes, void* stream);
/* a bare MLP (gcbf.nn.MLP.forward, mlp.py:44-47) through the same chain code */
typedef struct gcbf_mlp_ctx { uint64_t opaque[64]; } gcbf_mlp_ctx;
size_t gcbf_mlp_forward_workspace_bytes(const gcbf_linear_desc* layers, int n_layers, int rows, int save_ctx);
size_t gcbf_mlp_backward_workspace_bytes(const gcbf_linear_desc* layers, int n_layers, int rows);
int gcbf_mlp_forward(const gcbf_linear_desc* layers, int n_layers, int refresh_weights, const float* x, int ldx, int rows,
                     float* out, int ld_out, void* workspace, size_t workspace_bytes, gcbf_mlp_ctx* ctx, void* stream);
int gcbf_mlp_backward(const gcbf_linear_desc* layers, int n_layers, const gcbf_mlp_ctx* ctx, const float* d_out, int ld_dout,
                      float* d_x /* [rows, K0] or NULL */, int skip_wgrad, void* workspace, size_t workspace_bytes, void* stream);

/* One inner iteration of GCBF.update (gcbf/algo/gcbf.py:158-226) in three calls, so that data-parallel callers can put
 * their two collectives in between (loss partial sums after `relink`, gradient bucket after `backward`):
 *   gcbf_step_forward : h = cbf(graphs), actions = actor(graphs) (side stream), masks, forward_graph, h_next = cbf(graphs_next);
 *                       starts the re-linked radius graph on the side stream
 *   gcbf_step_relink  : waits for the re-linked edge count (the step's ONE host sync), h_next_new = cbf(re-linked graphs),
 *                       loss partial sums -> partial[16]; returns GCBF_E_WORKSPACE (+ *needed_bytes) BEFORE launching anything
 *                       if workspace2 is too small for the re-linked graph -- call again with a larger one
 *   gcbf_step_backward: loss gradients from the (all-reduced) partials, the three backward passes, scalars[8]
 * All device results live in the caller's workspaces; `out` reports where. */
typedef struct gcbf_step_desc {
  gcbf_net_desc cbf, actor;
  gcbf_env_cfg env;
  const float* goal; const float* lqr_gain;     /* goal [num_agents, ld_goal] (or [num_graphs * num_agents, ld_goal] with goal_per_graph); LQR gain or NULL (DubinsCar) */
  int32_t ld_goal, state_dim, pos_dim, action_dim;
  int32_t graph_metric;                          /* K1 metric: 0 SimpleCar, 1 DubinsCar / SimpleDrone */
  float comm_radius;
  float alpha, eps, coef_unsafe, coef_safe, coef_hdot, coef_action;
  float* grad_bucket; int64_t grad_bucket_floats;   /* zeroed by gcbf_step_backward before the gradients accumulate (NULL: caller zeroes) */
  int32_t goal_per_graph; int32_t pad_;             /* != 0: every graph of the batch has its own goal set (batches collected by vectorised rollouts) */
} gcbf_step_desc;

typedef struct gcbf_step_batch {
  const float* states; int32_t ld_state;       /* [B*N, state_dim] */
  const float* x;                              /* [B*N, node_dim] */
  const float* edge_attr;                      /* [E, edge_dim] */
  const int64_t* edge_index;                   /* [2, E] target-sorted */
  const int32_t* rowptr;                       /* CSR over all B*N nodes */
  const float* u_ref;                          /* [B*n, action_dim] (the STORED nominal control, gnn_controller.py:46) */
  const int64_t* row_index;                    /* agent rows (nonzero(agent_mask)) or NULL when every node is an agent */
  int64_t num_edges; int32_t num_nodes; int32_t num_agents_total;
} gcbf_step_batch;

typedef struct gcbf_step_out {   /* device pointers into the workspaces, valid until the workspaces are reused */
  float* h; float* actions; float* h_next; float* h_next_new; float* hdot; float* scalars;   /* [M,1] [M,a] [M,1] [M] [M] [8] */
  uint8_t* safe; uint8_t* unsafe;                                                        /* [M] each */
  double* partial;                                                                       /* [16] */
  int64_t* edge_index_new; int64_t num_edges_new;                                        /* re-linked graph [2, E'] */
} gcbf_step_out;

typedef struct gcbf_step_ctx { uint64_t opaque[800]; } gcbf_step_ctx;

size_t gcbf_step_workspace_bytes(const gcbf_step_desc* d, const gcbf_step_batch* b);            /* workspace (forward + backward) */
size_t gcbf_step_relink_workspace_bytes(const gcbf_step_desc* d, const gcbf_step_batch* b, int64_t num_edges_new);
int gcbf_step_forward(const gcbf_step_desc* d, const gcbf_step_batch* b, void* workspace, size_t workspace_bytes,
                      gcbf_step_ctx* ctx, gcbf_step_out* out, void* stream, void* side_stream /* NULL: single stream */);
int gcbf_step_relink(const gcbf_step_desc* d, const gcbf_step_batch* b, gcbf_step_ctx* ctx, void* workspace2,
                     size_t workspace2_bytes, size_t* needed_bytes, gcbf_step_out* out, void* stream, void* side_stream);
/* events (optional, 4 cudaEvent_t): recorded when a gradient range is final, so that a data-parallel caller can start its all-reduce
 * while the rest of the backward still runs: [0] cbf gamma + head, [1] all of cbf, [2] actor gamma + head, [3] all of actor */
int gcbf_step_backward(const gcbf_step_desc* d, const gcbf_step_batch* b, gcbf_step_ctx* ctx, gcbf_step_out* out, void* const* events,
                       void* stream, void* side_stream);

/* GCBF.apply, the test-time controller (gcbf/algo/gcbf.py:260-309; what gcbf/trainer/trainer.py:124 and test.py run), for ONE graph
 * (d->env.num_graphs == 1): the actor's action where the nominal zero action violates the h_dot condition, then up to max_iter + 1
 * rounds of forward_graph -> CBF -> d mean(relu(-h_dot - alpha h)) / d action and one Adam(lr) step per violating agent (the
 * reference's per-agent optimisers as one kernel), plus `action -= rand * lr * noise * grad` (gcbf.py:305) with the caller's standard
 * normals noise[(max_iter + 1), num_agents, action_dim] (NULL allowed when rand == 0).  Uses d->cbf, d->actor, d->env, goal / gain,
 * alpha, action_dim, state_dim; ignores the loss coefficients and the gradient bucket (no weight gradient is computed).  One host sync
 * per round (the violating-agent count, as the reference's `if loss_h_dot <= 0`).  action [num_agents, action_dim] (pitch ld_action);
 * *iterations (host, optional) = Adam rounds done. */
size_t gcbf_apply_workspace_bytes(const gcbf_step_desc* d, const gcbf_step_batch* graph);
int gcbf_apply(const gcbf_step_desc* d, const gcbf_step_batch* graph, float lr, float rand, const float* noise, int max_iter,
               float* action, int ld_action, int* iterations, void* workspace, size_t workspace_bytes, void* stream);
/* The same controller for d->env.num_graphs graphs of nodes_per_graph nodes each (agents first, edges inside the graphs, as the
 * radius-graph kernels make them) in one call: many evaluation episodes step at once.  Goals are shared, or one set per graph with
 * d->goal_per_graph.  noise [(max_iter + 1), num_agents_total, action_dim]: round k of graph g reads rows g*n .. g*n+n-1 of slice k,
 * so concatenated per-graph draws reproduce per-graph calls.  Per graph g the result is gcbf_apply on graph g alone: the mean in
 * the loss runs over g's n agents, Adam runs per agent, and g is done at the first round where none of its agents violates or the
 * round counter passed max_iter; from then on nothing of g changes (no Adam step, no noise, its flags are not re-evaluated), while
 * its rows keep going through the passes until the slowest graph is done.  rounds (device int32[num_graphs], required) = the Adam
 * rounds each graph did (gcbf_apply's *iterations for that graph); *iterations (host, optional) = those of the slowest graph.  Still
 * one host sync per round (the number of graphs still refining).  Spectral norm: the CBF passes run in the order of a single call
 * (h, actor, nominal h_next, one per round) and power iteration depends on the weights alone, so pass k uses the sigma of pass k
 * of a single call, and afterwards the CBF's u, v are those a single call on the slowest graph leaves. */
size_t gcbf_apply_batch_workspace_bytes(const gcbf_step_desc* d, const gcbf_step_batch* batch);
int gcbf_apply_batch(const gcbf_step_desc* d, const gcbf_step_batch* batch, float lr, float rand, const float* noise, int max_iter,
                     float* action, int ld_action, int32_t* rounds, int* iterations, void* workspace, size_t workspace_bytes, void* stream);

/* CBF level-set field: h of chosen agents over a grid of two state dimensions -- the data of plot_cbf_contour
 * (gcbf/trainer/utils.py:226-298, what plot_cbf.py draws), for B graphs and A agents in one call.
 * A probe t = ((b * num_probe_agents + ai) * ny + iy) * nx + ix is graph b's agent a = agents[ai] with state[x_dim] = xs[ix] and
 * state[y_dim] = ys[iy] (utils.py:262-267; xs, ys fp32, the rounding of the reference's write into its fp32 state tensor), everyone else
 * fixed; h[t] = CBFGNN(graph)[a] evaluated on that state (utils.py:268-273).  h_a depends only on a's in-edges and x_a, so instead of
 * n_mesh^2 copies of every graph each probe becomes one extra target node with its own in-edges (a "probe graph"):
 *   relink == 0  the in-edges of a in the given edge_index, in their order, with edge_attr = g(s_j) - g(s'_t) recomputed
 *                (the reference's fixed edge_index, utils.py:268-269; default);
 *   relink != 0  every node j != a of graph b inside the radius of s'_t under the K1 rule (metric / comm_radius as the radius graph:
 *                SimpleCar agents only, DubinsCar / SimpleDrone agents and obstacles), ascending j: the edges gcbf_radius_graph_*
 *                would give target a on the moved state.
 * The probes go through the CBF net (gcbf_net_forward's chain, GEMM dispatch unchanged) in chunks of at most max_probes probes and
 * max_edges probe edges (the workspace is sized for min(max_edges, chunk probes * (nodes_per_graph - 1)) edges); every chunk uses the 1/sigma of ONE spectral-norm power iteration done at the start of the call, so a call
 * advances the CBF's u, v exactly once, as the reference's single cbf(plot_data) does.  ONE host sync per call: the per-probe edge
 * counts are counted on the device for all probes and read back to split the probes into chunks (stream-ordered: the call returns
 * with the field still being computed).  max_edges must be < 2^31 and at least the largest probe's edge count (nodes_per_graph - 1
 * always suffices), else GCBF_E_INVALID.  Preconditions not checked on the device: agent ids in [0, num_agents), the given graph's
 * edge_index target-sorted with rowptr its CSR over all num_graphs * nodes_per_graph nodes (fixed mode).
 * gcbf_cbf_field_workspace_bytes: dry run of the call for these sizes (0 for an invalid descriptor); gcbf_cbf_field checks the size
 * before launching anything. */
typedef struct gcbf_field_desc {
  gcbf_net_desc cbf;                      /* the CBF net (n_head > 0, one output column) */
  gcbf_env_cfg env;                       /* env, num_graphs, nodes_per_graph, num_agents (the radii / dt are not used) */
  const float* states; const float* x;    /* [num_graphs * nodes_per_graph, ld_state], [.., node_dim] */
  const int64_t* edge_index; const int32_t* rowptr; int64_t num_edges;   /* the given graph (read in fixed mode only) */
  const int32_t* agents;                  /* [num_probe_agents] device int32, ids in [0, num_agents) */
  const float* xs; const float* ys;       /* [nx], [ny] device fp32 grid values */
  int64_t max_edges;                      /* probe-edge bound of a chunk */
  int32_t ld_state, state_dim, pos_dim, graph_metric;
  float comm_radius; int32_t relink;
  int32_t num_probe_agents, x_dim, y_dim, nx, ny;
  int32_t max_probes;                     /* probe bound of a chunk */
} gcbf_field_desc;
size_t gcbf_cbf_field_workspace_bytes(const gcbf_field_desc* d);
/* h [num_graphs * num_probe_agents * ny * nx] fp32; info (host int64[2], optional) = chunks the probes ran in, probe edges in all */
int gcbf_cbf_field(const gcbf_field_desc* d, float* h, int64_t* info, void* workspace, size_t workspace_bytes, void* stream);
/* The probe graphs themselves, for inspection (same two-call protocol and edge order as gcbf_radius_graph_count / _fill; d->cbf and the
 * chunk bounds are not read): count writes rowptr[T + 1] (int32 exclusive scan of the per-probe edge counts, T = num_graphs *
 * num_probe_agents * ny * nx; rowptr[T] is the total, which must stay below 2^31); fill writes edge_index [2, num_edges] with source =
 * the original node id (b * nodes_per_graph + j) and target = the probe id t, sorted (t asc, source asc), and edge_attr [num_edges,
 * edge_dim] = g(s_source) - g(s'_t).  These are the edges and features gcbf_cbf_field feeds the CBF. */
int gcbf_cbf_field_probe_count(const gcbf_field_desc* d, int32_t* rowptr, void* stream);
int gcbf_cbf_field_probe_fill(const gcbf_field_desc* d, const int32_t* rowptr, int64_t* edge_index, int64_t num_edges, float* edge_attr,
                              void* stream);

/* Batched episode reset of a vectorised rollout (num_envs copies of one env, nodes_per_graph = num_agents + num_obs rows each, agents
 * first): in ONE launch, every env e that is done -- step_count[e] >= max_steps, or (reach != NULL) all reach[e * num_agents + i] set,
 * the reference's `done` of env.step -- is re-sampled in place with the algorithm of that env's reset() (gcbf/env/<env>.py):
 *   SimpleCar    agents, then goals in [0, area]^2, each set with pairwise spacing > agent_dist / goal_dist;
 *   DubinsCar    num_obs obstacles [x, y, theta, v] uniform in [0, area]^2 x [0, 2 pi) x [0, obs_speed_limit); agents and goals as above
 *                and farther than the clearance from every obstacle; agent / goal headings uniform in [-pi, pi), speeds 0;
 *   SimpleDrone  num_obs static obstacles uniform in [0, area]^3; agents and goals as DubinsCar; velocities 0, goal columns past 3 zero.
 * Rejection rule: candidate c is rejected iff sum_d (p_d - c_d)^2 <= min_dist2 for a placed point p (clear2 for an obstacle), every
 * operation rounded on its own, d ascending.  The candidates of a point set are tried in order; a set whose first max_tries candidates
 * do not place all its points sets failed[e] (1 agents, 2 goals; 0 on success).  Random numbers: Philox4x32-10, key = seed, counter =
 * (draw index, first_env + e, new episode number, stream: 0 obstacles, 1 agents, 2 goals, 3 headings), uniform = (word >> 8) 2^-24;
 * a reset depends only on (seed, first_env + e, episode, stream, draw index).  A reset env gets step_count[e] = 0 and episode[e] + 1;
 * an env that is not done is left untouched.  No host sync; one warp and (num_agents + num_obs) * pos_dim floats of shared memory per env. */
typedef struct gcbf_reset_desc {
  uint64_t seed;
  float* states;              /* [num_envs * (num_agents + num_obs), ld_state] */
  float* goals;               /* [num_envs * num_agents, ld_goal]; columns [0, goal_dim) are written */
  int32_t* step_count;        /* [num_envs] device */
  int32_t* episode;           /* [num_envs] device: the current episode; a reset draws episode[e] + 1 */
  int32_t* failed;            /* [num_envs] device, written for every reset env */
  const uint8_t* reach;       /* [num_envs * num_agents] device, or NULL: done on the step counter alone */
  int32_t env, num_envs, num_agents, num_obs;
  int32_t ld_state, ld_goal, goal_dim, max_steps;
  int32_t max_tries, first_env;
  float area, agent_dist2, goal_dist2, clear2, obs_speed_limit, pad_;
} gcbf_reset_desc;
int gcbf_env_reset_batch(const gcbf_reset_desc* d, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * MACBF, the paper's baseline algorithm (gcbf/algo/macbf.py:20-239; SURVEY 8f-4): the kernels it needs beyond the ones above.
 * Its networks are small MLPs (gcbf/nn/gnn.py:82-135: per-edge CBF (8 + d_e) -> 64 -> 128 -> 64 -> 1; actor message
 * (8 + d_e) -> 64 -> 128, MAX aggregation, 128 -> 64 -> 128 -> 64 -> a, head 2a -> 512 -> 128 -> 32 -> a) and run on
 * gcbf_mlp_forward / gcbf_mlp_backward.
 *
 * Top-k filtered radius graph = `env.add_communication_links` of an env built with max_neighbors = k (train.py:30: k = 12):
 *   metric 1 (gcbf/env/dubins_car.py:730-746, simple_drone.py:316-333): edges to the k nearest nodes that are inside the radius
 *            (torch.topk on the distance row; equal distances: lower index first);
 *   metric 0 (gcbf/env/simple_car.py:32-33, 249-252): torch_cluster's cap -- the first k + 1 hits in ascending source index, the
 *            target itself included, self loop dropped.
 * Same two-call protocol and output order (target asc, source asc) as gcbf_radius_graph_count / _fill. */
int gcbf_radius_graph_topk_count(const float* states, int ld_state, int pos_dim, int num_graphs, int nodes_per_graph, int num_agents,
                                 float radius, int metric, int max_neighbors, int32_t* rowptr, void* stream);
int gcbf_radius_graph_topk_fill(const float* states, int ld_state, int pos_dim, int num_graphs, int nodes_per_graph, int num_agents,
                                float radius, int metric, int max_neighbors, const int32_t* rowptr, int64_t* edge_index,
                                int64_t num_edges, void* stream);
/* env.safe_mask / unsafe_mask(data, return_edge=True) (simple_car.py:307-311, 332-336; dubins_car.py:819-823, 844-848;
 * simple_drone.py:380-384, 405-409): dist = ||edge_attr[:, :pos_dim]||; safe = dist > 4R, unsafe = dist < 2R. */
int gcbf_edge_masks(const float* edge_attr, int ld_edge_attr, int pos_dim, int64_t num_edges, double agent_radius, uint8_t* safe,
                    uint8_t* unsafe, void* stream);
/* MessagePassing(aggr='max') (gcbf/nn/gnn.py:116-119) over the CSR of a target-sorted edge list: out[i, c] = max over the
 * incoming edges of msg[e, c], 0 for a node without incoming edges; argmax [num_nodes, channels] (edge id or -1) routes the
 * gradient: d_msg[argmax[i, c], c] = d_out[i, c], everything else 0. */
int gcbf_seg_max_fwd(const float* msg, int ld_msg, const int32_t* rowptr, int num_nodes, int channels, float* out, int ld_out,
                     int32_t* argmax, void* stream);
int gcbf_seg_max_bwd(const float* d_out, int ld_dout, const int32_t* argmax, int num_nodes, int channels, float* d_msg, int ld_dmsg,
                     int64_t num_edges, void* stream);
/* Losses of MACBF.update (macbf.py:140-181) over PER-EDGE h / h_next [num_edges] and per-agent actions [num_agents, action_dim], in
 * the two passes of gcbf_loss_partials / gcbf_loss_grads (ranks may all-reduce `partial` in between).  partial: double[16] =
 * GCBF_LP_SUM_UNSAFE .. GCBF_LP_SUM_ACT as above with GCBF_LP_CNT_ALL = num_edges, then [9] = #(h_dot + alpha h >= 0),
 * [10] = num_agents.  scalars: float[8] = loss_unsafe, loss_safe, loss_h_dot, loss_action, acc_unsafe, acc_safe, total loss,
 * acc_derivative. */
int gcbf_macbf_loss_partials(const float* h, const float* h_next, const uint8_t* safe, const uint8_t* unsafe, int64_t num_edges,
                             const float* action, int action_dim, int64_t num_agents, float alpha, float eps, float dt,
                             double* partial, void* stream);
int gcbf_macbf_loss_grads(const float* h, const float* h_next, const uint8_t* safe, const uint8_t* unsafe, int64_t num_edges,
                          const float* action, int action_dim, int64_t num_agents, float alpha, float eps, float dt,
                          float coef_unsafe, float coef_safe, float coef_hdot, float coef_action, const double* partial, float* d_h,
                          float* d_h_next, float* d_action, float* scalars, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Analytic h_dot (SURVEY 8f-3; an ADDITIVE alternative to the finite difference of gcbf/algo/gcbf.py:193-207, which the training
 * loss uses by default; the backward entry points below train through it): h_dot_i = sum_k (dh_i/ds_k) . f(s_k, u_k) with the edges held fixed, as a forward-mode pass.  The linear layers
 * of the tangent reuse gcbf_linear_fwd* (no bias, no activation) and gcbf_act_bwd (activation derivative); the other pieces:
 *   gcbf_state_dot         x_dot = f(x, clamp(action + u_ref)) for every node (dynamics of simple_car.py:78-89, dubins_car.py:110-132,
 *                          simple_drone.py:103-120; u_ref [num_graphs * num_agents, a] from gcbf_u_ref; freeze != 0: the single-graph
 *                          reach-freeze, needs goal [num_agents, >= pos_dim] (goal_per_graph != 0: one goal set per graph))
 *   gcbf_edge_attr_tangent d/dt edge_attr = g'(s_j) s_dot_j - g'(s_i) s_dot_i            [E, edge_dim]
 *   gcbf_attn_aggr_tangent d/dt sum_e softmax(gate)_e msg_e given d msg [E, C], d gate [E] and the forward's att [E]
 * ------------------------------------------------------------------------------------------------- */
int gcbf_state_dot(const gcbf_env_cfg* cfg, const float* states, int ld_state, const float* action, const float* u_ref,
                   const float* goal, int ld_goal, int goal_per_graph, int freeze, float* state_dot, int ld_out, void* stream);
int gcbf_edge_attr_tangent(int env, const float* states, int ld_state, const float* state_dot, int ld_sdot, const int64_t* edge_index,
                           int64_t num_edges, float* t_edge_attr, void* stream);
int gcbf_attn_aggr_tangent(const float* msg, int ld_msg, const float* t_msg, int ld_tmsg, const float* att, const float* t_gate,
                           const int32_t* rowptr, int num_nodes, int channels, float* t_aggr, int ld_taggr, void* stream);

/* ---------------------------------------------------------------------------------------------------
 * Backward of the analytic h_dot pass: the opt-in CBF-condition loss of GCBF.params['h_dot'] = 'analytic', which trains through
 * h_dot = J_h(s) . f(s, clamp(u + u_ref)) instead of the finite difference of gcbf/algo/gcbf.py:193-207.  Deterministic, no float atomics.
 *   gcbf_attn_aggr_tangent_bwd  VJP of gcbf_attn_aggr_tangent.  With tau = d L / d t_aggr_i, p_e = msg_e . tau, q_e = t_msg_e . tau,
 *                               gbar_i = sum_k a_k t_gate_k, P_i = sum_k a_k p_k:  d_t_msg_e = a_e tau,  d_t_gate_e = a_e (p_e - P_i), and the
 *                               second-order terms  d_msg_e += a_e (t_gate_e - gbar_i) tau,  d_gate_e += a_e (r_e - sum_k a_k r_k) with
 *                               r_e = q_e + t_gate_e (p_e - P_i) - gbar_i p_e, added onto the primal gcbf_attn_aggr_bwd gradients
 *                               (accumulate = 0: written).  One warp per target; any channel count and pitch.  The edge arrays may be
 *                               null when the batch has no edges.
 *   gcbf_act_tangent_bwd        element-wise, y = act(z), y_dot = act'(z) z_dot:  ReLU  dZ = [Y > 0] dY, dTZ = [Y > 0] dTY;  tanh  dTZ =
 *                               (1 - Y^2) dTY, dZ = (1 - Y^2)(dY - 2 Y TZ dTY) (TZ: the pre-activation tangent z_dot, read for tanh only);
 *                               none  identity.
 *   gcbf_state_dot_bwd          d L / d action [num_graphs * num_agents, a] from d L / d x_dot [nodes, >= state_dim]: the VJP of gcbf_state_dot
 *                               (same arguments) through the clamp (gradient passes where -lim <= action + u_ref <= lim, as torch.clamp) and
 *                               the reach-freeze (zero for frozen agents); obstacle rows carry no action.  accumulate: add onto d_action.
 *   gcbf_edge_attr_bwd_ordered  d states += d edge_attr . d edge_attr / d states (the VJP of gcbf_edge_attr_fwd, equal to gcbf_edge_attr_bwd
 *                               to rounding) summed in a fixed order per node: bit-reproducible.  d_states has pitch ld_state and is
 *                               accumulated into.  PRECONDITION: edge_index[1] (targets) sorted ascending, as every graph this library
 *                               builds is (each node's target-side run is found by binary search; unsorted edges give wrong gradients).  Since the edge tangent is linear in s_dot with the same Jacobian, this is also its VJP.
 *   gcbf_loss_partials_hdot /   gcbf_loss_partials / gcbf_loss_grads with h_dot an input: same partial layout, scalars and masked means;
 *   gcbf_loss_grads_hdot        d_hdot = d loss / d h_dot takes the place of d_h_next.
 * ------------------------------------------------------------------------------------------------- */
int gcbf_attn_aggr_tangent_bwd(const float* msg, int ld_msg, const float* t_msg, int ld_tmsg, const float* att, const float* t_gate,
                               const int32_t* rowptr, int num_nodes, int channels, const float* d_t_aggr, int ld_dtaggr, float* d_t_msg,
                               int ld_dtmsg, float* d_t_gate, float* d_msg, int ld_dmsg, float* d_gate, int accumulate, void* stream);
int gcbf_act_tangent_bwd(const float* dY, const float* dTY, const float* Y, const float* TZ, int64_t count, int act, float* dZ, float* dTZ,
                         void* stream);
int gcbf_state_dot_bwd(const gcbf_env_cfg* cfg, const float* states, int ld_state, const float* action, const float* u_ref,
                       const float* goal, int ld_goal, int goal_per_graph, int freeze, const float* d_state_dot, int ld_dsdot,
                       float* d_action, int accumulate, void* stream);
int gcbf_edge_attr_bwd_ordered(int env, const float* states, int ld_state, const int64_t* edge_index, int64_t num_edges, int num_nodes,
                               const float* d_edge_attr, float* d_states, void* stream);
int gcbf_loss_partials_hdot(const float* h, const float* hdot, const float* action, int action_dim, const uint8_t* safe,
                            const uint8_t* unsafe, int64_t num_agents_total, float alpha, float eps, double* partial, void* stream);
int gcbf_loss_grads_hdot(const float* h, const float* hdot, const float* action, int action_dim, const uint8_t* safe,
                         const uint8_t* unsafe, int64_t num_agents_total, float alpha, float eps, float coef_unsafe, float coef_safe,
                         float coef_hdot, float coef_action, const double* partial, float* d_h, float* d_hdot, float* d_action,
                         float* scalars, void* stream);

/* instrumentation (bench.py): kernels launched by the chain-level calls since the last reset, and optional CUDA-event timing of
 * every linear-layer launch (kind 0 forward / 1 data-grad / 2 weight-grad on the tensor cores, 3 fp32 linear kernels, 4 operand
 * preparation = amax + fp16 split) */
long long gcbf_launch_count(int reset);
typedef struct gcbf_time_rec { double ms; double flops; int32_t kind; int32_t M, N, K; } gcbf_time_rec;
int gcbf_timing_enable(int on);
int gcbf_timing_collect(gcbf_time_rec* out, int max_records, int* count);   /* synchronises the device; clears the records */
/* 0 auto, 1 force the fp32 SIMT kernels, 2 force the tensor-core path (tests) -- what gcbf_b200.ops.GEMM_IMPL was */
int gcbf_set_gemm_impl(int impl);

#ifdef __cplusplus
}
#endif
#endif /* GCBF_B200_H */
