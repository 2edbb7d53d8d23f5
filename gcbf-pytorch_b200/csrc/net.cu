// Chain-level host code: one C-ABI call per GNN pass (gcbf_net_forward / gcbf_net_backward) and per bare MLP
// (gcbf_mlp_forward / gcbf_mlp_backward).  It sequences the kernels of this library the way the reference sequences ATen calls in
//   gcbf/nn/mlp.py:44-47            Linear -> ReLU -> ... -> Linear (-> Tanh), spectral-norm pre-hook per layer (mlp.py:21,33)
//   gcbf/nn/gnn.py:27-36, 59-73     cat[x_i, x_j, e_ij] -> phi -> AttentionalAggregation(gate_nn) -> gamma(cat[aggr, x])
//   gcbf/algo/gcbf.py:37-55         CBFGNN.forward: layer -> x[agent_mask] -> feat_2_CBF
//   gcbf/controller/gnn_controller.py:29-48   GNNController.forward: layer -> x[agent_mask] -> feat_2_action(cat[x, u_ref])
// and their autograd backward.  Nothing here allocates device memory: every activation, fp16 companion, amax word and scratch
// gradient is a bump allocation out of the caller's workspace; the *_workspace_bytes queries replay the same allocation sequence
// without launching.  Per layer the dispatch rule is: tensor cores (3xFP16 wgmma kernel, gemm_wgmma_f16.cu) when
// gcbf_linear_h_supported(M, N, K), else the fp32 kernels behind gcbf_linear_* (skinny-K / row-streaming / SIMT tile).
#include <atomic>
#include <vector>

#include "chain.h"

namespace gcbf {
namespace chain {

std::atomic<long long> g_launches{0};
static int g_gemm_impl = 0;
static bool g_timing = false;
bool timing_on() { return g_timing; }
struct Rec { cudaEvent_t e0, e1; double flops; int kind, M, N, K; };
static std::vector<Rec> g_recs;
static std::vector<cudaEvent_t> g_event_pool;

static cudaEvent_t pool_event() {
  if (!g_event_pool.empty()) { cudaEvent_t e = g_event_pool.back(); g_event_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}

bool use_h(int M, int N, int K) {
  if (g_gemm_impl == 1) return false;
  if (g_gemm_impl == 2) return true;
  return gcbf_linear_h_supported(M, N, K) != 0;
}

// ---- timed launches ------------------------------------------------------------------------------------------------
struct Timed {
  bool on; Rec r; cudaStream_t st;
  Timed(Run& R, int kind, double flops, int M, int N, int K) : on(g_timing && !R.dry), st(R.st) {
    if (on) { r.e0 = pool_event(); r.e1 = pool_event(); r.flops = flops; r.kind = kind; r.M = M; r.N = N; r.K = K; cudaEventRecord(r.e0, st); }
  }
  ~Timed() { if (on) { cudaEventRecord(r.e1, st); g_recs.push_back(r); } }
};

// ---- operand preparation -------------------------------------------------------------------------------------------
// amax (unless the producer supplied it) + fp16 [hi|lo] split of x[rows, cols] (pitch ld); optional column sums into `colsum`
// (accumulated: it is a bias's gradient target)
int split_h(Run& R, const float* x, int ld, int rows, int cols, const void* amax, float* colsum, H16* out) {
  const int ld_h = (cols + 7) / 8 * 8;
  out->buf = R.ws.alloc((size_t)2 * rows * ld_h * 2);
  out->ld = ld_h; out->rows = rows; out->cols = cols; out->sr = 0; out->sc = 0;
  void* own = nullptr;
  if (!amax) own = R.amax_slot();
  out->amax = amax ? amax : own;
  if (R.dry) return 0;
  Timed t(R, 4, 0.0, rows, cols, 0);
  if (!amax) { CHAIN_CALL(gcbf_amax_f32(x, ld, rows, cols, own, 0, R.st)); R.launched(1); }
  CHAIN_CALL(gcbf_split_f16(x, ld, rows, cols, out->amax, out->buf, ld_h, colsum, 1, R.st));
  R.launched(1);
  return 0;
}

int refresh_weight_companions(Run& R, const gcbf_linear_desc* const* layers, int n) {
  if (R.dry) return 0;
  gcbf_split_desc d[4 * GCBF_MAX_MLP_LAYERS];
  int cnt = 0;
  for (int i = 0; i < n; ++i) {
    const gcbf_linear_desc& L = *layers[i];
    if (!L.Wh || !L.w_amax) continue;
    bool dup = false;
    for (int j = 0; j < cnt; ++j) dup |= (d[j].src == L.W);
    if (dup) continue;
    d[cnt].src = L.W; d[cnt].ld = L.ldw; d[cnt].rows = L.N; d[cnt].cols = L.K; d[cnt].ld_h = L.ldwh; d[cnt].amax_slot = L.w_amax; d[cnt].dst = L.Wh;
    ++cnt;
  }
  if (!cnt) return 0;
  Timed t(R, 4, 0.0, 0, 0, 0);
  CHAIN_CALL(gcbf_amax_split_batched(d, cnt, R.st));
  R.launched(2 * ((cnt + 15) / 16));
  return 0;
}

// one power iteration on every spectral-normalised layer of `layers` (4 launches); inv_sigma[i] / u, v snapshots per layer
int sn_power_iter(Run& R, const gcbf_linear_desc* const* layers, int n, bool snapshot, const float** inv_sigma, const float** us,
                  const float** vs) {
  gcbf_sn_layer sl[4 * GCBF_MAX_MLP_LAYERS];
  int idx[4 * GCBF_MAX_MLP_LAYERS];
  int cnt = 0;
  size_t need = 0;
  for (int i = 0; i < n; ++i) {
    inv_sigma[i] = nullptr; us[i] = nullptr; vs[i] = nullptr;
    if (layers[i]->u) { idx[cnt++] = i; need += gcbf_sn_workspace_floats(layers[i]->N, layers[i]->K); }
  }
  if (!cnt) return 0;
  float* inv = (float*)R.ws.alloc((size_t)cnt * 4);
  float* wsf = (float*)R.ws.alloc(need * 4);
  for (int c = 0; c < cnt; ++c) {
    const gcbf_linear_desc& L = *layers[idx[c]];
    sl[c].W = L.W; sl[c].ldw = L.ldw; sl[c].N = L.N; sl[c].K = L.K; sl[c].pad_ = 0; sl[c].u = L.u; sl[c].v = L.v; sl[c].inv_sigma = inv + c;
    inv_sigma[idx[c]] = inv + c;
  }
  if (!R.dry) { CHAIN_CALL(gcbf_sn_power_iter_batched(sl, cnt, wsf, need, R.st)); R.launched(4); }
  if (snapshot) {
    // the backward's sigma-gradient needs the u, v of ITS forward (later forwards of the same net advance them)
    for (int c = 0; c < cnt; ++c) {
      const gcbf_linear_desc& L = *layers[idx[c]];
      float* su = (float*)R.ws.alloc((size_t)L.N * 4);
      float* sv = (float*)R.ws.alloc((size_t)L.K * 4);
      us[idx[c]] = su; vs[idx[c]] = sv;
      if (!R.dry) {
        CHAIN_CUDA(cudaMemcpyAsync(su, L.u, (size_t)L.N * 4, cudaMemcpyDeviceToDevice, R.st));
        CHAIN_CUDA(cudaMemcpyAsync(sv, L.v, (size_t)L.K * 4, cudaMemcpyDeviceToDevice, R.st));
      }
    }
  }
  return 0;
}

// ---- MLP chain -------------------------------------------------------------------------------------------------------
// Companions written by the producing GEMM's epilogue ("emission", gemm_wgmma_f16.cu): when a tensor-core layer's output (forward)
// or input gradient (backward) feeds another tensor-core layer, the producer writes it directly as a tile-scaled fp16 [hi|lo]
// companion -- no amax pass, no split pass, no fp32 copy in HBM; the ReLU mask of the backward is read from the hi plane and the
// bias gradient (column sums of dZ) is accumulated by the producing data-grad epilogue.  GCBF_EPI_H=0 keeps the split kernels.
static int g_epi_h = -1;
static int g_epi_h_bwd = 1;      // GCBF_EPI_H_BWD=0: no emission in the backward (data-grad epilogue: mask + companion + column sums).  History of
                                 // the in-step A/B at C3: with the spilling epilogue of the 10-warp kernel the emitting data-grad cost 4.71 -> 6.24 ms
                                 // against 0.89 ms of amax + split saved (off); with the 12-warp setmaxnreg kernel, two staging boxes and
                                 // 256-element chunks for the consumer it is 3.71 -> 3.99 ms: the step gains ~1 ms (on)
static bool epi_h_enabled() {
  if (g_epi_h < 0) {
    const char* e = getenv("GCBF_EPI_H");
    const char* k = getenv("GCBF_TC_KCH");
    g_epi_h = (e && e[0] == '0') ? 0 : 1;
    if (k && atoi(k) > 4) g_epi_h = 0;          // tile-scaled operands need promotion chunks of <= 128 K-elements
    const char* b = getenv("GCBF_EPI_H_BWD");
    g_epi_h_bwd = (b && b[0] == '0') ? 0 : 1;
  }
  return g_epi_h == 1 && g_gemm_impl != 1;
}
// may a [M, width] tensor produced by a tensor-core layer be emitted as a companion for a consumer layer with `consumer_n` outputs?
static bool can_emit(int M, int width, int consumer_n) { return epi_h_enabled() && width > 128 && consumer_n > 0 && use_h(M, consumer_n, width); }
static bool can_emit_bwd(int M, int width, int consumer_n) { return can_emit(M, width, consumer_n) && g_epi_h_bwd == 1; }

static gcbf_h16 h16_desc(const H16& h) {
  gcbf_h16 d;
  d.buf = h.buf; d.amax = const_cast<void*>(h.amax); d.ld = h.ld; d.rows = h.rows; d.cols = h.cols;
  d.amax_row_stride = h.sr; d.amax_col_stride = h.sc; d.pad_ = 0;
  return d;
}
static gcbf_h16 weight_desc(const gcbf_linear_desc& L) {
  gcbf_h16 d;
  d.buf = L.Wh; d.amax = L.w_amax; d.ld = L.ldwh; d.rows = L.N; d.cols = L.K; d.amax_row_stride = 0; d.amax_col_stride = 0; d.pad_ = 0;
  return d;
}
// buffers of a tile-scaled companion an epilogue is about to write
static H16 alloc_tiled(Run& R, int rows, int cols) {
  H16 h{};
  h.ld = (cols + 7) / 8 * 8; h.rows = rows; h.cols = cols;
  h.buf = R.ws.alloc((size_t)2 * rows * h.ld * 2);
  h.sr = (cols + 255) / 256; h.sc = 1;
  h.amax = R.ws.alloc((size_t)((rows + 127) / 128) * h.sr * 4);
  return h;
}

// y = MLP(x).  x: fp32 input (may be nullptr when x_h is given); x_h: its companion if a producer emitted one; x_amax: per-tensor
// amax word of x when its producer reduced it.  next_width > 0: the output feeds a linear layer of that many out-features.
// `out`: where the LAST layer writes its fp32 output (pitch ld_out), or nullptr for a workspace buffer; out_h (optional): receives the
// emitted companion of the output when the consumer qualifies (buf == nullptr otherwise) -- the fp32 output is then written only
// if need_f32_out.
int mlp_forward(Run& R, const gcbf_linear_desc* layers, int n, const float* x, int ldx, int M, const H16* x_h, const void* x_amax,
                int next_width, const float* const* inv_sigma, const float* const* us, const float* const* vs, MlpCtx* ctx, float* out,
                int ld_out, bool need_f32_out, H16* out_h, const float** y, int* ldy, const void** y_amax) {
  if (ctx) { memset(ctx, 0, sizeof(*ctx)); ctx->n = n; ctx->M = M; ctx->acts[0] = x; ctx->ld[0] = ldx; }
  const float* cur = x;
  int ldc = ldx;
  H16 cur_h = x_h ? *x_h : H16{};
  const void* cur_amax = x_amax;
  if (out_h) *out_h = H16{};
  for (int l = 0; l < n; ++l) {
    const gcbf_linear_desc& L = layers[l];
    const int N = L.N, K = L.K;
    const bool lastl = (l == n - 1);
    const int nxt = !lastl ? layers[l + 1].N : next_width;
    const bool h = use_h(M, N, K) && M > 0;
    const bool sk_emit = !h && !lastl && K <= 16 && M >= 64 && N >= 64 && cur && g_gemm_impl == 0 && can_emit(M, N, nxt);
    const bool emit = sk_emit || (h && can_emit(M, N, nxt) && (!lastl || out_h != nullptr));
    const bool f32 = !emit || (lastl && need_f32_out);
    void* ya = (!emit && nxt > 0 && use_h(M, nxt, N)) ? R.amax_slot() : nullptr;
    float* dst = nullptr; int ldd = N;
    if (f32) {
      if (lastl && out) { dst = out; ldd = ld_out; }
      else dst = (float*)R.ws.alloc((size_t)M * N * 4);
    }
    H16 yh{};
    if (h) {
      if (!L.Wh) { set_error("layer [%d x %d] runs on the tensor cores but its descriptor has no weight companion", N, K); return GCBF_E_INVALID; }
      if (!cur_h.buf) { if (int rc = split_h(R, cur, ldc, M, K, cur_amax, nullptr, &cur_h)) return rc; }
      if (emit) yh = alloc_tiled(R, M, N);
      if (!R.dry) {
        Timed t(R, 0, 2.0 * M * N * K, M, N, K);
        const gcbf_h16 X = h16_desc(cur_h), W = weight_desc(L), Y = h16_desc(yh);
        CHAIN_CALL(gcbf_linear_fwd_t(&X, &W, L.b, inv_sigma[l], L.act, dst, ldd, emit ? &Y : nullptr, ya, M, N, K, R.st));
        R.launched(1);
      }
    } else if (sk_emit) {
      // skinny-K layer in front of a tensor-core layer: companion only (each tile computed twice, nothing re-read)
      yh = alloc_tiled(R, M, N);
      if (!R.dry) {
        Timed t(R, 3, 2.0 * M * N * K, M, N, K);
        const gcbf_h16 Y = h16_desc(yh);
        CHAIN_CALL(gcbf_linear_fwd_emit(cur, ldc, L.W, L.ldw, L.b, inv_sigma[l], L.act, &Y, M, N, K, R.st));
        R.launched(1);
      }
    } else {
      if (!cur && M > 0) { set_error("mlp_forward: layer %d needs its fp32 input", l); return GCBF_E_INVALID; }
      if (!R.dry) {
        Timed t(R, 3, 2.0 * M * N * K, M, N, K);
        CHAIN_CALL(gcbf_linear_fwd(cur, ldc, L.W, L.ldw, L.b, inv_sigma[l], dst, ldd, M, N, K, L.act, g_gemm_impl == 1 ? 1 : 0, ya, R.st));
        R.launched(ya ? 2 : 1);
      }
    }
    if (ctx) {
      ctx->acts[l + 1] = dst; ctx->ld[l + 1] = ldd;
      ctx->acts_h[l] = h ? cur_h : H16{};
      ctx->inv_sigma[l] = inv_sigma[l]; ctx->u[l] = us[l]; ctx->v[l] = vs[l];
    }
    cur = dst; ldc = ldd; cur_amax = ya; cur_h = yh;
  }
  if (out_h) *out_h = cur_h;
  *y = cur; *ldy = ldc;
  if (y_amax) *y_amax = cur_amax;
  return 0;
}

__global__ void vec_add_kernel(float* __restrict__ dst, const float* __restrict__ src, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] += src[i];
}
int vec_add(Run& R, float* dst, const float* src, int64_t n) {
  if (R.dry || n == 0) return 0;
  vec_add_kernel<<<ceil_div(n, 256), 256, 0, R.st>>>(dst, src, n);
  CHAIN_CUDA(cudaGetLastError());
  R.launched(1);
  return 0;
}

// Backward of the chain.  dy [M, N_last] (pitch ld_dy) -- or its emitted companion dy_h (then dy may be nullptr and the bias gradient
// of the last layer has already been accumulated by the producer iff dy_colsum_done); dy_amax: per-tensor amax word of dy if the
// producer reduced it.  need_dx: produce the input gradient -- into dx_out (pitch ld_dx, optionally accumulated) or a workspace
// buffer; dx_amax: word that receives max|dx| if the input-gradient GEMM runs on the tensor cores (*dx_amax_valid).  dx_h (optional):
// the caller's consumer is a tensor-core layer with `dx_consumer_n` outputs whose bias gradient lives at dx_colsum: if the producer
// qualifies, dx is emitted as a companion only (*dx == nullptr, dx_h->buf != nullptr) and its column sums are added to dx_colsum.
int mlp_backward(Run& R, const gcbf_linear_desc* layers, int n, const MlpCtx& ctx, const float* dy, int ld_dy, const H16* dy_h,
                 bool dy_colsum_done, bool need_dx, float* dx_out, int ld_dx, bool dx_accumulate, const void* dy_amax, void* dx_amax,
                 bool skip_wgrad, H16* dx_h, int dx_consumer_n, float* dx_colsum, const float** dx, int* ld_dx_res, bool* dx_amax_valid) {
  const int M = ctx.M;
  const int last = n - 1;
  const float* dz = dy;
  int lddz = ld_dy;
  H16 dzh = dy_h ? *dy_h : H16{};
  bool colsum_done = dy_h ? dy_colsum_done : false;
  if (dx_h) *dx_h = H16{};
  if (layers[last].act != GCBF_ACT_NONE) {
    const int N = layers[last].N;
    if (!dz || ld_dy != N || ctx.ld[last + 1] != N || !ctx.acts[last + 1]) { set_error("mlp_backward: output activation needs dense fp32 d_out / output"); return GCBF_E_INVALID; }
    float* t = (float*)R.ws.alloc((size_t)M * N * 4);
    if (!R.dry) { CHAIN_CALL(gcbf_act_bwd(dz, ctx.acts[last + 1], t, (int64_t)M * N, layers[last].act, R.st)); R.launched(1); }
    dz = t;
  }
  const void* dz_amax = (layers[last].act == GCBF_ACT_NONE) ? dy_amax : nullptr;
  if (dx_amax_valid) *dx_amax_valid = false;
  for (int l = last; l >= 0; --l) {
    const gcbf_linear_desc& L = layers[l];
    const float* x_in = ctx.acts[l];
    const int ldx = ctx.ld[l];
    const float* isg = ctx.inv_sigma[l];
    const int N = L.N, K = L.K;
    const bool wgrad = !skip_wgrad && L.gW;
    if (use_h(M, N, K) && M > 0) {
      // one fp16 companion of dz serves the weight-grad (MN-major A) and the data-grad (K-major A); the bias gradient (column
      // sums of dz) is fused into the split -- or was accumulated by the epilogue that emitted the companion
      if (!dzh.buf) {
        if (int rc = split_h(R, dz, lddz, M, N, dz_amax, (wgrad && L.gb) ? L.gb : nullptr, &dzh)) return rc;
      } else if (wgrad && L.gb && !colsum_done) {
        set_error("mlp_backward: emitted gradient companion without its bias gradient"); return GCBF_E_INVALID;
      }
      const gcbf_h16 dZ = h16_desc(dzh), W = weight_desc(L);
      if (wgrad) {
        H16 xh = ctx.acts_h[l];
        if (!xh.buf) { if (int rc = split_h(R, x_in, ldx, M, K, nullptr, nullptr, &xh)) return rc; }
        const gcbf_h16 X = h16_desc(xh);
        if (L.u) {
          float* dW = (float*)R.ws.alloc((size_t)N * K * 4);
          float* fx = (float*)R.ws.alloc(gcbf_sn_workspace_floats(N, K) * 4);
          if (!R.dry) {
            { Timed t(R, 2, 2.0 * M * N * K, M, N, K);
              CHAIN_CALL(gcbf_linear_bwd_weight_t(&dZ, &X, isg, dW, K, 0, M, N, K, R.st)); }
            CHAIN_CALL(gcbf_sn_grad_fixup(dW, K, L.W, L.ldw, N, K, ctx.u[l], ctx.v[l], isg, fx, L.gW, L.ldgw, R.st));
            R.launched(3);
          }
        } else if (!R.dry) {
          Timed t(R, 2, 2.0 * M * N * K, M, N, K);
          CHAIN_CALL(gcbf_linear_bwd_weight_t(&dZ, &X, isg, L.gW, L.ldgw, 1, M, N, K, R.st));
          R.launched(1);
        }
      }
      // ReLU mask of the layer below: from its fp32 output, or from the hi plane of that output's companion
      const gcbf_h16 maskh = h16_desc(ctx.acts_h[l]);
      const bool mask_h = (x_in == nullptr);
      if (l > 0) {
        const gcbf_linear_desc& P = layers[l - 1];
        const bool emit = can_emit_bwd(M, K, P.K) && use_h(M, P.N, P.K);
        const bool pw = !skip_wgrad && P.gW && P.gb;
        void* na = (!emit && use_h(M, K, P.K)) ? R.amax_slot() : nullptr;
        float* o = emit ? nullptr : (float*)R.ws.alloc((size_t)M * K * 4);
        H16 oh{};
        if (emit) oh = alloc_tiled(R, M, K);
        if (!R.dry) {
          Timed t(R, 1, 2.0 * M * N * K, M, N, K);
          const gcbf_h16 O = h16_desc(oh);
          CHAIN_CALL(gcbf_linear_bwd_data_t(&dZ, &W, isg, mask_h ? nullptr : x_in, ldx, mask_h ? &maskh : nullptr, o, K, 0, emit ? &O : nullptr,
                                            (emit && pw) ? P.gb : nullptr, na, M, N, K, R.st));
          R.launched(1);
        }
        dz = o; lddz = K; dz_amax = na; dzh = oh; colsum_done = emit && pw;
      } else if (need_dx) {
        const bool emit = dx_h && !dx_out && !dx_accumulate && can_emit_bwd(M, K, dx_consumer_n);
        float* o = dx_out; int ldo = ld_dx;
        if (!o && !emit) { o = (float*)R.ws.alloc((size_t)M * K * 4); ldo = K; }
        H16 oh{};
        if (emit) oh = alloc_tiled(R, M, K);
        if (!R.dry) {
          Timed t(R, 1, 2.0 * M * N * K, M, N, K);
          const gcbf_h16 O = h16_desc(oh);
          CHAIN_CALL(gcbf_linear_bwd_data_t(&dZ, &W, isg, nullptr, 0, nullptr, o, ldo, dx_accumulate ? 1 : 0, emit ? &O : nullptr,
                                            (emit && !skip_wgrad) ? dx_colsum : nullptr, emit ? nullptr : dx_amax, M, N, K, R.st));
          R.launched(1);
        }
        dz = o; lddz = ldo;
        if (emit) *dx_h = oh;
        if (dx_amax_valid) *dx_amax_valid = (!emit && dx_amax != nullptr);
      } else {
        dz = nullptr;
      }
      if (l > 0) continue;
      break;
    }
    if (!dz && M > 0) { set_error("mlp_backward: layer %d needs its fp32 output gradient", l); return GCBF_E_INVALID; }
    dz_amax = nullptr;
    dzh = H16{};
    const int impl = g_gemm_impl == 1 ? 1 : 0;
    if (wgrad) {
      if (L.u) {
        float* dW = (float*)R.ws.alloc((size_t)N * K * 4);
        float* db = (float*)R.ws.alloc((size_t)N * 4);
        float* fx = (float*)R.ws.alloc(gcbf_sn_workspace_floats(N, K) * 4);
        if (!R.dry) {
          { Timed t(R, 3, 2.0 * M * N * K, M, N, K);
            CHAIN_CALL(gcbf_linear_bwd_weight(dz, lddz, x_in, ldx, isg, dW, K, L.gb ? db : nullptr, M, N, K, 0, impl, R.st)); }
          CHAIN_CALL(gcbf_sn_grad_fixup(dW, K, L.W, L.ldw, N, K, ctx.u[l], ctx.v[l], isg, fx, L.gW, L.ldgw, R.st));
          R.launched(4);
        }
        if (L.gb) { if (int rc = vec_add(R, L.gb, db, N)) return rc; }
      } else if (!R.dry) {
        Timed t(R, 3, 2.0 * M * N * K, M, N, K);
        CHAIN_CALL(gcbf_linear_bwd_weight(dz, lddz, x_in, ldx, isg, L.gW, L.ldgw, L.gb, M, N, K, 1, impl, R.st));
        R.launched(2);
      }
    }
    if (l > 0) {
      // hidden ReLU of layer l-1 folded into the epilogue: dz_{l-1} = (dz_l W_l) * (y_{l-1} > 0)
      float* o = (float*)R.ws.alloc((size_t)M * K * 4);
      if (!R.dry) {
        Timed t(R, 3, 2.0 * M * N * K, M, N, K);
        CHAIN_CALL(gcbf_linear_bwd_data(dz, lddz, L.W, L.ldw, isg, x_in, ldx, o, K, M, N, K, 0, impl, R.st));
        R.launched(1);
      }
      dz = o; lddz = K;
    } else if (need_dx) {
      float* o = dx_out; int ldo = ld_dx;
      if (!o) { o = (float*)R.ws.alloc((size_t)M * K * 4); ldo = K; }
      if (!R.dry) {
        Timed t(R, 3, 2.0 * M * N * K, M, N, K);
        CHAIN_CALL(gcbf_linear_bwd_data(dz, lddz, L.W, L.ldw, isg, nullptr, 0, o, ldo, M, N, K, dx_accumulate ? 1 : 0, impl, R.st));
        R.launched(1);
      }
      dz = o; lddz = ldo;
    } else {
      dz = nullptr;
    }
  }
  if (dx) *dx = dz;
  if (ld_dx_res) *ld_dx_res = lddz;
  return 0;
}

static int check_mlp(const gcbf_linear_desc* layers, int n, const char* what) {
  if (n < 1 || n > GCBF_MAX_MLP_LAYERS) { set_error("%s: %d layers (1..%d supported)", what, n, GCBF_MAX_MLP_LAYERS); return GCBF_E_INVALID; }
  for (int l = 0; l < n; ++l) {
    const gcbf_linear_desc& L = layers[l];
    if (!L.W || !L.b || L.N <= 0 || L.K <= 0 || L.ldw < L.K || (L.u == nullptr) != (L.v == nullptr)) { set_error("%s: layer %d descriptor", what, l); return GCBF_E_INVALID; }
    if (l > 0 && layers[l - 1].N != L.K) { set_error("%s: layer %d in-features %d != previous out-features %d", what, l, L.K, layers[l - 1].N); return GCBF_E_INVALID; }
    if (l < n - 1 && L.act != GCBF_ACT_RELU) { set_error("%s: hidden activation of layer %d must be ReLU (mlp.py:13)", what, l); return GCBF_E_INVALID; }
  }
  return 0;
}

// ---- the GNN pass ------------------------------------------------------------------------------------------------------
static int collect_layers(const gcbf_net_desc& net, const gcbf_linear_desc** all) {
  int n = 0;
  for (int i = 0; i < net.n_phi; ++i) all[n++] = &net.phi[i];
  for (int i = 0; i < net.n_gate; ++i) all[n++] = &net.gate[i];
  for (int i = 0; i < net.n_gamma; ++i) all[n++] = &net.gamma[i];
  for (int i = 0; i < net.n_head; ++i) all[n++] = &net.head[i];
  return n;
}

int check_net(const gcbf_net_desc* net) {
  if (!net) { set_error("null net descriptor"); return GCBF_E_INVALID; }
  if (int rc = check_mlp(net->phi, net->n_phi, "phi")) return rc;
  if (int rc = check_mlp(net->gate, net->n_gate, "gate_nn")) return rc;
  if (int rc = check_mlp(net->gamma, net->n_gamma, "gamma")) return rc;
  if (net->n_head && check_mlp(net->head, net->n_head, "head")) return GCBF_E_INVALID;
  const int kin = 2 * net->node_dim + net->edge_dim;
  if (net->phi[0].K != kin || net->phi[net->n_phi - 1].N != net->phi_dim || net->gate[0].K != net->phi_dim ||
      net->gate[net->n_gate - 1].N != 1 || net->gamma[0].K != net->phi_dim + net->node_dim ||
      (net->n_head && net->head[0].K != net->gamma[net->n_gamma - 1].N + net->head_extra_dim)) {
    set_error("net descriptor: layer widths do not chain (phi in %d, phi_dim %d, gamma in %d)", net->phi[0].K, net->phi_dim, net->gamma[0].K);
    return GCBF_E_INVALID;
  }
  return 0;
}

int net_forward(Run& R, const gcbf_net_desc& net, const float* x, const float* edge_attr, const int64_t* edge_index,
                const int32_t* rowptr, int64_t E64, int Nn, const int64_t* row_index, int rows, const float* head_extra, float* out,
                int ld_out, NetCtx* ctx) {
  const int E = (int)E64;
  const int nd = net.node_dim, C = net.phi_dim, kin = 2 * nd + net.edge_dim;
  const bool save = ctx != nullptr;
  if (ctx) { memset(ctx, 0, sizeof(*ctx)); ctx->E = E; ctx->Nn = Nn; ctx->R = rows; }
  float* ein = (float*)R.ws.alloc((size_t)E * kin * 4);
  if (!R.dry && E > 0) { CHAIN_CALL(gcbf_edge_input_fwd(x, nd, edge_attr, net.edge_dim, edge_index, E, ein, kin, R.st)); R.launched(1); }
  // the power iterations depend on the weights only: all spectral-normalised layers of the net in one batched call
  const gcbf_linear_desc* all[4 * GCBF_MAX_MLP_LAYERS];
  const int nall = collect_layers(net, all);
  const float *isg[4 * GCBF_MAX_MLP_LAYERS], *us[4 * GCBF_MAX_MLP_LAYERS], *vs[4 * GCBF_MAX_MLP_LAYERS];
  if (int rc = sn_power_iter(R, all, nall, save, isg, us, vs)) return rc;
  if (net.refresh_weights) { if (int rc = refresh_weight_companions(R, all, nall)) return rc; }
  const int o_gate = net.n_phi, o_gamma = o_gate + net.n_gate, o_head = o_gamma + net.n_gamma;
  const float *msg, *gate, *feat;
  int ldm, ldg, ldf;
  const void *msg_amax = nullptr, *feat_amax = nullptr;
  H16 msg_h{}, feat_h{};
  // phi's output is needed twice: as fp32 by the aggregation and (as a companion, when the gate's first layer is a tensor-core
  // layer) by gate_nn -- the last phi layer writes both
  if (int rc = mlp_forward(R, net.phi, net.n_phi, ein, kin, E, nullptr, nullptr, net.gate[0].N, isg, us, vs, save ? &ctx->phi : nullptr, nullptr, 0,
                           true, &msg_h, &msg, &ldm, &msg_amax)) return rc;                      // gnn.py:30-32
  if (int rc = mlp_forward(R, net.gate, net.n_gate, msg, ldm, E, msg_h.buf ? &msg_h : nullptr, msg_amax, 0, isg + o_gate, us + o_gate, vs + o_gate,
                           save ? &ctx->gate : nullptr, nullptr, 0, true, nullptr, &gate, &ldg, nullptr)) return rc;   // AttentionalAggregation.gate_nn
  float* gin_all = (float*)R.ws.alloc((size_t)Nn * (C + nd) * 4);
  float* att = (float*)R.ws.alloc((size_t)E * 4);
  if (!R.dry) {
    CHAIN_CALL(gcbf_attn_aggr_fwd(E ? msg : nullptr, C, E ? gate : nullptr, rowptr, Nn, C, E ? att : nullptr, gin_all, C + nd, R.st));
    CHAIN_CALL(gcbf_copy2d(x, nd, gin_all + C, C + nd, Nn, nd, R.st));                             // cat([aggr_out, x])  gnn.py:35
    R.launched(2);
  }
  const float* gin = gin_all;
  if (row_index) {
    float* g = (float*)R.ws.alloc((size_t)rows * (C + nd) * 4);
    if (!R.dry) { CHAIN_CALL(gcbf_rows_gather(gin_all, C + nd, row_index, g, C + nd, rows, C + nd, R.st)); R.launched(1); }
    gin = g;
  }
  const bool has_head = net.n_head > 0;
  const bool chain_head = has_head && net.head_extra_dim == 0;                          // the head reads gamma's output in place
  // gamma's output feeds the head directly when nothing is concatenated (CBF): then only its companion is written
  if (int rc = mlp_forward(R, net.gamma, net.n_gamma, gin, C + nd, rows, nullptr, nullptr, chain_head ? net.head[0].N : 0, isg + o_gamma,
                           us + o_gamma, vs + o_gamma, save ? &ctx->gamma : nullptr, has_head ? nullptr : out, ld_out, !chain_head,
                           chain_head ? &feat_h : nullptr, &feat, &ldf, &feat_amax)) return rc;   // gnn.py:34-36
  if (has_head) {
    const int F = net.gamma[net.n_gamma - 1].N;
    const float* hin = feat;
    int ldh = ldf;
    if (net.head_extra_dim > 0) {                                                        // cat([x, data.u_ref])  gnn_controller.py:46
      float* hcat = (float*)R.ws.alloc((size_t)rows * (F + net.head_extra_dim) * 4);
      if (!R.dry) {
        CHAIN_CALL(gcbf_copy2d(feat, ldf, hcat, F + net.head_extra_dim, rows, F, R.st));
        CHAIN_CALL(gcbf_copy2d(head_extra, net.head_extra_dim, hcat + F, F + net.head_extra_dim, rows, net.head_extra_dim, R.st));
        R.launched(2);
      }
      hin = hcat; ldh = F + net.head_extra_dim;
    }
    const float* y; int ldy;
    if (int rc = mlp_forward(R, net.head, net.n_head, hin, ldh, rows, (chain_head && feat_h.buf) ? &feat_h : nullptr,
                             chain_head ? feat_amax : nullptr, 0, isg + o_head, us + o_head, vs + o_head, save ? &ctx->head : nullptr, out,
                             ld_out, true, nullptr, &y, &ldy, nullptr)) return rc;
  }
  if (ctx) { ctx->msg = msg; ctx->att = att; }
  return 0;
}

int net_backward(Run& R, const gcbf_net_desc& net, const NetCtx& ctx, const int32_t* rowptr, const int64_t* row_index,
                 const float* d_out, int ld_dout, float* d_edge_attr, bool skip_wgrad, cudaEvent_t gamma_done) {
  const int E = ctx.E, Nn = ctx.Nn, rows = ctx.R;
  const int nd = net.node_dim, C = net.phi_dim;
  const float* d_feat = d_out;
  int ld_dfeat = ld_dout;
  const void* d_feat_amax = nullptr;
  H16 d_feat_h{};
  const gcbf_linear_desc& GL = net.gamma[net.n_gamma - 1];
  const bool g_colsum = !skip_wgrad && GL.gW && GL.gb;
  if (net.n_head > 0) {
    void* slot = R.amax_slot();
    const float* d_hin; int ld_dhin; bool valid;
    // without a concatenated u_ref (CBF) the head's input gradient IS gamma's output gradient: emitted as a companion when both
    // sides are tensor-core layers (with gamma's last bias gradient = its column sums)
    const bool direct = net.head_extra_dim == 0;
    if (int rc = mlp_backward(R, net.head, net.n_head, ctx.head, d_out, ld_dout, nullptr, false, true, nullptr, 0, false, nullptr, slot, skip_wgrad,
                              direct ? &d_feat_h : nullptr, GL.K, g_colsum ? GL.gb : nullptr, &d_hin, &ld_dhin, &valid)) return rc;
    d_feat = d_hin; ld_dfeat = ld_dhin;         // the first F columns of d_hin (strided view when u_ref was concatenated)
    if (valid) d_feat_amax = slot;              // max over all of d_hin >= max over the d_feat columns: a valid (pow2) scale bound
  }
  const float* d_gin; int ld_dgin;
  if (int rc = mlp_backward(R, net.gamma, net.n_gamma, ctx.gamma, d_feat, ld_dfeat, d_feat_h.buf ? &d_feat_h : nullptr, g_colsum, true, nullptr, 0,
                            false, d_feat_amax, nullptr, skip_wgrad, nullptr, 0, nullptr, &d_gin, &ld_dgin, nullptr)) return rc;
  if (gamma_done && !R.dry) CHAIN_CUDA(cudaEventRecord(gamma_done, R.st));     // head + gamma gradients of this pass are enqueued
  const float* d_gin_all = d_gin;
  int ld_dga = ld_dgin;
  if (row_index) {
    float* z = (float*)R.ws.alloc((size_t)Nn * (C + nd) * 4);
    if (!R.dry) {
      CHAIN_CUDA(cudaMemsetAsync(z, 0, (size_t)Nn * (C + nd) * 4, R.st));
      CHAIN_CALL(gcbf_rows_scatter(d_gin, ld_dgin, row_index, z, C + nd, rows, C + nd, R.st));
      R.launched(1);
    }
    d_gin_all = z; ld_dga = C + nd;
  }
  float* d_msg = (float*)R.ws.alloc((size_t)E * C * 4);
  float* d_gate = (float*)R.ws.alloc((size_t)E * 4);
  if (!R.dry) {
    CHAIN_CALL(gcbf_attn_aggr_bwd(E ? ctx.msg : nullptr, C, E ? ctx.att : nullptr, rowptr, Nn, C, d_gin_all, ld_dga, E ? d_msg : nullptr, C,
                                  E ? d_gate : nullptr, 0, R.st));
    R.launched(1);
  }
  // gate MLP backward; its input gradient is accumulated onto the aggregation's d_msg
  void* slot = R.amax_slot();
  bool valid = false;
  if (int rc = mlp_backward(R, net.gate, net.n_gate, ctx.gate, d_gate, 1, nullptr, false, true, d_msg, C, true, nullptr, slot, skip_wgrad, nullptr, 0,
                            nullptr, nullptr, nullptr, &valid)) return rc;
  const float* d_ein; int ld_dein;
  if (int rc = mlp_backward(R, net.phi, net.n_phi, ctx.phi, d_msg, C, nullptr, false, d_edge_attr != nullptr, nullptr, 0, false,
                            valid ? slot : nullptr, nullptr, skip_wgrad, nullptr, 0, nullptr, &d_ein, &ld_dein, nullptr)) return rc;
  if (d_edge_attr && !R.dry && E > 0) {
    CHAIN_CALL(gcbf_copy2d(d_ein + 2 * nd, ld_dein, d_edge_attr, net.edge_dim, E, net.edge_dim, R.st));
    R.launched(1);
  }
  return 0;
}

}  // namespace chain
}  // namespace gcbf

using namespace gcbf;
using namespace gcbf::chain;

static_assert(sizeof(NetCtx) <= sizeof(gcbf_net_ctx), "gcbf_net_ctx too small");
static_assert(sizeof(MlpCtx) <= sizeof(gcbf_mlp_ctx), "gcbf_mlp_ctx too small");

extern "C" int gcbf_set_gemm_impl(int impl) {
  GCBF_REQUIRE(impl >= 0 && impl <= 2, "gcbf_set_gemm_impl: %d", impl);
  chain::g_gemm_impl = impl;
  return GCBF_OK;
}

extern "C" long long gcbf_launch_count(int reset) {
  const long long v = chain::g_launches.load();
  if (reset) chain::g_launches.store(0);
  return v;
}

extern "C" int gcbf_timing_enable(int on) {
  chain::g_timing = on != 0;
  if (!on) {
    for (auto& r : chain::g_recs) { chain::g_event_pool.push_back(r.e0); chain::g_event_pool.push_back(r.e1); }
    chain::g_recs.clear();
  }
  return GCBF_OK;
}

extern "C" int gcbf_timing_collect(gcbf_time_rec* out, int max_records, int* count) {
  GCBF_REQUIRE(count && (out || max_records == 0), "gcbf_timing_collect: bad arguments");
  GCBF_CUDA_OK(cudaDeviceSynchronize());
  int n = 0;
  for (auto& r : chain::g_recs) {
    if (n < max_records) {
      float ms = 0.f;
      cudaEventElapsedTime(&ms, r.e0, r.e1);
      out[n].ms = ms; out[n].flops = r.flops; out[n].kind = r.kind; out[n].M = r.M; out[n].N = r.N; out[n].K = r.K;
      ++n;
    }
    chain::g_event_pool.push_back(r.e0);
    chain::g_event_pool.push_back(r.e1);
  }
  *count = (int)chain::g_recs.size();
  chain::g_recs.clear();
  return GCBF_OK;
}

namespace gcbf { namespace chain {
static int64_t g_dummy_idx;
static float g_dummy_f;
// workspace bytes of a forward: the same allocation sequence, nothing launched
size_t net_fwd_bytes(const gcbf_net_desc& net, int64_t E, int Nn, int rows, bool has_row_index, bool save) {
  Run R(nullptr, 0, nullptr, true);
  NetCtx ctx;
  if (net_forward(R, net, nullptr, nullptr, nullptr, nullptr, E, Nn, has_row_index ? &g_dummy_idx : nullptr, rows, nullptr, &g_dummy_f,
                  net.n_head ? net.head[net.n_head - 1].N : net.gamma[net.n_gamma - 1].N, save ? &ctx : nullptr)) return 0;
  return R.ws.off;
}
// workspace bytes of a backward for a forward of these sizes (a dry forward supplies a context with the same companion layout)
size_t net_bwd_bytes(const gcbf_net_desc& net, int64_t E, int Nn, int rows, bool has_row_index, bool need_d_edge_attr, bool skip_wgrad) {
  Run F(nullptr, 0, nullptr, true);
  NetCtx ctx;
  const int64_t* ri = has_row_index ? &g_dummy_idx : nullptr;
  const int od = net.n_head ? net.head[net.n_head - 1].N : net.gamma[net.n_gamma - 1].N;
  if (net_forward(F, net, nullptr, nullptr, nullptr, nullptr, E, Nn, ri, rows, nullptr, &g_dummy_f, od, &ctx)) return 0;
  Run B(nullptr, 0, nullptr, true);
  if (net_backward(B, net, ctx, nullptr, ri, &g_dummy_f, od, need_d_edge_attr ? &g_dummy_f : nullptr, skip_wgrad)) return 0;
  return B.ws.off;
}
}}  // namespace gcbf::chain

extern "C" size_t gcbf_net_forward_workspace_bytes(const gcbf_net_desc* net, int64_t num_edges, int num_nodes, int rows, int save_ctx) {
  if (check_net(net)) return 0;
  return net_fwd_bytes(*net, num_edges, num_nodes, rows, true, save_ctx != 0) + 1024;      // (upper bound: assumes a row selection)
}

extern "C" size_t gcbf_net_backward_workspace_bytes(const gcbf_net_desc* net, int64_t num_edges, int num_nodes, int rows, int need_d_edge_attr) {
  if (check_net(net)) return 0;
  return net_bwd_bytes(*net, num_edges, num_nodes, rows, true, need_d_edge_attr != 0, false) + 1024;
}

extern "C" int gcbf_net_forward(const gcbf_net_desc* net, const float* x, const float* edge_attr, const int64_t* edge_index,
                                const int32_t* rowptr, int64_t num_edges, int num_nodes, const int64_t* row_index, int rows,
                                const float* head_extra, float* out, int ld_out, void* workspace, size_t workspace_bytes,
                                gcbf_net_ctx* ctx, void* stream) {
  if (int rc = check_net(net)) return rc;
  GCBF_REQUIRE(num_edges >= 0 && num_edges < (1ll << 31) && num_nodes >= 0 && rows >= 0, "gcbf_net_forward: bad sizes");
  GCBF_REQUIRE(out && rowptr && (num_nodes == 0 || x) && (num_edges == 0 || (edge_attr && edge_index)), "gcbf_net_forward: null pointer");
  GCBF_REQUIRE(row_index || rows == num_nodes, "gcbf_net_forward: rows != num_nodes needs row_index");
  GCBF_REQUIRE(net->head_extra_dim == 0 || head_extra, "gcbf_net_forward: head_extra is null");
  GCBF_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "gcbf_net_forward: workspace must be 256-byte aligned");
  const size_t need = net_fwd_bytes(*net, num_edges, num_nodes, rows, row_index != nullptr, ctx != nullptr);
  if (need > workspace_bytes) { set_error("gcbf_net_forward: workspace too small (%zu needed, %zu given)", need, workspace_bytes); return GCBF_E_WORKSPACE; }
  Run R(workspace, workspace_bytes, as_stream(stream), false);
  NetCtx* c = reinterpret_cast<NetCtx*>(ctx);
  int rc = net_forward(R, *net, x, edge_attr, edge_index, rowptr, num_edges, num_nodes, row_index, rows, head_extra, out, ld_out, c);
  if (c) { c->rowptr = rowptr; c->row_index = row_index; }
  return R.finish(rc, "gcbf_net_forward");
}

extern "C" int gcbf_net_backward(const gcbf_net_desc* net, const gcbf_net_ctx* ctx, const float* d_out, int ld_dout, float* d_edge_attr,
                                 int skip_wgrad, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = check_net(net)) return rc;
  GCBF_REQUIRE(ctx && d_out && workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "gcbf_net_backward: bad arguments");
  const NetCtx& c = *reinterpret_cast<const NetCtx*>(ctx);
  const size_t need = net_bwd_bytes(*net, c.E, c.Nn, c.R, c.row_index != nullptr, d_edge_attr != nullptr, skip_wgrad != 0);
  if (need > workspace_bytes) { set_error("gcbf_net_backward: workspace too small (%zu needed, %zu given)", need, workspace_bytes); return GCBF_E_WORKSPACE; }
  Run R(workspace, workspace_bytes, as_stream(stream), false);
  int rc = net_backward(R, *net, c, c.rowptr, c.row_index, d_out, ld_dout, d_edge_attr, skip_wgrad != 0);
  return R.finish(rc, "gcbf_net_backward");
}

// ---- bare MLP ---------------------------------------------------------------------------------------------------------------
static int mlp_fwd_run(Run& R, const gcbf_linear_desc* layers, int n, int refresh, const float* x, int ldx, int rows, float* out, int ld_out,
                       MlpCtx* ctx) {
  const gcbf_linear_desc* all[GCBF_MAX_MLP_LAYERS];
  for (int i = 0; i < n; ++i) all[i] = &layers[i];
  const float *isg[GCBF_MAX_MLP_LAYERS], *us[GCBF_MAX_MLP_LAYERS], *vs[GCBF_MAX_MLP_LAYERS];
  if (int rc = sn_power_iter(R, all, n, ctx != nullptr, isg, us, vs)) return rc;
  if (refresh) { if (int rc = refresh_weight_companions(R, all, n)) return rc; }
  const float* y; int ldy;
  return mlp_forward(R, layers, n, x, ldx, rows, nullptr, nullptr, 0, isg, us, vs, ctx, out, ld_out, true, nullptr, &y, &ldy, nullptr);
}

extern "C" size_t gcbf_mlp_forward_workspace_bytes(const gcbf_linear_desc* layers, int n_layers, int rows, int save_ctx) {
  if (!layers || check_mlp(layers, n_layers, "gcbf_mlp_forward_workspace_bytes")) return 0;
  Run R(nullptr, 0, nullptr, true);
  MlpCtx ctx;
  static float dummy;
  if (mlp_fwd_run(R, layers, n_layers, 0, &dummy, layers[0].K, rows, &dummy, layers[n_layers - 1].N, save_ctx ? &ctx : nullptr)) return 0;
  return R.ws.off + 1024;
}

extern "C" size_t gcbf_mlp_backward_workspace_bytes(const gcbf_linear_desc* layers, int n_layers, int rows) {
  if (!layers || check_mlp(layers, n_layers, "gcbf_mlp_backward_workspace_bytes")) return 0;
  Run F(nullptr, 0, nullptr, true);
  MlpCtx ctx;
  static float dummy;
  if (mlp_fwd_run(F, layers, n_layers, 0, &dummy, layers[0].K, rows, &dummy, layers[n_layers - 1].N, &ctx)) return 0;
  Run B(nullptr, 0, nullptr, true);
  if (mlp_backward(B, layers, n_layers, ctx, &g_dummy_f, layers[n_layers - 1].N, nullptr, false, true, nullptr, 0, false, nullptr, nullptr, false, nullptr, 0, nullptr,
                   nullptr, nullptr, nullptr)) return 0;
  return B.ws.off + 1024;
}

extern "C" int gcbf_mlp_forward(const gcbf_linear_desc* layers, int n_layers, int refresh_weights, const float* x, int ldx, int rows,
                                float* out, int ld_out, void* workspace, size_t workspace_bytes, gcbf_mlp_ctx* ctx, void* stream) {
  GCBF_REQUIRE(layers, "gcbf_mlp_forward: null layers");
  if (int rc = check_mlp(layers, n_layers, "gcbf_mlp_forward")) return rc;
  GCBF_REQUIRE(rows >= 0 && out && (rows == 0 || x) && ldx >= layers[0].K && ld_out >= layers[n_layers - 1].N, "gcbf_mlp_forward: bad arguments");
  GCBF_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "gcbf_mlp_forward: workspace must be 256-byte aligned");
  Run R(workspace, workspace_bytes, as_stream(stream), false);
  int rc = mlp_fwd_run(R, layers, n_layers, refresh_weights, x, ldx, rows, out, ld_out, reinterpret_cast<MlpCtx*>(ctx));
  return R.finish(rc, "gcbf_mlp_forward");
}

extern "C" int gcbf_mlp_backward(const gcbf_linear_desc* layers, int n_layers, const gcbf_mlp_ctx* ctx, const float* d_out, int ld_dout,
                                 float* d_x, int skip_wgrad, void* workspace, size_t workspace_bytes, void* stream) {
  GCBF_REQUIRE(layers && ctx && d_out, "gcbf_mlp_backward: null pointer");
  if (int rc = check_mlp(layers, n_layers, "gcbf_mlp_backward")) return rc;
  GCBF_REQUIRE(workspace && (reinterpret_cast<uintptr_t>(workspace) & 255) == 0, "gcbf_mlp_backward: workspace must be 256-byte aligned");
  Run R(workspace, workspace_bytes, as_stream(stream), false);
  const MlpCtx& c = *reinterpret_cast<const MlpCtx*>(ctx);
  int rc = mlp_backward(R, layers, n_layers, c, d_out, ld_dout, nullptr, false, d_x != nullptr, d_x, layers[0].K, false, nullptr, nullptr,
                        skip_wgrad != 0, nullptr, 0, nullptr, nullptr, nullptr, nullptr);
  return R.finish(rc, "gcbf_mlp_backward");
}
