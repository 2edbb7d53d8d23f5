// Internal declarations shared by the chain-level host code (net.cu: one GNN pass / one MLP per call; step.cu: the train step).
#pragma once
#include <atomic>

#include "common.cuh"

namespace gcbf {
namespace chain {

extern std::atomic<long long> g_launches;

// bump allocator over the caller's workspace; `dry` replays the allocation sequence of a call without touching memory
struct Bump {
  uint8_t* base; size_t cap; size_t off; bool overflow;
  void* alloc(size_t bytes) {
    const size_t need = (bytes + 255) & ~size_t(255);
    void* p = base + off;
    off += need;
    if (off > cap) overflow = true;
    return p;
  }
};

struct Run {
  Bump ws; cudaStream_t st; bool dry;
  uint32_t* pool; int pool_left;
  // dry runs bump a fake (never dereferenced, non-null, aligned) base so that "has a buffer" tests behave like the real run
  Run(void* workspace, size_t bytes, cudaStream_t s, bool dry_)
      : ws{dry_ ? reinterpret_cast<uint8_t*>(uintptr_t(1) << 20) : static_cast<uint8_t*>(workspace), dry_ ? ~size_t(0) : bytes, 0, false},
        st(s), dry(dry_), pool(nullptr), pool_left(0) {}
  // one device word for a tensor's max|x| (float bits)
  void* amax_slot() {
    if (pool_left == 0) { pool = static_cast<uint32_t*>(ws.alloc(64 * 4)); pool_left = 64; }
    --pool_left;
    return pool++;
  }
  void launched(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }
  int finish(int rc, const char* what) {
    if (rc == 0 && ws.overflow) { set_error("%s: workspace overflow (%zu > %zu bytes)", what, ws.off, ws.cap); return GCBF_E_WORKSPACE; }
    return rc;
  }
};

#define CHAIN_CALL(expr)            \
  do {                              \
    int _rc = (expr);               \
    if (_rc != 0) return _rc;       \
  } while (0)
#define CHAIN_CUDA(expr) GCBF_CUDA_OK(expr)

struct MlpCtx {
  int n, M;
  const float* acts[GCBF_MAX_MLP_LAYERS + 1];   // acts[0] = input, acts[l + 1] = output of layer l
  int ld[GCBF_MAX_MLP_LAYERS + 1];
  gcbf_h16 acts_h[GCBF_MAX_MLP_LAYERS];          // companion of acts[l] when layer l ran on the tensor cores (buf == nullptr otherwise)
  const float* inv_sigma[GCBF_MAX_MLP_LAYERS];
  const float* u[GCBF_MAX_MLP_LAYERS];           // spectral-norm vectors of THIS forward (snapshots)
  const float* v[GCBF_MAX_MLP_LAYERS];
};

struct NetCtx {
  MlpCtx phi, gate, gamma, head;
  const float* msg; const float* att;
  const int32_t* rowptr; const int64_t* row_index;
  int E, Nn, R;
};

bool use_h(int M, int N, int K);
bool timing_on();      // per-launch CUDA-event timing enabled (gcbf_timing_enable): stream capture is skipped then
int check_net(const gcbf_net_desc* net);
int net_forward(Run& R, const gcbf_net_desc& net, const float* x, const float* edge_attr, const int64_t* edge_index,
                const int32_t* rowptr, int64_t E, int Nn, const int64_t* row_index, int rows, const float* head_extra, float* out,
                int ld_out, NetCtx* ctx, const float* const* inv_sigma_in = nullptr);   // inv_sigma_in: skip the power iteration, use these
int net_backward(Run& R, const gcbf_net_desc& net, const NetCtx& ctx, const int32_t* rowptr, const int64_t* row_index,
                 const float* d_out, int ld_dout, float* d_edge_attr, bool skip_wgrad, cudaEvent_t gamma_done = nullptr);
int check_step(const gcbf_step_desc* d, const gcbf_step_batch* b, const char* what);   // step.cu
int vec_add(Run& R, float* dst, const float* src, int64_t n);
int collect_layers(const gcbf_net_desc& net, const gcbf_linear_desc** all);      // phi, gate, gamma, head in that order
int sn_power_iter(Run& R, const gcbf_linear_desc* const* layers, int n, bool snapshot, const float** inv_sigma, const float** us,
                  const float** vs);
int refresh_weight_companions(Run& R, const gcbf_linear_desc* const* layers, int n);
size_t net_fwd_bytes(const gcbf_net_desc& net, int64_t E, int Nn, int rows, bool has_row_index, bool save);
size_t net_bwd_bytes(const gcbf_net_desc& net, int64_t E, int Nn, int rows, bool has_row_index, bool need_d_edge_attr, bool skip_wgrad);

}  // namespace chain
}  // namespace gcbf
