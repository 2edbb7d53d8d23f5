// Per-thread last-error string + ABI version.
#include <stdarg.h>
#include "common.cuh"

namespace gcbf {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace gcbf

extern "C" const char* gcbf_last_error(void) { return gcbf::g_err; }
extern "C" int gcbf_abi_version(void) { return 6; }   // 2: fp16-companion tensor-core entry points (gcbf_linear_*_h); 3: chain-level entry points (gcbf_net_*, gcbf_mlp_*, gcbf_step_*); 4: + MACBF kernels (macbf.cu) and the analytic h_dot kernels (jvp.cu), nothing removed; 5: sm_90a build, gcbf_has_tcgen05 renamed gcbf_has_wgmma; later additions within 5 (nothing changed or removed): gcbf_apply_batch + gcbf_apply_batch_workspace_bytes, gcbf_cbf_field + gcbf_cbf_field_workspace_bytes (gcbf_field_desc), gcbf_env_reset_batch (gcbf_reset_desc); 6: gcbf_linear_*_h take gcbf_h16 descriptors and `products` (the raw-pointer signatures and gcbf_linear_*_t / _tp are gone)

// sizeof() of the ABI structures as this library was compiled (bindings check their mirrors against it):
// 0 gcbf_env_cfg, 1 gcbf_linear_desc, 2 gcbf_net_desc, 3 gcbf_step_desc, 4 gcbf_step_batch, 5 gcbf_step_out, 6 gcbf_net_ctx,
// 7 gcbf_mlp_ctx, 8 gcbf_step_ctx, 9 gcbf_time_rec, 10 gcbf_sn_layer, 11 gcbf_split_desc, 12 gcbf_h16, 13 gcbf_field_desc,
// 14 gcbf_reset_desc
extern "C" size_t gcbf_abi_struct_size(int which) {
  switch (which) {
    case 0: return sizeof(gcbf_env_cfg);
    case 1: return sizeof(gcbf_linear_desc);
    case 2: return sizeof(gcbf_net_desc);
    case 3: return sizeof(gcbf_step_desc);
    case 4: return sizeof(gcbf_step_batch);
    case 5: return sizeof(gcbf_step_out);
    case 6: return sizeof(gcbf_net_ctx);
    case 7: return sizeof(gcbf_mlp_ctx);
    case 8: return sizeof(gcbf_step_ctx);
    case 9: return sizeof(gcbf_time_rec);
    case 10: return sizeof(gcbf_sn_layer);
    case 11: return sizeof(gcbf_split_desc);
    case 12: return sizeof(gcbf_h16);
    case 13: return sizeof(gcbf_field_desc);
    case 14: return sizeof(gcbf_reset_desc);
    default: return 0;
  }
}
