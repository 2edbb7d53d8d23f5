// TEST INFRASTRUCTURE ONLY: the per-element functions of the batched episode reset (csrc/reset_core.h) built for the host, next to
// CUDA's own Philox4x32-10 (curand_philox4x32_x.h, compiled for the host with QUALIFIERS = static inline).  Compiled by
// tests/test_vector_train_cpu.py with g++ -ffp-contract=off.
#define QUALIFIERS static inline
#include <vector_types.h>
#include <curand_philox4x32_x.h>

#include "reset_core.h"

using namespace gcbf;

extern "C" {

void host_philox(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
  const reset::Philox4 p = reset::philox4x32_10(ctr[0], ctr[1], ctr[2], ctr[3], key[0], key[1]);
  for (int i = 0; i < 4; ++i) out[i] = p.w[i];
}

void curand_philox(const uint32_t* ctr, const uint32_t* key, uint32_t* out) {
  uint4 c;
  c.x = ctr[0]; c.y = ctr[1]; c.z = ctr[2]; c.w = ctr[3];
  uint2 k;
  k.x = key[0]; k.y = key[1];
  const uint4 r = curand_Philox4x32_10(c, k);
  out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}

void host_draw4(uint64_t seed, uint32_t env, uint32_t episode, uint32_t tag, uint32_t k, float* u) {
  reset::draw4(seed, env, episode, tag, k, u);
}

float host_dist2(const float* a, const float* b, int dim) { return reset::dist2(a, b, dim); }

int host_too_close(const float* p, const float* c, int dim, float min_dist2) { return reset::too_close(p, c, dim, min_dist2) ? 1 : 0; }

float host_heading(float u) { return reset::heading(u); }

}  // extern "C"
