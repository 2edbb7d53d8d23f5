// Per-element arithmetic of the batched episode reset (gcbf_env_reset_batch, csrc/reset.cu), written once for device and host:
// reset.cu's kernel is a loop around these functions, tests/host_driver/reset_host.cpp compiles them with g++ -ffp-contract=off for
// the CPU test-suite, and tests/reset_replica.py restates them in numpy.
//
// Random numbers: counter-based Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11), key = the 64-bit
// seed (low word first), counter = (draw index k, env id, episode number, stream tag).  Draw k of a stream is one Philox block; its
// words 0, 1, 2, 3 are the coordinates of candidate point k (or obstacle k's [x, y, theta, v], or agent k's [heading, goal heading]).
// A word becomes a uniform in [0, 1) as (word >> 8) * 2^-24, exact in fp32.  A draw therefore depends only on
// (seed, env, episode, stream, k), never on which other envs are reset in the same launch.
#pragma once
#include <stdint.h>

#include "graph_core.h"

namespace gcbf {
namespace reset {

enum Stream : uint32_t { kObstacles = 0, kAgents = 1, kGoals = 2, kHeadings = 3 };

struct Philox4 { uint32_t w[4]; };

GCBF_GHD uint32_t mulhi32(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) >> 32); }

GCBF_GHD Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint32_t lo0 = 0xD2511F53u * c0, hi0 = mulhi32(0xD2511F53u, c0);
    const uint32_t lo1 = 0xCD9E8D57u * c2, hi1 = mulhi32(0xCD9E8D57u, c2);
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
  }
  Philox4 o;
  o.w[0] = c0; o.w[1] = c1; o.w[2] = c2; o.w[3] = c3;
  return o;
}

GCBF_GHD float uniform01(uint32_t w) { return (float)(w >> 8) * 5.9604644775390625e-08f; }   // 2^-24

// the four uniforms of draw k of stream `tag` for (env, episode)
GCBF_GHD void draw4(uint64_t seed, uint32_t env, uint32_t episode, uint32_t tag, uint32_t k, float* u) {
  const Philox4 p = philox4x32_10(k, env, episode, tag, (uint32_t)seed, (uint32_t)(seed >> 32));
  for (int i = 0; i < 4; ++i) u[i] = uniform01(p.w[i]);
}

// squared distance sum_d (a_d - b_d)^2, d ascending, every operation rounded on its own (no FMA contraction)
GCBF_GHD float dist2(const float* a, const float* b, int dim) {
  float s = 0.f;
  for (int d = 0; d < dim; ++d) {
    const float diff = graph::sub_rn(a[d], b[d]);
    s = graph::add_rn(s, graph::mul_rn(diff, diff));
  }
  return s;
}

// the rejection rule: candidate c is rejected by point p iff dist2(p, c) <= min_dist2 (min_dist^2 rounded once on the host)
GCBF_GHD bool too_close(const float* p, const float* c, int dim, float min_dist2) { return dist2(p, c, dim) <= min_dist2; }

// candidate point k of a point set: side * u_d per coordinate
GCBF_GHD void candidate(uint64_t seed, uint32_t env, uint32_t episode, uint32_t tag, uint32_t k, int dim, float side, float* c) {
  float u[4];
  draw4(seed, env, episode, tag, k, u);
  for (int d = 0; d < dim; ++d) c[d] = graph::mul_rn(u[d], side);
}

// angle in [-pi, pi) from a uniform: u * 2pi - pi with the fp32 constants
GCBF_GHD float heading(float u) { return graph::sub_rn(graph::mul_rn(u, 6.28318548202514648f), 3.14159274101257324f); }

}  // namespace reset
}  // namespace gcbf
