// Batched episode reset (gcbf_env_reset_batch): every done env of a vectorised rollout is re-sampled in place, in ONE launch and
// without a host sync.  One warp per env:
//   1. done?   step counter >= max_steps, or every agent's reach flag set (the reference's `done` of env.step); else return
//   2. obstacles: plain uniform draws of stream kObstacles, one Philox block per obstacle
//   3. agents, then goals: the sequential rejection sampler of env/_sampling.py over the Philox stream of the set -- the 32 lanes test
//      candidates base .. base + 31 against the placed points (shared memory) and the obstacles, the lowest passing candidate is
//      accepted (ballot + ffs) and the search resumes right after it.  The result is exactly that of testing the candidates one by one.
//   4. headings (DubinsCar): stream kHeadings, word 0 the agent's, word 1 its goal's
//   5. step counter = 0, episode counter + 1, failure flag (0, or 1 / 2 when the agents / goals ran out of tries)
#include "common.cuh"
#include "reset_core.h"

namespace gcbf {
namespace reset {

constexpr unsigned kFull = 0xffffffffu;

struct Key {
  uint64_t seed;
  uint32_t env, episode;
};

// count points of stream `tag` into pts[0, count); 0 on success, 1 when the candidates [0, max_tries) ran out first
template <int PD>
__device__ int place(const Key& key, uint32_t tag, float side, float min_dist2, const float* obs, int num_obs, float clear2, int max_tries,
                     int count, float* pts, int lane) {
  int i = 0;
  int64_t base = 0;
  while (i < count) {
    const int64_t k = base + lane;
    bool ok = k < max_tries;
    float c[PD];
    for (int d = 0; d < PD; ++d) c[d] = 0.f;
    if (ok) {
      candidate(key.seed, key.env, key.episode, tag, (uint32_t)k, PD, side, c);
      for (int j = 0; j < i && ok; ++j) ok = !too_close(pts + j * PD, c, PD, min_dist2);
      for (int j = 0; j < num_obs && ok; ++j) ok = !too_close(obs + j * PD, c, PD, clear2);
    }
    const unsigned m = __ballot_sync(kFull, ok);
    if (m) {
      const int w = __ffs(m) - 1;
      for (int d = 0; d < PD; ++d) {
        const float v = __shfl_sync(kFull, c[d], w);
        if (lane == 0) pts[i * PD + d] = v;
      }
      __syncwarp();
      ++i;
      base += w + 1;
    } else {
      base += 32;
      if (base >= max_tries) return 1;
    }
  }
  return 0;
}

template <int ENV>
__global__ void __launch_bounds__(32) env_reset_kernel(gcbf_reset_desc d) {
  constexpr int PD = ENV == GCBF_ENV_SIMPLE_DRONE ? 3 : 2;
  constexpr int SD = ENV == GCBF_ENV_SIMPLE_DRONE ? 6 : 4;
  extern __shared__ float pts[];                      // [0, n): the set being placed, [n, n + o): obstacle positions
  const int e = blockIdx.x, lane = threadIdx.x;
  const int n = d.num_agents, o = d.num_obs, N = n + o;
  bool done = d.step_count[e] >= d.max_steps;
  if (!done && d.reach) {
    bool all = true;
    for (int i = lane; i < n; i += 32) all &= d.reach[(int64_t)e * n + i] != 0;
    done = __all_sync(kFull, all);
  }
  if (!done) return;
  const Key key{d.seed, (uint32_t)(d.first_env + e), (uint32_t)(d.episode[e] + 1)};
  float* obs = pts + n * PD;
  for (int j = lane; j < o; j += 32) {
    float u[4];
    draw4(key.seed, key.env, key.episode, kObstacles, (uint32_t)j, u);
    float s[SD];
    for (int c = 0; c < SD; ++c) s[c] = 0.f;
    for (int c = 0; c < PD; ++c) s[c] = graph::mul_rn(u[c], d.area);
    if (ENV == GCBF_ENV_DUBINS_CAR) {
      s[2] = graph::mul_rn(u[2], 6.28318548202514648f);
      s[3] = graph::mul_rn(u[3], d.obs_speed_limit);
    }
    float* row = d.states + ((int64_t)e * N + n + j) * d.ld_state;
    for (int c = 0; c < SD; ++c) row[c] = s[c];
    for (int c = 0; c < PD; ++c) obs[j * PD + c] = s[c];
  }
  __syncwarp();
  int fail = place<PD>(key, kAgents, d.area, d.agent_dist2, obs, o, d.clear2, d.max_tries, n, pts, lane) ? 1 : 0;
  if (!fail) {
    for (int i = lane; i < n; i += 32) {
      float* row = d.states + ((int64_t)e * N + i) * d.ld_state;
      for (int c = 0; c < SD; ++c) row[c] = c < PD ? pts[i * PD + c] : 0.f;
      if (ENV == GCBF_ENV_DUBINS_CAR) {
        float u[4];
        draw4(key.seed, key.env, key.episode, kHeadings, (uint32_t)i, u);
        row[2] = heading(u[0]);
      }
    }
    __syncwarp();
    fail = place<PD>(key, kGoals, d.area, d.goal_dist2, obs, o, d.clear2, d.max_tries, n, pts, lane) ? 2 : 0;
  }
  if (!fail) {
    for (int i = lane; i < n; i += 32) {
      float* row = d.goals + ((int64_t)e * n + i) * d.ld_goal;
      for (int c = 0; c < d.goal_dim; ++c) row[c] = c < PD ? pts[i * PD + c] : 0.f;
      if (ENV == GCBF_ENV_DUBINS_CAR && d.goal_dim > 2) {
        float u[4];
        draw4(key.seed, key.env, key.episode, kHeadings, (uint32_t)i, u);
        row[2] = heading(u[1]);
      }
    }
  }
  if (lane == 0) {
    d.step_count[e] = 0;
    d.episode[e] = (int32_t)key.episode;
    d.failed[e] = fail;
  }
}

static int check(const gcbf_reset_desc* d) {
  GCBF_REQUIRE(d, "gcbf_env_reset_batch: null descriptor");
  GCBF_REQUIRE(d->env >= GCBF_ENV_SIMPLE_CAR && d->env <= GCBF_ENV_SIMPLE_DRONE, "gcbf_env_reset_batch: unknown env %d", d->env);
  const int pd = d->env == GCBF_ENV_SIMPLE_DRONE ? 3 : 2, sd = d->env == GCBF_ENV_SIMPLE_DRONE ? 6 : 4;
  GCBF_REQUIRE(d->num_envs >= 1 && d->num_agents >= 1 && d->num_obs >= 0, "gcbf_env_reset_batch: bad sizes (%d envs, %d agents, %d obstacles)",
               d->num_envs, d->num_agents, d->num_obs);
  GCBF_REQUIRE(d->env != GCBF_ENV_SIMPLE_CAR || d->num_obs == 0, "gcbf_env_reset_batch: SimpleCar has no obstacles");
  GCBF_REQUIRE(d->first_env >= 0, "gcbf_env_reset_batch: first_env < 0");
  const int64_t N = (int64_t)d->num_agents + d->num_obs;
  GCBF_REQUIRE(N * d->num_envs < (1ll << 31), "gcbf_env_reset_batch: too many nodes");
  GCBF_REQUIRE(N * pd * 4 <= 200 * 1024, "gcbf_env_reset_batch: %lld nodes per env do not fit in shared memory", (long long)N);
  GCBF_REQUIRE(d->states && d->goals && d->step_count && d->episode && d->failed, "gcbf_env_reset_batch: null pointer");
  GCBF_REQUIRE(d->ld_state >= sd, "gcbf_env_reset_batch: ld_state %d < state_dim %d", d->ld_state, sd);
  GCBF_REQUIRE(d->goal_dim >= pd && d->ld_goal >= d->goal_dim, "gcbf_env_reset_batch: goal_dim %d / ld_goal %d (need >= %d)", d->goal_dim,
               d->ld_goal, pd);
  GCBF_REQUIRE(d->max_tries >= 1, "gcbf_env_reset_batch: max_tries must be >= 1");
  GCBF_REQUIRE(d->area > 0.f && d->agent_dist2 >= 0.f && d->goal_dist2 >= 0.f && d->clear2 >= 0.f && d->obs_speed_limit >= 0.f,
               "gcbf_env_reset_batch: area / distances must be finite and non-negative");
  return 0;
}

template <int ENV>
static int launch(const gcbf_reset_desc& d, cudaStream_t st) {
  const int pd = ENV == GCBF_ENV_SIMPLE_DRONE ? 3 : 2;
  const size_t smem = (size_t)(d.num_agents + d.num_obs) * pd * 4;
  if (smem > 48 * 1024) GCBF_CUDA_OK(cudaFuncSetAttribute(env_reset_kernel<ENV>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  env_reset_kernel<ENV><<<d.num_envs, 32, smem, st>>>(d);
  GCBF_LAUNCH_OK();
  return 0;
}

}  // namespace reset
}  // namespace gcbf

extern "C" int gcbf_env_reset_batch(const gcbf_reset_desc* d, void* stream) {
  using namespace gcbf::reset;
  if (int rc = check(d)) return rc;
  cudaStream_t st = gcbf::as_stream(stream);
  switch (d->env) {
    case GCBF_ENV_SIMPLE_CAR: return launch<GCBF_ENV_SIMPLE_CAR>(*d, st);
    case GCBF_ENV_DUBINS_CAR: return launch<GCBF_ENV_DUBINS_CAR>(*d, st);
    default: return launch<GCBF_ENV_SIMPLE_DRONE>(*d, st);
  }
}
