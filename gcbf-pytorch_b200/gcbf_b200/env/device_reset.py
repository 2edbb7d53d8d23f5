"""Batched episode reset on the device (csrc/reset.cu, `gcbf_env_reset_batch`): every done env of a vectorised rollout is re-sampled
in place by the algorithm of its env's reset() -- same box, spacings and obstacle clearance, read from the env class attributes
RESET_AGENT_SPACING / RESET_GOAL_SPACING / RESET_CLEARANCE -- with Philox4x32-10 draws keyed by (seed, env id, episode, stream, draw
index) instead of torch's host generator.  One launch, no host sync."""
import ctypes
from typing import Optional

import numpy as np
import torch

from .. import _C, ops

MAX_TRIES = 200000            # per point set, as sample_separated's max_tries
FAILED_SET = {1: 'agents', 2: 'goals'}


def reset_spec(env) -> dict:
    """The constants of env.reset() as the kernel reads them: fp32 area, squared spacings / clearance (each rounded once from the
    double), obstacle speed limit, obstacle count, goal columns."""
    p = env._params
    R = p[env.RADIUS_KEY]
    clear = env.RESET_CLEARANCE[0] * R + env.RESET_CLEARANCE[1] * p.get('obs_point_r', 0.0)
    agent, goal = env.RESET_AGENT_SPACING * R, env.RESET_GOAL_SPACING * R
    return dict(area=float(np.float32(p['area_size'])), agent_dist=agent, goal_dist=goal, clearance=clear,
                agent_dist2=float(np.float32(agent * agent)), goal_dist2=float(np.float32(goal * goal)),
                clear2=float(np.float32(clear * clear)), obs_speed_limit=float(np.float32(p.get('obs_speed_limit', 0.0))),
                num_obs=int(env.num_obstacles), goal_dim=int(env.RESET_GOAL_DIM))


def reset_batch(env, states: torch.Tensor, goals: torch.Tensor, step_count: torch.Tensor, episode: torch.Tensor, failed: torch.Tensor,
                seed: int, reach: Optional[torch.Tensor] = None, max_steps: Optional[int] = None, max_tries: int = MAX_TRIES,
                first_env: int = 0) -> None:
    """Re-sample in place every env e of the batch with step_count[e] >= max_steps (default env.max_episode_steps) or, given reach
    [B, n] bool, all its agents at their goals.  states [B * N, s] and goals [B * n, >= RESET_GOAL_DIM] fp32; step_count, episode,
    failed int32 [B] (a reset env gets step_count 0, episode + 1 and failed 0, or 1 / 2 when its agents / goals could not be placed in
    max_tries candidates).  Env e draws from the Philox stream of env id first_env + e.  Arguments are checked before any launch."""
    B = int(step_count.numel())
    for name, t, dt in (('step_count', step_count, torch.int32), ('episode', episode, torch.int32), ('failed', failed, torch.int32)):
        if t.dtype != dt or t.numel() != B or not t.is_contiguous():
            raise ValueError(f'reset_batch: {name} must be a contiguous int32 tensor of {B} entries')
    n, N = env.num_agents, env.nodes_per_graph
    spec = reset_spec(env)
    st, ld = ops._mat(states)
    gl, ldg = ops._mat(goals)
    if st.shape[0] != B * N or gl.shape[0] != B * n or st.data_ptr() != states.data_ptr() or gl.data_ptr() != goals.data_ptr():
        raise ValueError(f'reset_batch: states must be [{B * N}, s] and goals [{B * n}, g], written in place')
    if reach is not None and (reach.dtype != torch.bool or reach.numel() != B * n):
        raise ValueError(f'reset_batch: reach must be bool with {B * n} entries')
    _C.require_cuda(states, goals, step_count, episode, failed, reach)
    d = _C.ResetDesc()
    d.seed = int(seed) & ((1 << 64) - 1)
    d.states, d.goals = _C.ptr(st), _C.ptr(gl)
    d.step_count, d.episode, d.failed = _C.ptr(step_count), _C.ptr(episode), _C.ptr(failed)
    d.reach = None if reach is None else _C.ptr(reach.contiguous())
    d.env, d.num_envs, d.num_agents, d.num_obs = ops.ENV_IDS[env.ENV_NAME], B, n, spec['num_obs']
    d.ld_state, d.ld_goal, d.goal_dim = ld, ldg, min(spec['goal_dim'], gl.shape[1])
    d.max_steps = int(env.max_episode_steps if max_steps is None else max_steps)
    d.max_tries, d.first_env = int(max_tries), int(first_env)
    d.area, d.agent_dist2, d.goal_dist2, d.clear2 = spec['area'], spec['agent_dist2'], spec['goal_dist2'], spec['clear2']
    d.obs_speed_limit = spec['obs_speed_limit']
    _C.call('gcbf_env_reset_batch', ctypes.byref(d))


def raise_on_failure(env, failed: np.ndarray, first_env: int = 0, max_tries: int = MAX_TRIES):
    """RuntimeError naming the first env whose reset could not place a point set (failed: host int32 [B] from reset_batch)."""
    bad = np.nonzero(failed)[0]
    if bad.size == 0:
        return
    e, spec = int(bad[0]), reset_spec(env)
    what = FAILED_SET.get(int(failed[e]), f'code {int(failed[e])}')
    spacing = spec['agent_dist'] if what == 'agents' else spec['goal_dist']
    clear = f' and clearance {spec["clearance"]:g} from {spec["num_obs"]} obstacles' if spec['num_obs'] else ''
    raise RuntimeError(f'device reset of env {first_env + e} ({bad.size} env(s) failed): could not place {env.num_agents} {what} with '
                       f'spacing {spacing:g}{clear} in a box of side {spec["area"]:g} within {max_tries} candidates; increase area_size')
