"""Vectorised rollouts on the device (SURVEY section 8f-2): `num_envs` independent copies of one environment -- each with its own
initial state, obstacles and goal set -- advance as ONE batch per step.

The reference's data collection is one environment stepped from Python (gcbf/trainer/trainer.py:60-70): per env step one actor
forward on a single 16-agent graph (gcbf/algo/gcbf.py:128-139), one `env.step` (simple_car.py:146-176: u_ref, clamp, dynamics,
radius graph, collision masks) and one `unsafe_mask(...).any()` host sync -- ~5 ms of host time per 16-agent step (SURVEY section 6).
Here one `step()` is: u_ref for all envs (`gcbf_u_ref_multi`, per-env goals), ONE batched radius graph + edge features, ONE actor
forward over the block-diagonal batch, the unsafe masks in one launch, ONE dynamics launch (`gcbf_step_fwd_multi`, every env is a
single graph -> reach-freeze branch), and an append of all `num_envs` graphs to the device-resident replay ring with the
safe / unsafe flags staying on the device.  The only host sync per step is the batched radius graph's edge count.

Episode semantics follow the reference's `step`: an env is done when t reaches max_episode_steps or when all its agents are
within dist2goal of their goals.  Two ways to start the next episode:
  - host resets (reset_seed=None, the default): env.reset() per finished env; "all agents reached" is checked on the device and the
    flags are read back every `reset_check_every` steps, so a finished env may run a few extra steps before it is re-sampled (its
    agents are frozen at their goals by then);
  - device resets (reset_seed=<int>): per-env step and episode counters live on the device, and after every dynamics step ONE
    `gcbf_env_reset_batch` launch (env/device_reset.py) re-samples every done env in place, so it starts its next episode on the very
    next step.  No host reads of the done flags.
"""
import ctypes
from typing import Callable, Dict, Optional, Sequence

import numpy as np
import torch

from .. import _C, ops
from ..data import Data


class VectorRollout:
    def __init__(self, env, algo, num_envs: int, reset_check_every: int = 16, states: Optional[torch.Tensor] = None,
                 goals: Optional[torch.Tensor] = None, reset_seed: Optional[int] = None):
        """states [num_envs * N, s] / goals [num_envs * n, goal_dim]: explicit initial conditions (e.g. synthetic BASELINE states:
        the reference's rejection sampler cannot place >~ 290 agents, SURVEY section 0); default: env.reset() per env.

        reset_seed: None keeps the host resets above.  An integer switches to device resets: the initial states are episode 0 of every
        env drawn by `gcbf_env_reset_batch` with this seed, and every done env is re-sampled on the device right after the step that
        finished it (env e's episode k depends only on (reset_seed, e, k)).  In that mode the per-env step counters `t_dev` and
        episode counters `episode` are device tensors and the host array `self.t` is NOT authoritative (it counts steps since
        construction); a reset that cannot place its points raises RuntimeError at the next step's edge-count sync (or
        `check_resets()`)."""
        self.env, self.algo, self.B = env, algo, int(num_envs)
        self.n, self.N = env.num_agents, env.nodes_per_graph
        self.dev = env.device
        self.reset_check_every = reset_check_every
        self.states: Optional[torch.Tensor] = None       # [B * N, s]
        self.goals: Optional[torch.Tensor] = None        # [B * n, goal_dim]
        self.t = np.zeros(self.B, dtype=np.int64)
        self.steps = 0
        self._done_host = None
        self._auto_reset = states is None
        self.reset_seed = None if reset_seed is None else int(reset_seed)
        if self.reset_seed is not None:
            if states is not None:
                raise ValueError('VectorRollout: reset_seed draws the initial states on the device; do not pass states / goals')
            self._auto_reset = False
            self._init_device_resets()
        elif states is None:
            self.reset()
        else:
            self.states = states.to(self.dev, torch.float32).contiguous().clone()
            self.goals = goals.to(self.dev, torch.float32).contiguous().clone()

    # ---- device side: episode management by gcbf_env_reset_batch ------------------------------------------------------------
    def _init_device_resets(self):
        from ..env.device_reset import reset_spec
        env, B = self.env, self.B
        self.states = torch.zeros(B * self.N, env.state_dim, device=self.dev, dtype=torch.float32)
        self.goals = torch.zeros(B * self.n, reset_spec(env)['goal_dim'], device=self.dev, dtype=torch.float32)
        self.t_dev = torch.full((B,), int(env.max_episode_steps), device=self.dev, dtype=torch.int32)    # every env is due
        self.episode = torch.full((B,), -1, device=self.dev, dtype=torch.int32)                          # -> episode 0
        self._failed = torch.zeros(B, device=self.dev, dtype=torch.int32)
        self._failed_host = torch.zeros(B, dtype=torch.int32).pin_memory()
        self._failed_ev = None
        self._device_reset(None)
        # as after host resets, the env's own goal set (read where a batch carries no per-graph goals) is the last env's
        env.set_goal(self.goals[(B - 1) * self.n:].clone())

    def _device_reset(self, reach: Optional[torch.Tensor]):
        """One gcbf_env_reset_batch launch over the batch and an asynchronous copy of the failure flags (read by check_resets)."""
        from ..env.device_reset import reset_batch
        reset_batch(self.env, self.states, self.goals, self.t_dev, self.episode, self._failed, self.reset_seed, reach=reach)
        self._failed_host.copy_(self._failed, non_blocking=True)
        self._failed_ev = torch.cuda.Event()
        self._failed_ev.record()

    def check_resets(self):
        """Raise RuntimeError if the last device reset could not place an env's agents or goals (waits for that reset only)."""
        if self.reset_seed is None or self._failed_ev is None:
            return
        from ..env.device_reset import raise_on_failure
        self._failed_ev.synchronize()
        self._failed_ev = None
        raise_on_failure(self.env, self._failed_host.numpy())

    # ---- host side: initial conditions (the reference's rejection sampler, one env at a time) -------------------------
    def _sample_one(self):
        data = self.env.reset()
        return data.states.detach().clone(), self.env._goal.detach().clone()

    def reset(self, which=None):
        idx = range(self.B) if which is None else which
        if self.states is None:
            st, gl = self._sample_one()
            self.states = st.new_zeros(self.B * self.N, st.shape[1])
            self.goals = gl.new_zeros(self.B * self.n, gl.shape[1])
        for i in idx:
            st, gl = self._sample_one()
            self.states[i * self.N:(i + 1) * self.N] = st
            self.goals[i * self.n:(i + 1) * self.n] = gl
            self.t[i] = 0

    # ---- one vectorised step ------------------------------------------------------------------------------------------------
    def keep(self, which):
        """Keep only the environments `which` (ascending indices into the current batch), in that order: the others drop out of the
        batch and cost nothing from the next step on."""
        if self.reset_seed is not None:
            raise NotImplementedError('VectorRollout.keep: device resets draw by env id; dropping envs is not supported with reset_seed')
        idx = torch.as_tensor(np.asarray(which, dtype=np.int64))
        nodes = (idx.unsqueeze(1) * self.N + torch.arange(self.N)).reshape(-1).to(self.dev)
        agents = (idx.unsqueeze(1) * self.n + torch.arange(self.n)).reshape(-1).to(self.dev)
        self.states = self.states[nodes].contiguous()
        self.goals = self.goals[agents].contiguous()
        self.t = self.t[idx.numpy()]
        self.B = int(idx.numel())
        self._done_host = None

    def step(self, prob: float = 0.0, store: bool = True, policy: Optional[Callable] = None) -> Dict[str, torch.Tensor]:
        """All envs advance one step under the actor (each env's action zeroed with probability `prob`, the reference's
        exploration schedule gcbf.py:131-132), or under `policy(batch)` -- e.g. `algo.apply_batch`, the test-time controller --
        which gets the collated batch with u_ref and the per-env goal sets (`batch.goal`).  Returns device tensors: reach [B, n],
        collision [B, n] (after the step), is_safe [B] (before the step: what the stored graph is labelled with, gcbf.py:133-137),
        action, and the step's inputs states [B * N, s] (pre-step), u_ref [B * n, a] and goals [B * n, goal_dim] (with device resets,
        tensors no later step or reset writes to); plus edge_count."""
        if policy is None:
            with torch.no_grad():
                return self._step(prob, store, None)
        return self._step(prob, store, policy)

    def _step(self, prob: float, store: bool, policy: Optional[Callable]) -> Dict[str, torch.Tensor]:
        env, B, n, N = self.env, self.B, self.n, self.N
        cfg = env._cfg(B)
        st, ld = ops._mat(self.states)
        goal, ldg = ops._mat(self.goals)
        a_dim = env.action_dim
        u_ref = torch.empty(B * n, a_dim, device=self.dev, dtype=torch.float32)
        _C.call('gcbf_u_ref_multi', ctypes.byref(cfg), _C.ptr(st), ld, _C.ptr(goal), ldg, _C.ptr(env._gain()), _C.ptr(u_ref))
        data = env.add_communication_links(env.make_graph(self.states))          # ONE radius graph + edge features for all envs
        if self.reset_seed is not None:
            self.check_resets()                      # the edge count above synchronised: the last reset's flags are on the host
        data.update(Data(u_ref=u_ref))
        if policy is None:
            action = self.algo.actor(data)                                       # ONE actor forward (block-diagonal batch)
        else:
            data.update(Data(goal=self.goals))
            action = policy(data).detach()
        if prob > 0:
            keep = torch.from_numpy((np.random.rand(B) >= prob).astype(np.float32)).to(self.dev, non_blocking=True)
            action = action * keep.repeat_interleave(n).unsqueeze(1)
        masks = env._masks(data)
        is_safe = ~masks[1].view(B, n).any(dim=1)
        if store:
            buf = self.algo.buffer
            if not hasattr(buf, 'append_batch'):
                raise RuntimeError('vectorised rollouts store into the device replay ring: call algo.use_device_replay() first')
            buf.append_batch(self.states.view(B, N, -1), u_ref.view(B, n, a_dim), is_safe, self.goals.view(B, n, -1))
        nxt = torch.empty_like(st)
        pass_mask = torch.empty(B * n, a_dim, device=self.dev, dtype=torch.uint8)
        # every env is a SINGLE graph in the reference's loop: reach-freeze branch of dynamics() (dubins_car.py:126-130)
        _C.call('gcbf_step_fwd_multi', ctypes.byref(cfg), _C.ptr(st), ld, _C.ptr(action.contiguous()), _C.ptr(goal), ldg,
                _C.ptr(env._gain()), 1, _C.ptr(nxt), _C.ptr(pass_mask))
        self.states = nxt
        pd = env.POS_DIM
        agents = nxt.view(B, N, -1)[:, :n, :pd]
        reach = (agents - self.goals.view(B, n, -1)[:, :, :pd]).norm(dim=2) < env._params['dist2goal']
        coll_data = env.make_graph(nxt)
        collision = env._masks(coll_data)[2].view(B, n)
        self.t += 1
        self.steps += 1
        out = dict(reach=reach, collision=collision, is_safe=is_safe, action=action, states=st, u_ref=u_ref, goals=self.goals,
                   edge_count=int(data.edge_index.shape[1]))
        if self.reset_seed is not None:
            # done envs start their next episode right away: counters and re-sampling on the device, no host read of the flags
            self.goals = self.goals.clone()          # the returned goals stay those of this step
            self.t_dev += 1
            self._device_reset(reach)
            return out
        # episode ends: time limit known on the host; "all agents reached" read back with a delay (no sync in the common step)
        if not self._auto_reset:
            return out
        if self._done_host is not None and self.steps % self.reset_check_every == 0:
            flags, ev = self._done_host
            ev.synchronize()
            done = np.nonzero(flags.numpy())[0].tolist()
            self._done_host = None
            if done:
                self.reset(done)
        if self._done_host is None:
            flags = torch.empty(B, dtype=torch.bool).pin_memory()
            flags.copy_(reach.all(dim=1), non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
            self._done_host = (flags, ev)
        timeout = np.nonzero(self.t >= env.max_episode_steps)[0].tolist()
        if timeout:
            self.reset(timeout)
        return out


def evaluate_episodes(env, algo, seeds: Sequence[int], rand: Optional[float] = 30, max_iter: int = 30,
                      max_steps: Optional[int] = None) -> Dict[str, object]:
    """Test-time evaluation episodes (reference gcbf/trainer/utils.py:127-223 `eval_ctrl_epi`, one episode per seed) stepped as ONE
    batch: per step, u_ref for every live episode, `algo.apply_batch` (the test-time controller over all of them at once), the dynamics
    with the single-graph reach-freeze branch, the radius graph, reach / collision and the env's per-agent reward.

    Initial states and goals come from `set_seed(seed); env.reset()`, one seed after another, so they are those of a sequential
    evaluation with the same seeds.  An episode ends when its step count reaches `max_steps` (default env.max_episode_steps) or all its
    agents are at their goals; it then drops out of the batch and its statistics stay as they were at its last step.

    Returns per-episode numpy arrays `reward` (sum over steps of the mean agent reward), `length`, `safe` (fraction of agents that never
    collided), `reach` (fraction at their goals at the end) and `success` (both), and `mean` / `std` of each over the episodes (what
    the reference's test.py prints), and every episode's last states `final_states` [S, nodes_per_graph, state_dim]."""
    from ..trainer.utils import set_seed
    from .macbf import MACBF
    if isinstance(algo, MACBF):
        raise NotImplementedError('evaluate_episodes: MACBF has no batched test-time controller; evaluate it one episode at a time')
    if not hasattr(algo, 'apply_batch'):
        raise NotImplementedError(f'evaluate_episodes: {type(algo).__name__} has no apply_batch')
    seeds = [int(s) for s in seeds]
    S, n, N, pd = len(seeds), env.num_agents, env.nodes_per_graph, env.POS_DIM
    max_steps = int(env.max_episode_steps if max_steps is None else max_steps)
    states, goals = [], []
    for s in seeds:
        set_seed(s)
        data = env.reset()
        states.append(data.states.detach().clone())
        goals.append(env._goal.detach().clone())
    vr = VectorRollout(env, algo, S, states=torch.cat(states), goals=torch.cat(goals))
    dev, d2g = vr.dev, env._params['dist2goal']
    reward = torch.zeros(S, device=dev, dtype=torch.float64)
    length = np.zeros(S, dtype=np.int64)
    safe = torch.ones(S, n, device=dev, dtype=torch.bool)
    reach = torch.zeros(S, n, device=dev, dtype=torch.bool)
    prev_reach = (vr.states.view(S, N, -1)[:, :n, :pd] - vr.goals.view(S, n, -1)[:, :, :pd]).norm(dim=2) < d2g
    final = vr.states.view(S, N, -1).clone()
    per_env_reward = torch.vmap(env._reward)                 # the env's own reward, one episode per batch entry
    live = np.arange(S)

    def policy(batch):
        return algo.apply_batch(batch, rand=rand, max_iter=max_iter)

    while live.size:
        out = vr.step(store=False, policy=policy)
        L = live.size
        r = per_env_reward(out['action'].view(L, n, -1), out['reach'], prev_reach, out['collision'])      # [L, n]
        li = torch.from_numpy(live).to(dev)
        reward.index_add_(0, li, r.to(torch.float64).mean(dim=1))
        safe[li] = safe[li] & ~out['collision']
        reach[li] = out['reach']
        length[live] += 1
        prev_reach = out['reach']
        done = (vr.t >= max_steps) | out['reach'].all(dim=1).cpu().numpy()
        if done.any():
            ended = np.nonzero(done)[0]
            final[torch.from_numpy(live[ended]).to(dev)] = vr.states.view(L, N, -1)[torch.from_numpy(ended).to(dev)]
            stay = np.nonzero(~done)[0]
            if stay.size:
                vr.keep(stay)
                prev_reach = prev_reach[torch.from_numpy(stay).to(dev)]
            live = live[stay]
    frac = lambda m: m.sum(dim=1).cpu().numpy() / n           # noqa: E731  (agent counts / n, as eval_ctrl_epi divides)
    res = {'reward': reward.cpu().numpy(), 'length': length, 'safe': frac(safe), 'reach': frac(reach), 'success': frac(safe & reach)}
    stats = list(res.items())
    res['mean'] = {k: float(np.mean(v)) for k, v in stats}
    res['std'] = {k: float(np.std(v)) for k, v in stats}
    res['final_states'] = final.cpu()
    res['seeds'] = seeds
    return res
