"""Outer training loop with the call surface of the reference's `gcbf.trainer.Trainer` (gcbf/trainer/trainer.py:15-141):
`Trainer(env, env_test, algo, log_dir).train(steps, eval_interval, eval_epi)` and `.eval(step, eval_epi)`.

The loop itself is host glue; what it drives -- the actor forward inside `algo.step`, `env.step`, `algo.update`, and
`algo.apply` during evaluation -- is the kernel path.  Behaviour kept from the reference: the exploration probability decays
linearly from 1 to 0 over the run, u_ref is attached to a graph before the algorithm sees it, checkpoints go to
`<log_dir>/models/step_<k>`, the evaluation episodes use the test-time controller and report the mean episode reward, the
fraction of agents that never collided and the fraction that reached their goal.  TensorBoard is optional (scalars are dropped
when it is not installed); progress lines go to stdout.

`Trainer(..., num_envs=B)` runs the same loop vectorised: B training envs step as one batch (algo/rollout.py's VectorRollout with
device episode resets seeded by `seed`), the transitions of one update interval are staged on the device and appended to the replay
ring env-major just before `update()`, and evaluation runs its episodes as one batch (`evaluate_episodes`).  `steps`,
`eval_interval` and the update cadence still count transitions: a vector step is B of them."""
import os
import random
import time
from typing import Dict, Optional, Tuple

import numpy as np
import torch

from ..algo.rollout import VectorRollout, evaluate_episodes
from ..data import Data


class _DropScalars:
    def add_scalar(self, *args, **kwargs):
        return None


def _make_writer(path: str):
    try:
        from torch.utils.tensorboard import SummaryWriter
        return SummaryWriter(log_dir=path)
    except Exception:
        return _DropScalars()


class Trainer:

    def __init__(self, env, env_test, algo, log_dir: str, num_envs: Optional[int] = None, seed: int = 0):
        """num_envs=None: the reference's loop, one env transition at a time.  num_envs=B: the vectorised loop (module docstring); it
        needs B to divide algo.batch_size into segments of at least 3 steps (the update's seg_len), an algorithm with a device replay
        ring and no data-parallel group, and `seed` keys the device episode resets."""
        self.env, self.env_test, self.algo = env, env_test, algo
        self.num_envs = None if num_envs is None else int(num_envs)
        self.seed = int(seed)
        if self.num_envs is not None:
            self._check_vectorised()
        self.log_dir = log_dir
        self.model_dir = os.path.join(log_dir, 'models')
        os.makedirs(self.model_dir, exist_ok=True)
        self.writer = _make_writer(os.path.join(log_dir, 'summary'))

    def _check_vectorised(self):
        from ..algo.macbf import MACBF
        algo, B = self.algo, self.num_envs
        if isinstance(algo, MACBF):
            raise NotImplementedError('Trainer(num_envs=...): MACBF has no device replay ring; train it with num_envs=None')
        if getattr(algo, 'process_group', None) is not None:
            raise NotImplementedError('Trainer(num_envs=...): data-parallel training (algo.process_group) is not supported')
        if B < 1 or algo.batch_size % B != 0 or algo.batch_size // B < 3:
            raise ValueError(f'Trainer(num_envs={B}): batch_size {algo.batch_size} must be a multiple of num_envs with at least 3 '
                             'vector steps per update interval (the update samples segments of 3 consecutive steps)')
        if not getattr(algo, 'device_replay', False):
            if algo.buffer.size or algo.memory.size:
                raise ValueError('Trainer(num_envs=...): the algorithm already holds host replay data; the vectorised loop needs '
                                 'algo.use_device_replay() before any data is collected')
            algo.use_device_replay()

    # ---- rollout --------------------------------------------------------------------------------------------
    @staticmethod
    def _with_u_ref(env, graph):
        graph.update(Data(u_ref=env.u_ref(graph)))
        return graph

    def _rollout_step(self, graph, explore_prob: float):
        """One environment transition of the training env; returns the graph the next transition starts from."""
        env, algo = self.env, self.algo
        self._with_u_ref(env, graph)
        action = algo.step(graph, prob=explore_prob)
        nxt, reward, done, _ = env.step(action)
        self._with_u_ref(env, nxt)
        algo.post_step(graph, action, reward, done, nxt)
        return env.reset() if done else nxt

    # ---- training -------------------------------------------------------------------------------------------
    def train(self, steps: int, eval_interval: int, eval_epi: int):
        if self.num_envs is not None:
            return self._train_vectorised(steps, eval_interval, eval_epi)
        t0 = time.time()
        graph = self.env.reset()
        last_update: Optional[Dict[str, float]] = None
        for k in range(steps):
            step = k + 1
            graph = self._rollout_step(graph, explore_prob=1.0 - k / steps)
            if self.algo.is_update(step):
                last_update = self.algo.update(step, self.writer)
            if eval_interval > 0 and step % eval_interval == 0:
                self._checkpoint_and_report(step, eval_epi, last_update, time.time() - t0)
        print(f'> Done in {time.time() - t0:.0f} seconds')

    def _make_rollout(self):
        return VectorRollout(self.env, self.algo, self.num_envs, reset_seed=self.seed)

    def _train_vectorised(self, steps: int, eval_interval: int, eval_epi: int):
        """Vector step k moves B envs one transition each (transitions k B + 1 .. (k + 1) B) under exploration probability
        1 - k B / steps per env.  T = batch_size / B vector steps make one update interval; their (states, u_ref, is_safe, goals)
        are staged on the device and appended env-major -- env 0's T steps in order, then env 1's, ... -- so a sampled segment of
        the ring is consecutive steps of one env.  update() then runs every batch_size transitions, as in the reference."""
        t0 = time.time()
        B, algo = self.num_envs, self.algo
        T = algo.batch_size // B
        vr = self._make_rollout()
        stage = None
        last_update: Optional[Dict[str, float]] = None
        for k in range((steps + B - 1) // B):
            out = vr.step(prob=1.0 - k * B / steps, store=False)
            parts = (out['states'].view(B, self.env.nodes_per_graph, -1), out['u_ref'].view(B, self.env.num_agents, -1),
                     out['is_safe'], out['goals'].view(B, self.env.num_agents, -1))
            if stage is None:
                stage = [p.new_empty((B, T) + tuple(p.shape[1:])) for p in parts]
            for buf, p in zip(stage, parts):
                buf[:, k % T] = p
            done, step = k * B, (k + 1) * B
            if (k + 1) % T == 0:
                vr.check_resets()
                algo.buffer.append_batch(*(buf.flatten(0, 1) for buf in stage[:2]), stage[2].flatten(),
                                         stage[3].flatten(0, 1))
                last_update = algo.update(step, self.writer)
            if eval_interval > 0 and step // eval_interval > done // eval_interval:
                self._checkpoint_and_report(step, eval_epi, last_update, time.time() - t0)
        print(f'> Done in {time.time() - t0:.0f} seconds')

    def _checkpoint_and_report(self, step: int, eval_epi: int, last_update, elapsed: float):
        if eval_epi > 0:
            reward, info = self.eval(step, eval_epi)
            extras = ''.join(f', {name}: {value}' for name, value in info.items())
            print(f'step: {step}, time: {elapsed:.0f}s, reward: {reward:.2f}{extras}')
        if last_update is not None:
            print(f'step: {step}' + ''.join(f', {name}: {value:.3f}' for name, value in last_update.items()))
        self.algo.save(os.path.join(self.model_dir, f'step_{step}'))
        self.algo._env = self.env                      # eval() pointed the algorithm at the test env

    # ---- evaluation -----------------------------------------------------------------------------------------
    def _episode(self, env) -> Tuple[float, float, torch.Tensor]:
        """One episode under `algo.apply`: (sum over steps of the mean agent reward, fraction of agents that never collided,
        per-agent reach flags of the last step)."""
        never_hit = torch.ones(env.num_agents, dtype=torch.bool)
        reach = torch.zeros(env.num_agents, dtype=torch.bool)
        total = 0.0
        graph = env.reset()
        done = False
        while not done:
            action = self.algo.apply(self._with_u_ref(env, graph))
            graph, reward, done, info = env.step(action)
            total += float(np.mean(reward))
            hit = info.get('collision')
            if hit is not None and len(hit):
                never_hit[torch.as_tensor(hit).cpu().long()] = False
            if 'reach' in info:
                reach = torch.as_tensor(info['reach']).cpu().bool()
        return total, float(never_hit.float().mean()), reach

    def eval(self, step: int, eval_epi: int) -> Tuple[float, dict]:
        """Mean episode reward over `eval_epi` episodes and {'safe': fraction of agents that never collided, 'reach': ...}.
        With num_envs=None, episodes run one by one under algo.apply and 'reach' is the reach fraction of the last episode's last
        step (the reference's report).  With num_envs set, the episodes run as one batch (`evaluate_episodes`) from seeds
        np.random.randint(100000, size=eval_epi) (as the reference's test.py) and 'reach' is the mean over the episodes; the
        random / numpy / torch generator states are restored afterwards, so the training stream does not restart from an
        evaluation seed."""
        if self.num_envs is not None:
            return self._eval_vectorised(step, eval_epi)
        env = self.env_test
        self.algo._env = env
        rewards, safe, reach = [], [], torch.zeros(env.num_agents, dtype=torch.bool)
        for _ in range(eval_epi):
            r, s, reach = self._episode(env)
            rewards.append(r)
            safe.append(s)
        mean_reward, mean_safe = float(np.mean(rewards)), float(np.mean(safe))
        self.writer.add_scalar('test/reward', mean_reward, step)
        self.writer.add_scalar('test/safe_rate', mean_safe, step)
        return mean_reward, {'safe': round(mean_safe, 2), 'reach': round(float(reach.float().mean()), 2)}

    def _eval_vectorised(self, step: int, eval_epi: int) -> Tuple[float, dict]:
        seeds = np.random.randint(100000, size=eval_epi)
        saved = (random.getstate(), np.random.get_state(), torch.get_rng_state(),
                 torch.cuda.get_rng_state_all() if torch.cuda.is_available() else None)
        self.algo._env = self.env_test
        try:
            res = evaluate_episodes(self.env_test, self.algo, seeds)
        finally:
            random.setstate(saved[0])
            np.random.set_state(saved[1])
            torch.set_rng_state(saved[2])
            if saved[3] is not None:
                torch.cuda.set_rng_state_all(saved[3])
        mean_reward, mean_safe = float(res['mean']['reward']), float(res['mean']['safe'])
        self.writer.add_scalar('test/reward', mean_reward, step)
        self.writer.add_scalar('test/safe_rate', mean_safe, step)
        return mean_reward, {'safe': round(mean_safe, 2), 'reach': round(float(res['mean']['reach']), 2)}
