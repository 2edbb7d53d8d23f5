"""The training loop timed on the GPU, one step at a time against vectorised: `python tools/train_loop_bench.py`.

Prints one JSON line per entry, and first the card's name and power limit (an absolute time is only worth something next to them):
  interval  one full update interval -- batch_size = 512 transitions of collection and one update() (10 inner iterations) -- through
            Trainer.train(steps=512) with num_envs=None (the reference's loop: one env transition per actor forward / env.step) and
            with num_envs in {8, 32, 128} (VectorRollout with device resets, env-major staging), run alternately; collection time is
            the interval minus the update, timed by synchronising around update()
  reset     a burst of 128 episode resets: host VectorRollout.reset() (env.reset() per env) against ONE gcbf_env_reset_batch of
            128 done envs, SimpleCar at n = 16 and n = 64
  eval      Trainer.eval with 3 episodes one by one (algo.apply) against vectorised (evaluate_episodes), and vectorised with 32
Envs: SimpleCar n = 16 and DubinsCar n = 16 with 8 obstacles (the reference's train.py defaults otherwise).  Nothing is written to the
tree: checkpoints / summaries go to a temporary directory."""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, 'gcbf-pytorch_b200'), os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')):
    sys.path.insert(0, p)

from gcbf_b200.algo.rollout import VectorRollout  # noqa: E402
from gcbf_b200.env import make_env  # noqa: E402
from gcbf_b200.env.device_reset import reset_batch  # noqa: E402
from gcbf_b200.synth import seeded_algo  # noqa: E402
from gcbf_b200.trainer import Trainer  # noqa: E402
from gcbf_b200.trainer.utils import set_seed  # noqa: E402

DEV = torch.device('cuda:0')
ENVS = [('SimpleCar', 16, {}), ('DubinsCar', 16, {'num_obs': 8})]


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:
        out = f'nvidia-smi unavailable: {ex!r}'
    return {'card': out or torch.cuda.get_device_name(0)}


def emit(d):
    print(json.dumps(d), flush=True)


def _setup(name, n, params, num_envs, tmp):
    set_seed(0)
    env, algo = seeded_algo(name, n, DEV, 0, params)
    env_test = make_env(name, n, DEV, params=env._params)
    tr = Trainer(env, env_test, algo, tmp, num_envs=num_envs, seed=0)
    algo._env = env
    spent = {'update': 0.0}
    update = algo.update

    def timed(step, writer=None):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = update(step, writer)
        torch.cuda.synchronize()
        spent['update'] += time.perf_counter() - t0
        return out

    algo.update = timed
    return tr, spent


def interval_leg(name, n, params, reps=3):
    modes = [None, 8, 32, 128]
    runs = {}
    with tempfile.TemporaryDirectory() as tmp:
        for m in modes:
            runs[m] = _setup(name, n, params, m, os.path.join(tmp, str(m)))
            runs[m][0].train(512, 0, 0)                         # warm-up interval (also fills memory, as a running job has)
        res = {m: [] for m in modes}
        for _ in range(reps):
            for m in modes:
                tr, spent = runs[m]
                spent['update'] = 0.0
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                tr.train(512, 0, 0)
                torch.cuda.synchronize()
                wall = time.perf_counter() - t0
                res[m].append((wall, spent['update']))
    for m in modes:
        wall = float(np.median([w for w, _ in res[m]]))
        upd = float(np.median([u for _, u in res[m]]))
        emit({'leg': 'interval', 'env': name, 'n': n, 'obs': params.get('num_obs', 0), 'num_envs': m or 'existing loop',
              'interval_ms': round(wall * 1e3, 1), 'update_ms': round(upd * 1e3, 1), 'collect_ms': round((wall - upd) * 1e3, 1),
              'transitions_per_s': round(512 / max(wall - upd, 1e-9), 0), 'reps': reps})


def reset_leg(n, B=128, reps=5):
    env, algo = seeded_algo('SimpleCar', n, DEV, 0)
    set_seed(0)
    vr = VectorRollout(env, algo, B)
    host = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        vr.reset()
        torch.cuda.synchronize()
        host.append(time.perf_counter() - t0)
    states = torch.zeros(B * n, 4, device=DEV)
    goals = torch.zeros(B * n, 2, device=DEV)
    ep = torch.zeros(B, device=DEV, dtype=torch.int32)
    failed = torch.zeros(B, device=DEV, dtype=torch.int32)
    dev = []
    for r in range(reps + 1):
        t = torch.full((B,), env.max_episode_steps, device=DEV, dtype=torch.int32)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        reset_batch(env, states, goals, t, ep, failed, 0)
        b.record()
        b.synchronize()
        if r:                                                    # the first launch loads the module
            dev.append(a.elapsed_time(b) / 1e3)
    assert int(failed.abs().sum()) == 0
    emit({'leg': 'reset', 'env': 'SimpleCar', 'n': n, 'envs': B, 'host_reset_ms': round(float(np.median(host)) * 1e3, 2),
          'device_reset_ms': round(float(np.median(dev)) * 1e3, 4), 'reps': reps})


def eval_leg(name, n, params):
    with tempfile.TemporaryDirectory() as tmp:
        for m, epi in ((None, 3), (8, 3), (8, 32)):
            tr, _ = _setup(name, n, params, m, os.path.join(tmp, str(m)))
            cbf = {k: v.clone() for k, v in tr.algo.cbf.state_dict().items()}
            np.random.seed(1)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            reward, info = tr.eval(0, epi)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0
            tr.algo.cbf.load_state_dict(cbf)
            emit({'leg': 'eval', 'env': name, 'n': n, 'obs': params.get('num_obs', 0), 'mode': 'vectorised' if m else 'existing loop',
                  'episodes': epi, 'wall_s': round(wall, 2), 'reward': round(reward, 3), **info})


def main():
    assert torch.cuda.is_available(), 'train_loop_bench needs a GPU'
    emit(card())
    for name, n, params in ENVS:
        interval_leg(name, n, params)
    for n in (16, 64):
        reset_leg(n)
    eval_leg('SimpleCar', 16, {})


if __name__ == '__main__':
    main()
