"""Train-step time with the finite-difference h_dot (the default) and the analytic h_dot (GCBF.params['h_dot'] = 'analytic'), run
alternately in one process on the BASELINE configurations C1-C3.  Device events around each step after a warm-up; prints the median, the peak
device memory of each mode measured with that mode's model alone on the device, the card's name and its power limit.  Exits non-zero if a
configuration failed.

    python tools/hdot_train_bench.py [--steps 10] [--warmup 3] [--configs C1,C2,C3] [--out FILE.json]
"""
import argparse
import gc
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'gcbf-pytorch_b200'))

from gcbf_b200 import synth  # noqa: E402

# BASELINE.md configurations: (env, agents, obstacles, graphs per batch, area)
CONFIGS = {'C1': ('SimpleCar', 16, 0, 1, 4.0), 'C2': ('SimpleCar', 256, 0, 32, 16.0), 'C3': ('DubinsCar', 1024, 32, 64, 32.0)}


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader'], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'
    except (OSError, subprocess.TimeoutExpired):
        power = 'unknown'
    return name, power


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--configs', default='C1,C2,C3')
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('hdot_train_bench needs a CUDA device')
    dev = torch.device('cuda:0')
    name, power = card()
    results, failed = [], False
    for cfg in a.configs.split(','):
        try:
            row = run_config(cfg, a, dev)
        except torch.OutOfMemoryError as e:
            row = dict(config=cfg, error='out of memory: ' + str(e).splitlines()[0])
            failed = True
        torch.cuda.empty_cache()
        results.append(row)
        print(json.dumps(row), flush=True)
    summary = dict(gpu=name, power_limit=power, steps=a.steps, warmup=a.warmup, results=results)
    print(json.dumps(dict(gpu=name, power_limit=power)))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(summary, f, indent=1)
    if failed:
        raise SystemExit('a configuration failed')


def _make(cfg, mode, dev):
    env_name, n, obs, B, area = CONFIGS[cfg]
    sb = synth.make_states(env_name, n, obs, B, area, 5)
    env, algo = synth.seeded_algo(env_name, n, dev, 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    algo.params['h_dot'] = mode
    return algo, synth.product_batch(env, sb, dev)


def peak_alone(cfg, mode, a, dev):
    """Peak device memory of `warmup` steps with only this mode's model, batch and workspaces allocated (bytes; includes the
    weights, optimiser state and batch)."""
    gc.collect()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated(dev)
    algo, data = _make(cfg, mode, dev)
    torch.cuda.reset_peak_memory_stats(dev)
    for _ in range(a.warmup):
        algo.train_step(data)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated(dev) - base
    del algo, data
    gc.collect()
    torch.cuda.empty_cache()
    return peak


def run_config(cfg, a, dev):
    """Peak memory of each mode alone, then both modes on one configuration, timed alternately; the row printed for it."""
    env_name, n, obs, B, area = CONFIGS[cfg]
    modes = ('finite_difference', 'analytic')
    peak = {m: peak_alone(cfg, m, a, dev) for m in modes}
    algos = {m: _make(cfg, m, dev) for m in modes}
    times = {m: [] for m in algos}
    for m, (algo, data) in algos.items():
        for _ in range(a.warmup):
            algo.train_step(data)
    torch.cuda.synchronize()
    for _ in range(a.steps):
        for m, (algo, data) in algos.items():                 # alternate the two modes
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            algo.train_step(data)
            e1.record()
            e1.synchronize()
            times[m].append(e0.elapsed_time(e1))
    row = dict(config=cfg, env=env_name, agents=n * B, edges=int(algos['analytic'][1].edge_index.shape[1]))
    for m in algos:
        row[m] = dict(median_ms=statistics.median(times[m]), min_ms=min(times[m]), max_ms=max(times[m]), peak_mem_mb=peak[m] / 2 ** 20)
    return row


if __name__ == '__main__':
    main()
