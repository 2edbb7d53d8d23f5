"""Batched test-time controller and vectorised evaluation episodes, timed on the GPU: `python tools/controller_batch_bench.py`.

Prints one JSON line per entry, and first the card's name and power limit (an absolute time is only worth something next to them):
  controller_batch  GCBF.apply_batch (gcbf_apply_batch, csrc/apply.cu) over all graphs of C1x256 (256 graphs x 16 agents) and of C3
                    (64 graphs x 1024 agents) in one call, against the same graphs through one GCBF.apply call each, timed in the
                    same run; max against mean Adam rounds shows what the done graphs that keep going through the passes cost
  evaluation        evaluate_episodes (algo/rollout.py) on 64 C1-size episodes for at most 20 steps each, in agent*steps/s
Nothing is written to the tree."""
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.argv = [sys.argv[0]]
import bench  # noqa: E402  (build_case: the BASELINE configs as bench.py builds them)


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:                      # the numbers below still stand; say why the card line is missing
        out = f'nvidia-smi unavailable: {ex!r}'
    return {'card': out or torch.cuda.get_device_name(0)}


def controller_batch_leg(cfg_name, dev, calls=2):
    """The test-time controller over ALL graphs of the config in one call (GCBF.apply_batch = gcbf_apply_batch in csrc/apply.cu), with
    the reference's settings (lr 0.1, rand 30, up to 31 Adam rounds), against the same graphs through one GCBF.apply call each, timed in
    the same run.  Done graphs keep going through the passes until the slowest is done: max against mean rounds shows what that costs."""
    sb, env, algo = bench.build_case(cfg_name, dev, 0)
    B, n, N = sb.num_graphs, sb.num_agents, sb.nodes_per_graph
    batch = env.graph_from_states(sb.states.to(dev))
    algo.apply_batch(batch)
    torch.cuda.synchronize()
    rounds = []
    t0 = time.perf_counter()
    for _ in range(calls):
        algo.apply_batch(batch)
        rounds.append(algo.last_apply_batch_rounds)
    torch.cuda.synchronize()
    wall = (time.perf_counter() - t0) / calls * 1e3
    r = torch.stack(rounds).double()
    singles = [env.graph_from_states(sb.states[g * N:(g + 1) * N].to(dev)) for g in range(B)]
    algo.apply(singles[0])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for g in range(B):
        algo.apply(singles[g])
    torch.cuda.synchronize()
    wall_single = (time.perf_counter() - t0) * 1e3
    return {'workload': f'{cfg_name}: GCBF.apply_batch on {B} graphs x {n} agents ({int(batch.edge_index.shape[1])} edges) in one call',
            'wall_ms_per_call': round(wall, 3), 'max_rounds': int(r.max()), 'mean_rounds': round(float(r.mean()), 2),
            'agent_actions_per_s': round(B * n / (wall / 1e3), 1),
            'single_apply_wall_ms_for_all_graphs': round(wall_single, 3), 'speedup_vs_single_calls': round(wall_single / wall, 2)}


def evaluation_leg(dev, episodes=64, steps=20):
    """Vectorised test-time evaluation (gcbf_b200/algo/rollout.py::evaluate_episodes): `episodes` C1-size episodes (SimpleCar, 16
    agents, 4 x 4 area, seeds 0..episodes-1) stepped as one batch under GCBF.apply_batch for at most `steps` steps each.  Wall time
    includes the host-side resets (the reference's rejection sampler, one seed after another)."""
    from gcbf_b200.algo.rollout import evaluate_episodes
    sb, env, algo = bench.build_case('C1', dev, 0)
    evaluate_episodes(env, algo, range(2), max_steps=2)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = evaluate_episodes(env, algo, range(episodes), max_steps=steps)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    agent_steps = int(res['length'].sum()) * sb.num_agents
    return {'workload': f'C1: evaluate_episodes, {episodes} episodes x {sb.num_agents} agents, at most {steps} steps, GCBF.apply_batch '
                        '(rand 30, max_iter 30)', 'wall_s': round(wall, 3), 'agent_steps': agent_steps,
            'agent_steps_per_s': round(agent_steps / wall, 1), 'mean_length': round(float(res['length'].mean()), 2)}


if __name__ == '__main__':
    dev = torch.device('cuda', 0)
    print(json.dumps(card()), flush=True)
    for c in ('C1x256', 'C3'):
        print(json.dumps(controller_batch_leg(c, dev)), flush=True)
    print(json.dumps(evaluation_leg(dev)), flush=True)
    print(json.dumps(card()), flush=True)
