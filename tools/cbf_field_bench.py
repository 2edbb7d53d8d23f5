"""CBF level-set fields timed on the GPU: `python tools/cbf_field_bench.py [--reps N]`.

Prints the card's name and power limit first, then one JSON line per entry (CUDA-event times, median of --reps calls after a warm-up):
  c1_one_agent   C1 (SimpleCar, 16 agents), one agent on a 30 x 30 grid: GCBF.cbf_field (probe graphs, gcbf_cbf_field) against the
                 reference's construction through this library's module API (CBFGNN on a Batch of 900 copies of the graph)
  c3_all_agents  one C3-sized graph (DubinsCar, 1024 agents + 32 obstacles), ALL 1024 agents on a 30 x 30 grid (921,600 probes), fixed
                 and relink modes: ms, probes/s, fp32-equivalent TFLOP/s of the CBF's layers on the probe rows, peak memory
  c3_copies      the copy construction for ONE agent of that graph (900 copies), where it fits in memory
Exits non-zero if a configuration fails.  Nothing is written to the tree."""
import argparse
import json
import os
import subprocess
import sys
import traceback

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'gcbf-pytorch_b200'))

from gcbf_b200 import synth  # noqa: E402
from gcbf_b200.data import Data  # noqa: E402
from gcbf_b200.synth import product_batch, seeded_algo  # noqa: E402

DEV = torch.device('cuda')


def card():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as ex:
        out = f'nvidia-smi unavailable: {ex!r}'
    return {'card': out or torch.cuda.get_device_name(0)}


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    return float(np.median(ms))


def cbf_flops(env, probe_edges, probes):
    """fp32-equivalent FLOPs of the CBF layers on the probe rows: phi + gate per edge, gamma + head per probe (2 * M * N * K)."""
    ein = 2 * env.node_dim + env.edge_dim
    per_edge = 2 * (ein * 2048 + 2048 * 2048 + 2048 * 256) + 2 * (256 * 128 + 128 * 128 + 128)
    per_probe = 2 * ((256 + env.node_dim) * 2048 + 2048 * 2048 + 2048 * 1024) + 2 * (1024 * 512 + 512 * 128 + 128 * 32 + 32)
    return per_edge * probe_edges + per_probe * probes


def copies(env, data, agent, xs, ys):
    N = data.states.shape[0]
    M = len(xs) * len(ys)
    st = data.states.repeat(M, 1)
    gx, gy = np.meshgrid(np.asarray(xs, np.float32), np.asarray(ys, np.float32))
    rows = torch.arange(M, device=DEV) * N + agent
    st[rows, 0] = torch.from_numpy(gx.reshape(-1)).to(DEV)
    st[rows, 1] = torch.from_numpy(gy.reshape(-1)).to(DEV)
    E = data.edge_index.shape[1]
    ei = data.edge_index.repeat(1, M) + (torch.arange(M, device=DEV) * N).repeat_interleave(E).unsqueeze(0)
    fields = dict(x=data.x.repeat(M, 1), states=st, edge_index=ei, edge_attr=env.edge_attr(st, ei))
    if hasattr(data, 'agent_mask'):
        fields['agent_mask'] = data.agent_mask.repeat(M)
    return Data(**fields)


def setup(cfg):
    c = dict(synth.CONFIGS[cfg])
    sb = synth.make_states(c['env'], c['num_agents'], c['num_obs'], 1, c['area_size'], c['seed'])
    env, algo = seeded_algo(sb.env, sb.num_agents, DEV, 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    data = product_batch(env, sb, DEV)
    lims = (torch.zeros(env.state_dim), torch.full((env.state_dim,), float(c['area_size'])))
    return sb, env, algo, data, lims


def c1_leg(reps):
    sb, env, algo, data, lims = setup('C1')
    agent = int(torch.argmax(torch.bincount(data.edge_index[1], minlength=sb.num_agents)[:sb.num_agents]))
    xs, ys, _ = algo.cbf_field(data, agents=agent, lims=lims)
    t_field = timed(lambda: algo.cbf_field(data, agents=agent, lims=lims), reps)

    def copy_call():
        with torch.no_grad():
            algo.cbf(copies(env, data, agent, xs, ys))
    t_copies = timed(copy_call, reps)
    return dict(entry='c1_one_agent', probes=900, edges=int(data.edge_index.shape[1]), cbf_field_ms=round(t_field, 3),
                copies_ms=round(t_copies, 3), speedup=round(t_copies / t_field, 1))


def c3_leg(reps):
    sb, env, algo, data, lims = setup('C3')
    n = sb.num_agents
    out = []
    for relink in (False, True):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t = timed(lambda: algo.cbf_field(data, agents=list(range(n)), lims=lims, relink=relink), reps)
        peak = torch.cuda.max_memory_allocated() - base
        edges = algo.last_field_edges
        T = n * 900
        rec = dict(entry='c3_all_agents', mode='relink' if relink else 'fixed', probes=T, chunks=algo.last_field_chunks, ms=round(t, 1),
                   probes_per_s=round(T / t * 1e3), peak_gb=round(peak / 1e9, 2))
        rec['probe_edges'] = edges
        rec['tflops_fp32_equiv'] = round(cbf_flops(env, edges, T) / (t * 1e-3) / 1e12, 1)
        out.append(rec)
    agent = 0
    xs, ys = algo.field_grid(lims, 0, 1, 30)
    try:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()

        def copy_call():
            with torch.no_grad():
                algo.cbf(copies(env, data, agent, xs, ys))
        t = timed(copy_call, max(1, reps // 3))
        out.append(dict(entry='c3_copies', agents=1, copies=900, edges=int(data.edge_index.shape[1]) * 900, ms=round(t, 1),
                        peak_gb=round((torch.cuda.max_memory_allocated() - base) / 1e9, 2)))
    except torch.cuda.OutOfMemoryError as ex:
        out.append(dict(entry='c3_copies', agents=1, copies=900, fits=False, error=str(ex).splitlines()[0]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    print(json.dumps(card()), flush=True)
    failed = False
    for leg in (c1_leg, c3_leg):
        try:
            res = leg(a.reps)
            for r in (res if isinstance(res, list) else [res]):
                print(json.dumps(r), flush=True)
        except Exception:
            failed = True
            traceback.print_exc()
        torch.cuda.empty_cache()
    sys.exit(1 if failed else 0)


if __name__ == '__main__':
    main()
