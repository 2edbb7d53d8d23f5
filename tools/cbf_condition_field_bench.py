"""CBF-condition fields timed on the GPU: `python tools/cbf_condition_field_bench.py [--reps N]`.

Prints the card's name and power limit first, then one JSON line per entry (CUDA-event times, median of --reps calls after a warm-up):
  c1_one_agent   C1 (SimpleCar, 16 agents), one agent on a 30 x 30 grid: GCBF.cbf_condition_field (two-hop probe graphs) against the
                 copies route (a Batch of 900 copies of the graph: actor, then h_dot_analytic with the freeze)
  c3_all_agents  one C3-sized graph (DubinsCar, 1024 agents + 32 obstacles), ALL 1024 agents on a 30 x 30 grid (921,600 probes), fixed
                 and relink modes: ms, probes/s, two-hop edges, chunks, peak memory
  c3_copies      the copies route for ONE agent of that graph (900 copies), where it fits in memory
Exits non-zero if a configuration fails.  Nothing is written to the tree."""
import argparse
import json
import os
import sys
import traceback

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from cbf_field_bench import DEV, card, copies, setup, timed  # noqa: E402
from gcbf_b200.data import Data  # noqa: E402


def copies_call(algo, env, data, agent, xs, ys):
    with torch.no_grad():
        batch = copies(env, data, agent, xs, ys)
        batch.update(Data(u_ref=env.u_ref(batch)))
        u = algo.actor(batch)
        algo.h_dot_analytic(batch, u, freeze=True)


def c1_leg(reps):
    sb, env, algo, data, lims = setup('C1')
    agent = int(torch.argmax(torch.bincount(data.edge_index[1], minlength=sb.num_agents)[:sb.num_agents]))
    xs, ys, _, _ = algo.cbf_condition_field(data, agents=agent, lims=lims)
    t_field = timed(lambda: algo.cbf_condition_field(data, agents=agent, lims=lims), reps)
    t_copies = timed(lambda: copies_call(algo, env, data, agent, xs, ys), reps)
    return dict(entry='c1_one_agent', probes=900, two_hop_edges=algo.last_field_edges, field_ms=round(t_field, 3),
                copies_ms=round(t_copies, 3), speedup=round(t_copies / t_field, 1))


def c3_leg(reps):
    sb, env, algo, data, lims = setup('C3')
    n = sb.num_agents
    out = []
    for relink in (False, True):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t = timed(lambda: algo.cbf_condition_field(data, agents=list(range(n)), lims=lims, relink=relink), reps)
        peak = torch.cuda.max_memory_allocated() - base
        T = n * 900
        out.append(dict(entry='c3_all_agents', mode='relink' if relink else 'fixed', probes=T, chunks=algo.last_field_chunks,
                        two_hop_edges=algo.last_field_edges, ms=round(t, 1), probes_per_s=round(T / t * 1e3), peak_gb=round(peak / 1e9, 2)))
    xs, ys = algo.field_grid(lims, 0, 1, 30)
    try:
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        t = timed(lambda: copies_call(algo, env, data, 0, xs, ys), max(1, reps // 3))
        out.append(dict(entry='c3_copies', agents=1, copies=900, ms=round(t, 1),
                        peak_gb=round((torch.cuda.max_memory_allocated() - base) / 1e9, 2)))
    except torch.cuda.OutOfMemoryError as ex:
        out.append(dict(entry='c3_copies', agents=1, copies=900, fits=False, error=str(ex).splitlines()[0]))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=3)
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
