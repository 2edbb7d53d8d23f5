"""Train-step time and output drift of GCBF.params['matmul'] = 'fp16' (one fp16 tensor-core product) against the default 'fp32'
(3xFP16), on the C3 and C2 train steps.

    python tools/matmul_precision_bench.py [--steps 10] [--warmup 3] [--configs C3,C2] [--out file.json]

Per config, in one process: the two modes alternate step by step on the same weights and batch (apply_optim=False, so the weights
do not move); each step is timed with CUDA events and the median over --steps is reported.  One more step per mode runs with the
library's per-launch event timer: the largest forward / data-grad / weight-grad launches are listed.  The drift: one step per mode
from the same weights and spectral-norm state -- max |dh|, max |du|, the loss scalars, and the per-net cosine between the two
modes' gradients.  The card name, its power limit and the SM clock are sampled in the same run (nvidia-smi query)."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, 'gcbf-pytorch_b200'), ROOT]

import bench  # noqa: E402
from gcbf_b200 import native  # noqa: E402


def gpu_state():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm', '--format=csv,noheader', '-i', '0'],
                           capture_output=True, text=True, timeout=20).stdout.strip()
        name, power, clock = [s.strip() for s in q.split(',')]
        return dict(gpu=name, power_limit=power, sm_clock=clock)
    except Exception as e:                       # noqa: BLE001 - the numbers are still reported without it
        return dict(gpu=torch.cuda.get_device_name(0), error=str(e))


def snapshot(algo):
    return {n: {k: v.clone() for k, v in m.state_dict().items()} for n, m in (('cbf', algo.cbf), ('actor', algo.actor))}


def restore(algo, snap):
    algo.cbf.load_state_dict(snap['cbf'])
    algo.actor.load_state_dict(snap['actor'])


def timed_step(algo, data):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    algo.train_step(data, apply_optim=False)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def launches(algo, data):
    native.fn('gcbf_timing_enable')(1)
    algo.train_step(data, apply_optim=False)
    torch.cuda.synchronize()
    recs = (native.TimeRec * 4096)()
    cnt = ctypes.c_int(0)
    native.check(native.fn('gcbf_timing_collect')(recs, 4096, ctypes.byref(cnt)), 'gcbf_timing_collect')
    native.fn('gcbf_timing_enable')(0)
    out = {}
    for r in recs[:min(cnt.value, 4096)]:
        if r.kind in (0, 1, 2):
            name = ('forward', 'data-grad', 'weight-grad')[r.kind]
            if name not in out or r.flops > out[name]['flops']:
                out[name] = dict(M=r.M, N=r.N, K=r.K, ms=round(r.ms, 3), flops=r.flops)
    for v in out.values():
        v['tflops'] = round(v.pop('flops') / v['ms'] / 1e9, 1)
    return out


def drift(algo, data, snap):
    res = {}
    for mode in ('fp32', 'fp16'):
        restore(algo, snap)
        algo.set_matmul(mode)
        r = algo.train_step(data, apply_optim=False)
        torch.cuda.synchronize()
        g = {n: torch.cat([p.grad.reshape(-1).double() for p in m.parameters()]) for n, m in (('cbf', algo.cbf), ('actor', algo.actor))}
        res[mode] = (r['h'].detach().double().clone(), r['actions'].detach().double().clone(), r['scalars'].tolist(), g)
    (h32, u32, s32, g32), (h16, u16, s16, g16) = res['fp32'], res['fp16']
    names = ('loss_unsafe', 'loss_safe', 'loss_h_dot', 'loss_action', 'acc_unsafe', 'acc_safe', 'total_loss')
    return dict(max_dh=(h16 - h32).abs().max().item(), max_du=(u16 - u32).abs().max().item(),
                h_absmax=h32.abs().max().item(), u_absmax=u32.abs().max().item(),
                scalars_fp32={k: s32[i] for i, k in enumerate(names)}, scalars_fp16={k: s16[i] for i, k in enumerate(names)},
                grad_cosine={k: float(torch.nn.functional.cosine_similarity(g16[k], g32[k], dim=0)) for k in g32})


def run(cfg, args, dev):
    sb, env, algo = bench.build_case(cfg, dev, 0)
    data = env.graph_from_states(sb.states.to(dev))
    snap = snapshot(algo)
    rec = dict(config=cfg, edges=int(data.edge_index.shape[1]), agents=int(data.u_ref.shape[0]))
    rec['drift'] = drift(algo, data, snap)
    times = {'fp32': [], 'fp16': []}
    for mode in ('fp32', 'fp16'):
        algo.set_matmul(mode)
        for _ in range(args.warmup):
            timed_step(algo, data)
    for _ in range(args.steps):
        for mode in ('fp32', 'fp16'):
            algo.set_matmul(mode)
            times[mode].append(timed_step(algo, data))
    rec['step_ms_median'] = {m: round(statistics.median(t), 2) for m, t in times.items()}
    rec['step_ms_range'] = {m: [round(min(t), 2), round(max(t), 2)] for m, t in times.items()}
    rec['speedup'] = round(rec['step_ms_median']['fp32'] / rec['step_ms_median']['fp16'], 3)
    rec['launches'] = {}
    for mode in ('fp32', 'fp16'):
        algo.set_matmul(mode)
        rec['launches'][mode] = launches(algo, data)
    rec.update(gpu_state())
    restore(algo, snap)
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--configs', default='C3,C2')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda', 0)
    recs = []
    for cfg in args.configs.split(','):
        rec = run(cfg, args, dev)
        print(json.dumps(rec), flush=True)
        recs.append(rec)
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(recs, f, indent=1)


if __name__ == '__main__':
    main()
