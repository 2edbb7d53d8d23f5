"""Where the epilogue of the 3xFP16 wgmma GEMM costs time: every tensor-core launch shape of the C3 train step, timed with the
epilogue the step gives it and again with a plain fp32 output.

    python tools/epilogue_probe.py [--config C3] [--reps 10] [--out file.json]

1. One train step with the library's per-launch event timer lists the tensor-core launches (kind, M, N, K, count, in-step ms).
2. Each forward / data-grad shape is then launched on its own (device events over --reps launches after 2 warm-ups):
   - `epilogue`: the options the train step uses for it (net.cu `mlp_forward` / `mlp_backward`): a forward of a hidden layer
     applies bias, alpha and ReLU and emits the tile-scaled companion only; a last layer writes fp32.  A data-grad of a layer above a
     hidden layer takes the ReLU mask from the hi plane of that layer's companion, and emits the companion plus column sums when
     the layer below runs on the tensor cores too (fp32 output otherwise).
   - `plain`: the same product with a fp32 output and no bias, alpha, activation, mask, emission or column sums.
   The difference per tile is (epilogue - plain) x SMs / tiles: the time one SM spends on one tile's extra epilogue work.
The card name, its power limit and the SM clock are read in the same run."""
import argparse
import ctypes
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, 'gcbf-pytorch_b200'), ROOT, os.path.join(ROOT, 'tools')]
os.environ['GCBF_TWO_STREAMS'] = '0'             # one stream: the in-step event pairs time one launch each

import bench  # noqa: E402
from gcbf_b200 import _C, native, ops  # noqa: E402
from matmul_precision_bench import gpu_state  # noqa: E402

KINDS = ('forward', 'data-grad', 'weight-grad')


def step_launches(cfg, dev):
    sb, env, algo = bench.build_case(cfg, dev, 0)
    data = env.graph_from_states(sb.states.to(dev))
    E, A = int(data.edge_index.shape[1]), int(sb.states.shape[0])
    for _ in range(2):
        algo.train_step(data, apply_optim=False)
    torch.cuda.synchronize()
    native.fn('gcbf_timing_enable')(1)
    algo.train_step(data, apply_optim=False)
    torch.cuda.synchronize()
    recs = (native.TimeRec * 65536)()
    cnt = ctypes.c_int(0)
    native.check(native.fn('gcbf_timing_collect')(recs, 65536, ctypes.byref(cnt)), 'gcbf_timing_collect')
    native.fn('gcbf_timing_enable')(0)
    shapes = {}
    for r in recs[:cnt.value]:
        if r.kind in (0, 1, 2):
            s = shapes.setdefault((r.kind, r.M, r.N, r.K), [0, 0.0])
            s[0] += 1
            s[1] += r.ms
    del algo, data, env, sb
    torch.cuda.empty_cache()
    return E, A, shapes


def tiled(rows, cols, dev):
    ld = (cols + 7) // 8 * 8
    buf = torch.zeros(2, rows, ld, device=dev, dtype=torch.float16)
    amax = torch.zeros((rows + 127) // 128, (cols + 255) // 256, device=dev, dtype=torch.int32)
    return ops.H16(buf, amax, rows, cols, ld, amax.shape[1], 1).desc(), (buf, amax)


def timeit(fn, n):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def probe(kind, M, N, K, tc_shapes, dev, reps):
    """(epilogue ms, plain ms, options) of one forward (Y[M,N] = X[M,K] W^T) or data-grad (dX[M,K] = dZ[M,N] W) shape."""
    g = torch.Generator(device=dev).manual_seed(M + N + K)
    W = torch.randn(N, K, device=dev, generator=g) / K ** 0.5
    wh = ops.split_h(W)
    Wd = wh.desc()
    isg = torch.full((1,), 0.9, device=dev)
    st = _C.stream()
    if kind == 0:
        f = native.fn('gcbf_linear_fwd_h')
        xh = ops.split_h(torch.randn(M, K, device=dev, generator=g))
        X = xh.desc()
        b = torch.randn(N, device=dev, generator=g) * 0.1
        y = torch.empty(M, N, device=dev)
        # a hidden layer of the step feeds a tensor-core layer: companion only; the last layer of a net writes fp32
        hidden = N > 128 and any(k == 0 and m == M and kk == N for (k, m, _, kk) in tc_shapes)
        Yh, keep = tiled(M, N, dev) if hidden else (None, None)
        opts = 'bias, alpha, ReLU, companion' if hidden else 'bias, alpha, fp32'
        epi = lambda: native.check(f(ctypes.byref(X), ctypes.byref(Wd), _C.ptr(b), _C.ptr(isg), ops.ACT_RELU if hidden else 0,
                                     None if hidden else _C.ptr(y), N, ctypes.byref(Yh) if hidden else None, None, M, N, K, st, 3), 'fwd')
        plain = lambda: native.check(f(ctypes.byref(X), ctypes.byref(Wd), None, None, 0, _C.ptr(y), N, None, None, M, N, K, st, 3), 'fwd')
    else:
        f = native.fn('gcbf_linear_bwd_data_h')
        dzh = ops.split_h(torch.randn(M, N, device=dev, generator=g) * 1e-3)
        DZ = dzh.desc()
        maskh = ops.split_h(torch.randn(M, K, device=dev, generator=g))
        MK = maskh.desc()
        dx = torch.empty(M, K, device=dev)
        colsum = torch.zeros(K, device=dev)
        # the layer below (K outputs) is a hidden layer; it runs on the tensor cores iff the step has a forward [M, K] launch
        # with a contraction wide enough to be one: then the data-grad emits its companion and the column sums
        emit = K > 128 and any(k == 0 and m == M and n == K for (k, m, n, _) in tc_shapes)
        mask = K > 128
        dXh, keep = tiled(M, K, dev) if emit else (None, None)
        opts = ', '.join(['alpha'] + (['hi-plane mask'] if mask else []) + (['companion, column sums'] if emit else ['fp32']))
        epi = lambda: native.check(f(ctypes.byref(DZ), ctypes.byref(Wd), _C.ptr(isg), None, 0, ctypes.byref(MK) if mask else None,
                                     None if emit else _C.ptr(dx), K, 0, ctypes.byref(dXh) if emit else None,
                                     _C.ptr(colsum) if emit else None, None, M, N, K, st, 3), 'dgrad')
        plain = lambda: native.check(f(ctypes.byref(DZ), ctypes.byref(Wd), None, None, 0, None, _C.ptr(dx), K, 0, None, None, None,
                                       M, N, K, st, 3), 'dgrad')
    t_e, t_p = timeit(epi, reps), timeit(plain, reps)
    t_e2, t_p2 = timeit(epi, reps), timeit(plain, reps)     # alternated twice: the lower of each pair is kept
    return min(t_e, t_e2), min(t_p, t_p2), opts


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', default='C3')
    ap.add_argument('--reps', type=int, default=10)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda', 0)
    state0 = gpu_state()
    E, A, shapes = step_launches(args.config, dev)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    print(f'{args.config}: E = {E}, agents = {A}; {state0}', flush=True)
    print(f'{"kind":11s} {"M":>7s} {"N":>5s} {"K":>5s} {"n":>3s} {"in step":>8s} | {"epilogue":>8s} {"TF iss":>6s} | {"plain":>8s} '
          f'{"TF iss":>6s} | {"diff/tile":>9s}  options', flush=True)
    rows = []
    for (kind, M, N, K), (n, ms) in sorted(shapes.items()):
        flops = 2.0 * M * N * K
        row = dict(kind=KINDS[kind], M=M, N=N, K=K, launches=n, in_step_ms=round(ms / n, 4))
        out_w = N if kind == 0 else K
        if kind in (0, 1) and out_w > 128:
            t_e, t_p, opts = probe(kind, M, N, K, shapes, dev, args.reps)
            tiles = -(-M // 128) * -(-out_w // 256)
            row.update(epilogue_ms=round(t_e, 4), plain_ms=round(t_p, 4), options=opts,
                       epilogue_issued_tflops=round(3 * flops / t_e / 1e9, 1), plain_issued_tflops=round(3 * flops / t_p / 1e9, 1),
                       diff_us_per_tile=round((t_e - t_p) * 1e3 * sms / tiles, 2))
            print(f'{KINDS[kind]:11s} {M:7d} {N:5d} {K:5d} {n:3d} {ms / n:8.3f} | {t_e:8.3f} {row["epilogue_issued_tflops"]:6.1f} | '
                  f'{t_p:8.3f} {row["plain_issued_tflops"]:6.1f} | {row["diff_us_per_tile"]:7.2f} us  {opts}', flush=True)
        else:
            print(f'{KINDS[kind]:11s} {M:7d} {N:5d} {K:5d} {n:3d} {ms / n:8.3f} |   (not probed: weight-grad or a 128-wide tile)', flush=True)
        rows.append(row)
    res = dict(config=args.config, E=E, agents=A, sms=sms, before=state0, after=gpu_state(), launches=rows)
    print(json.dumps(res), flush=True)
    if args.out:
        with open(args.out, 'w') as fh:
            json.dump(res, fh, indent=1)


if __name__ == '__main__':
    main()
