"""Isolated timing of the tensor-core forward / data-grad with the different output modes of the epilogue (fp32 only, companion only,
both; GCBF_EPI_STORE=direct switches the companion stores) at the real layer sizes.  python tools/emit_bench.py [M ...]"""
import ctypes, math, os, sys, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, 'gcbf-pytorch_b200')]
from gcbf_b200 import _C, native, ops
dev = torch.device('cuda:0')


def timeit(fn, n=6):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def tiled(rows, cols):
    ld = (cols + 7) // 8 * 8
    buf = torch.zeros(2, rows, ld, device=dev, dtype=torch.float16)
    tc = (cols + 255) // 256
    amax = torch.zeros((rows + 127) // 128, tc, device=dev, dtype=torch.int32)
    return ops.H16(buf, amax, rows, cols, ld, tc, 1).desc(), (buf, amax)


print('GCBF_EPI_STORE =', os.environ.get('GCBF_EPI_STORE', 'tma'), ' GCBF_TC_KCH =', os.environ.get('GCBF_TC_KCH', '4'))
for M in [int(a) for a in sys.argv[1:]] or [24196, 206139]:
    N = K = 2048
    x = torch.randn(M, K, device=dev); W = torch.randn(N, K, device=dev) / 45; b = torch.zeros(N, device=dev); dz = torch.randn(M, N, device=dev)
    xh, wh, dzh = ops.split_h(x), ops.split_h(W), ops.split_h(dz)
    X, Wd, DZ = xh.desc(), wh.desc(), dzh.desc()
    y = torch.empty(M, N, device=dev)
    yd, keep = tiled(M, N)
    colsum = torch.zeros(K, device=dev)
    fl = 2.0 * M * N * K
    F, D = native.fn('gcbf_linear_fwd_h'), native.fn('gcbf_linear_bwd_data_h')
    st = _C.stream()
    modes = {
        'fwd fp32 out': lambda: F(ctypes.byref(X), ctypes.byref(Wd), b.data_ptr(), None, 1, y.data_ptr(), N, None, None, M, N, K, st, 3),
        'fwd companion out': lambda: F(ctypes.byref(X), ctypes.byref(Wd), b.data_ptr(), None, 1, None, N, ctypes.byref(yd), None, M, N, K, st, 3),
        'fwd both': lambda: F(ctypes.byref(X), ctypes.byref(Wd), b.data_ptr(), None, 1, y.data_ptr(), N, ctypes.byref(yd), None, M, N, K, st, 3),
        'fwd from tile-scaled A': lambda: F(ctypes.byref(yd), ctypes.byref(Wd), b.data_ptr(), None, 1, y.data_ptr(), N, None, None, M, N, K, st, 3),
        'dgrad fp32 out, fp32 mask': lambda: D(ctypes.byref(DZ), ctypes.byref(Wd), None, x.data_ptr(), K, None, y.data_ptr(), K, 0, None, None, None, M, N, K, st, 3),
        'dgrad companion out, hi mask, colsum': lambda: D(ctypes.byref(DZ), ctypes.byref(Wd), None, None, 0, ctypes.byref(X), None, K, 0, ctypes.byref(yd),
                                                          colsum.data_ptr(), None, M, N, K, st, 3),
        'dgrad companion out, hi mask': lambda: D(ctypes.byref(DZ), ctypes.byref(Wd), None, None, 0, ctypes.byref(X), None, K, 0, ctypes.byref(yd), None, None,
                                                  M, N, K, st, 3),
    }
    for name, fn in modes.items():
        rc = fn()
        assert rc == 0, (name, _C.lib().gcbf_last_error())
        t = timeit(fn)
        print(f'[{M} x {N} x {K}] {name:40s} {t:7.3f} ms  {fl / t / 1e9:6.0f} TF', flush=True)
    del x, W, dz, xh, wh, dzh, y, keep
