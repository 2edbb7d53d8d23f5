"""GPU check of the wgmma 3xFP16 GEMM against fp64 and against the fp32 SIMT kernel, plus timing of its pieces.

GEMM_CHECK_TIMING_ONLY=1 skips the accuracy table; GEMM_CHECK_C3_ONLY=1 runs only the timing of the three products at the C3 layer
shape with the operand formats the train step uses (last section)."""
import ctypes, json, sys, os, math, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, 'gcbf-pytorch_b200')]
from gcbf_b200 import ops, _C, native
dev = torch.device('cuda:0')
print('has wgmma:', _C.lib().gcbf_has_wgmma())
C3_ONLY = bool(os.environ.get('GEMM_CHECK_C3_ONLY'))


def run(M, N, K, impl, scale_x=1.0, scale_dz=1.0):
    ops.GEMM_IMPL = impl
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g) * scale_x; W = torch.randn(N, K, generator=g) / math.sqrt(K); b = torch.randn(N, generator=g) * scale_x
    dz = torch.randn(M, N, generator=g) * scale_dz; rs = torch.randn(M, K, generator=g)
    xd, Wd, bd, dzd, rsd = x.to(dev), W.to(dev), b.to(dev), dz.to(dev), rs.to(dev)
    y = ops.linear_fwd(xd, Wd, bd, None, ops.ACT_RELU)
    dx = ops.linear_bwd_data(dzd, Wd, None, rsd)
    dW, db = ops.linear_bwd_weight(dzd, xd, None)
    torch.cuda.synchronize()
    x64, W64, dz64 = xd.double(), Wd.double(), dzd.double()
    ry = torch.relu(x64 @ W64.t() + bd.double()); rdx = (dz64 @ W64) * (rsd > 0); rdW = dz64.t() @ x64
    e = lambda a, r: ((a.double() - r).abs().max() / r.abs().max()).item()
    return e(y, ry), e(dx, rdx), e(dW, rdW), e(db, dz64.sum(0))


ACC_SHAPES = [] if os.environ.get('GEMM_CHECK_TIMING_ONLY') or C3_ONLY else [(256, 256, 96), (384, 128, 96), (1000, 2048, 2048), (2500, 256, 2048), (777, 2048, 260),
                                                                  (4096, 512, 1024), (300, 130, 100), (70000, 128, 256)]
for shape in ACC_SHAPES:
    for sx, sdz in [(1.0, 1.0), (1e-3, 1e-7)]:
        try:
            r2 = run(*shape, 2, sx, sdz)
            r1 = run(*shape, 1, sx, sdz)
            print(shape, f'scales {sx:g}/{sdz:g}', 'wgmma err y/dx/dW/db: %.2e %.2e %.2e %.2e' % r2, '| simt: %.2e %.2e %.2e %.2e' % r1, flush=True)
        except Exception as ex:
            print(shape, 'FAILED', ex, flush=True)


def timeit(fn, n=5):
    for _ in range(2):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize(); e0.record()
    for _ in range(n):
        fn()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


print('GCBF_TC_KCH =', os.environ.get('GCBF_TC_KCH', 'default (4)'))
for shape in [] if C3_ONLY else [(1000, 2048, 2048), (70000, 128, 256)]:
    print(shape, 'wgmma err y/dx/dW/db vs fp64: %.2e %.2e %.2e %.2e' % run(*shape, 2), flush=True)
# timing at the real layer size (C2: E = 24,196 edges, 2048 x 2048 layer)
ops.GEMM_IMPL = 0
for (M, N, K) in [] if C3_ONLY else [(24196, 2048, 2048), (8192, 2048, 2048), (24196, 256, 2048), (206139, 2048, 2048)]:
    x = torch.randn(M, K, device=dev); W = torch.randn(N, K, device=dev) / 45; b = torch.zeros(N, device=dev); dz = torch.randn(M, N, device=dev)
    xh, wh, dzh = ops.split_h(x), ops.split_h(W), ops.split_h(dz)
    am = torch.empty(1, device=dev, dtype=torch.int32)
    y = torch.empty(M, N, device=dev); dx = torch.empty(M, K, device=dev)
    fl = 2.0 * M * N * K
    t_amax = timeit(lambda: _C.call('gcbf_amax_f32', x.data_ptr(), K, M, K, am.data_ptr(), 0))
    t_split = timeit(lambda: _C.call('gcbf_split_f16', x.data_ptr(), K, M, K, xh.amax.data_ptr(), xh.buf.data_ptr(), xh.ld, None, 0))
    t_f = timeit(lambda: ops.linear_fwd_h(xh, wh, b, None, ops.ACT_RELU, out=y, out_amax=am))
    t_d = timeit(lambda: ops.linear_bwd_data_h(dzh, wh, None, x, out=dx, out_amax=am))
    t_w = timeit(lambda: ops.linear_bwd_weight_h(dzh, xh, None))
    print(f'[{M}x{N}x{K}] amax {t_amax*1e3:.0f} us ({M*K*4/t_amax/1e6:.0f} GB/s)  split {t_split*1e3:.0f} us ({M*K*8/t_split/1e6:.0f} GB/s)  '
          f'fwd {t_f:.3f} ms {fl/t_f/1e9:.0f} TF  dgrad {t_d:.3f} ms {fl/t_d/1e9:.0f} TF  wgrad {t_w:.3f} ms {fl/t_w/1e9:.0f} TF  (fp32-equivalent; x3 = fp16 MMA rate)', flush=True)
    del x, W, dz, xh, wh, dzh, y, dx


# ---- the three products at the C3 layer shape (206,139 edges x 2048 x 2048), in the operand formats of the train step ------------
# forward: per-tensor X and W, fp32 output + tile-scaled companion emitted (ReLU); data-grad: per-tensor dZ, ReLU mask from the hi
# plane of that companion, fp32 output + emitted companion + column sums; weight-grad: both operands tile-scaled (the two emitted
# companions) -- 128 CTAs of about 6,400 k-blocks each and no split, the mainloop alone.  Issued = 3 fp16 MMAs per product.
def tiled_desc(rows, cols):
    ld = (cols + 7) // 8 * 8
    buf = torch.zeros(2, rows, ld, device=dev, dtype=torch.float16)
    amax = torch.zeros((rows + 127) // 128, (cols + 255) // 256, device=dev, dtype=torch.int32)
    return ops.H16(buf, amax, rows, cols, ld, amax.shape[1], 1).desc(), (buf, amax)


M, N, K = 206139, 2048, 2048
torch.manual_seed(0)
x = torch.randn(M, K, device=dev); W = torch.randn(N, K, device=dev) / math.sqrt(K); b = torch.randn(N, device=dev) * 0.1
dz = torch.randn(M, N, device=dev) * 1e-3
xh, wh, dzh = ops.split_h(x), ops.split_h(W), ops.split_h(dz)
X, Wd, DZ = xh.desc(), wh.desc(), dzh.desc()
y = torch.empty(M, N, device=dev); Yh, keep_y = tiled_desc(M, N)
dx = torch.empty(M, K, device=dev); dXh, keep_dx = tiled_desc(M, K)
colsum = torch.zeros(K, device=dev)
dW = torch.empty(K, N, device=dev)
st = _C.stream()
f_fwd, f_dgrad, f_wgrad = native.fn('gcbf_linear_fwd_h'), native.fn('gcbf_linear_bwd_data_h'), native.fn('gcbf_linear_bwd_weight_h')
products = {
    'fwd': lambda: native.check(f_fwd(ctypes.byref(X), ctypes.byref(Wd), _C.ptr(b), None, ops.ACT_RELU, _C.ptr(y), N, ctypes.byref(Yh), None,
                                      M, N, K, st, 3), 'fwd'),
    'dgrad': lambda: native.check(f_dgrad(ctypes.byref(DZ), ctypes.byref(Wd), None, None, 0, ctypes.byref(Yh), _C.ptr(dx), K, 0,
                                          ctypes.byref(dXh), _C.ptr(colsum), None, M, N, K, st, 3), 'dgrad'),
    'wgrad': lambda: native.check(f_wgrad(ctypes.byref(dXh), ctypes.byref(Yh), None, _C.ptr(dW), N, 0, M, K, N, st, 3), 'wgrad'),
}
fl = 2.0 * M * N * K
res = {}
for name, fn in products.items():
    t = timeit(fn, n=20)
    res[name] = {'ms': round(t, 4), 'issued_tflops': round(3 * fl / t / 1e9, 1)}
    print(f'C3 [{M}x{N}x{K}] {name:5s} {t:.3f} ms  {fl / t / 1e9:.1f} TFLOP/s fp32-equivalent  {3 * fl / t / 1e9:.1f} TFLOP/s fp16 MMA issued',
          flush=True)
print(json.dumps({'c3_gemm': res}), flush=True)
