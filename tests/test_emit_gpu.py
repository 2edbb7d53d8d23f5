"""Companions written by the GEMM epilogues (tile-scaled fp16 [hi|lo], gcbf_linear_fwd_h / gcbf_linear_bwd_data_h) and consumed by all
three products.  The format is pinned bit-for-bit by the CPU model (oracle/fp16x3_model.py::split_tiled): a launch that writes BOTH
the fp32 output and its companion must produce exactly split_tiled(fp32 output)."""
import ctypes
import math

import pytest
import torch

import fp16x3_model as F16
from gcbf_b200 import _C, native, ops
from helpers import per_tensor, tiled_buffers

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0') if torch.cuda.is_available() else None


def _g(seed):
    return torch.Generator().manual_seed(seed)


def fwd(X, W, b, alpha, act, M, N, K, want_f32=True, emit=True):
    y = torch.empty(M, N, device=DEV) if want_f32 else None
    yd, ybuf, yamax = tiled_buffers(M, N)
    rc = native.fn('gcbf_linear_fwd_h')(ctypes.byref(X), ctypes.byref(W), _C.ptr(b), _C.ptr(alpha), act, _C.ptr(y), N,
                                        ctypes.byref(yd) if emit else None, None, M, N, K, _C.stream(), 3)
    native.check(rc, 'gcbf_linear_fwd_h')
    return y, (yd, ybuf, yamax)


@pytest.mark.parametrize('M,N,K', [(1000, 2048, 2048), (300, 256, 2048), (777, 2048, 260), (4100, 512, 1024), (256, 130 + 126, 96)])
def test_forward_emits_the_split_of_its_own_output(M, N, K):
    g = _g(M + N + K)
    x = torch.randn(M, K, generator=g) * torch.logspace(-2, 1, M).unsqueeze(1)        # rows spanning three decades: tiles differ in scale
    W, b = torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    xd, Wd, bd = x.to(DEV), W.to(DEV), b.to(DEV)
    alpha = torch.tensor([1.3], device=DEV)
    X, kx = per_tensor(xd)
    Wh, kw = per_tensor(Wd)
    y, (yd, ybuf, yamax) = fwd(X, Wh, bd, alpha, ops.ACT_RELU, M, N, K)
    torch.cuda.synchronize()
    want = torch.relu(1.3 * (xd.double() @ Wd.double().t()) + bd.double())
    assert ((y.double() - want).abs().max() / want.abs().max()).item() < 1e-5
    hi, lo, amax = F16.split_tiled(y.cpu())
    assert torch.equal(yamax.view(torch.float32).cpu(), amax)
    assert torch.equal(ybuf[0, :, :N].cpu(), hi) and torch.equal(ybuf[1, :, :N].cpu(), lo)
    # companion only (no fp32 output): same planes
    _, (yd2, ybuf2, yamax2) = fwd(X, Wh, bd, alpha, ops.ACT_RELU, M, N, K, want_f32=False)
    torch.cuda.synchronize()
    assert torch.equal(ybuf2, ybuf) and torch.equal(yamax2, yamax)


@pytest.mark.parametrize('M,N,K', [(1000, 2048, 2048), (2500, 256, 2048), (700, 512, 1024)])
def test_tile_scaled_operands_in_all_three_products(M, N, K):
    """y1 = relu(x W1^T) emitted; then forward (A tile-scaled), data-grad (A tile-scaled, mask from the hi plane, emitted output +
    column sums) and weight-grad (both operands tile-scaled) against fp64."""
    g = _g(M * 3 + N + K)
    x = torch.randn(M, K, generator=g) * torch.logspace(-1, 1, M).unsqueeze(1)
    W1, W2 = torch.randn(K, K, generator=g) / math.sqrt(K), torch.randn(N, K, generator=g) / math.sqrt(K)
    dz = torch.randn(M, N, generator=g) * torch.logspace(-4, -2, M).unsqueeze(1)
    xd, W1d, W2d, dzd = x.to(DEV), W1.to(DEV), W2.to(DEV), dz.to(DEV)
    X, k0 = per_tensor(xd)
    W1h, k1 = per_tensor(W1d)
    W2h, k2 = per_tensor(W2d)
    zero_b = torch.zeros(K, device=DEV)
    y1, (y1d, y1buf, y1amax) = fwd(X, W1h, zero_b, None, ops.ACT_RELU, M, K, K)                       # [M, K] hidden activation, emitted
    # forward through layer 2 from the emitted companion
    y2 = torch.empty(M, N, device=DEV)
    native.check(native.fn('gcbf_linear_fwd_h')(ctypes.byref(y1d), ctypes.byref(W2h), None, None, ops.ACT_NONE, _C.ptr(y2), N, None, None, M, N, K,
                                                _C.stream(), 3), 'fwd2')
    y1_64 = y1.double()
    e = lambda a, r: ((a.double() - r).abs().max() / r.abs().max()).item()
    assert e(y2, y1_64 @ W2d.double().t()) < 1e-5
    # data-grad of layer 2 with the ReLU mask of y1 from the hi plane, output emitted + fp32, column sums
    DZ, k3 = per_tensor(dzd)
    dx = torch.empty(M, K, device=DEV)
    dxd, dxbuf, dxamax = tiled_buffers(M, K)
    colsum = torch.zeros(K, device=DEV)
    native.check(native.fn('gcbf_linear_bwd_data_h')(ctypes.byref(DZ), ctypes.byref(W2h), None, None, 0, ctypes.byref(y1d), _C.ptr(dx), K, 0,
                                                     ctypes.byref(dxd), _C.ptr(colsum), None, M, N, K, _C.stream(), 3), 'dgrad')
    torch.cuda.synchronize()
    want_dx = (dzd.double() @ W2d.double()) * (y1 > 0)
    assert e(dx, want_dx) < 1e-5
    hi, lo, amax = F16.split_tiled(dx.cpu())
    assert torch.equal(dxamax.view(torch.float32).cpu(), amax)
    assert torch.equal(dxbuf[0, :, :K].cpu(), hi) and torch.equal(dxbuf[1, :, :K].cpu(), lo)
    assert ((colsum.double() - dx.double().sum(0)).abs().max() / dx.double().sum(0).abs().max()).item() < 1e-5
    # mask from the fp32 activation gives the same result
    dx2 = torch.empty(M, K, device=DEV)
    native.check(native.fn('gcbf_linear_bwd_data_h')(ctypes.byref(DZ), ctypes.byref(W2h), None, _C.ptr(y1), K, None, _C.ptr(dx2), K, 0, None, None,
                                                     None, M, N, K, _C.stream(), 3), 'dgrad2')
    assert torch.equal(dx2, dx)
    # weight-grad of layer 1 (dW1 = dx^T x... here: operands dx (emitted, tile-scaled) and y1 (emitted, tile-scaled)): dW = dx^T y1
    dW = torch.empty(K, K, device=DEV)
    native.check(native.fn('gcbf_linear_bwd_weight_h')(ctypes.byref(dxd), ctypes.byref(y1d), None, _C.ptr(dW), K, 0, M, K, K, _C.stream(), 3), 'wgrad')
    assert e(dW, dx.double().t() @ y1_64) < 1e-5
    # and mixed: per-tensor dZ with the tile-scaled activation (what the first backward layer of a chain sees)
    dW2 = torch.empty(N, K, device=DEV)
    native.check(native.fn('gcbf_linear_bwd_weight_h')(ctypes.byref(DZ), ctypes.byref(y1d), None, _C.ptr(dW2), K, 0, M, N, K, _C.stream(), 3), 'wgrad2')
    assert e(dW2, dzd.double().t() @ y1_64) < 1e-5


def test_cpu_model_of_tile_scaled_products_matches_the_kernel():
    """oracle/fp16x3_model.py::gemm_tiled_a (K consumed in 128-wide chunks, per-chunk descale) against the kernel on small
    integers-on-a-grid inputs where every in-chunk sum is exact in fp32 (so truncation inside the tensor core cannot differ)."""
    M, N, K = 256, 256, 512
    g = _g(9)
    x = (torch.randint(-8, 9, (M, K), generator=g).float() * torch.tensor([1.0, 2.0 ** -6]).repeat_interleave(128).unsqueeze(1))
    W = torch.randint(-8, 9, (N, K), generator=g).float() / 8
    xd, Wd = x.to(DEV), W.to(DEV)
    # emit the companion of x through an identity-like layer is not possible (it must come out of an epilogue): use y = relu(x) via W = I
    eye = torch.eye(K, device=DEV)
    X, k0 = per_tensor(xd.abs())
    Eh, k1 = per_tensor(eye)
    y, (yd, ybuf, yamax) = fwd(X, Eh, torch.zeros(K, device=DEV), None, ops.ACT_NONE, M, K, K)
    assert torch.equal(y, xd.abs())                                   # exact: small integers
    Wh, k2 = per_tensor(Wd)
    out = torch.empty(M, N, device=DEV)
    native.check(native.fn('gcbf_linear_fwd_h')(ctypes.byref(yd), ctypes.byref(Wh), None, None, ops.ACT_NONE, _C.ptr(out), N, None, None, M, N, K,
                                                _C.stream(), 3), 'fwd')
    want = F16.gemm_tiled_a(x.abs(), W)
    assert torch.equal(out.cpu(), want)


@pytest.mark.parametrize('M,N,K,act', [(5000, 2048, 13, 1), (300, 2048, 12, 1), (1000, 300, 14, 0), (129, 256, 16, 2)])
def test_skinny_forward_emits_the_split_of_the_fp32_kernel_output(M, N, K, act):
    """gcbf_linear_fwd_emit (first phi layer, in-features <= 16, companion only) against the fp32 skinny kernel + the CPU model of the
    tile-scaled split: bit-exact (same FMA order; the tile maximum is computed from the very values that are converted)."""
    g = _g(M + N + K)
    x, W, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g), torch.randn(N, generator=g)
    xd, Wd, bd = x.to(DEV), W.to(DEV), b.to(DEV)
    alpha = torch.tensor([0.9], device=DEV)
    y = ops.linear_fwd(xd, Wd, bd, alpha, act)
    assert _C.lib().gcbf_last_gemm_impl() == 3
    yd, ybuf, yamax = tiled_buffers(M, N)
    native.check(native.fn('gcbf_linear_fwd_emit')(_C.ptr(xd), K, _C.ptr(Wd), K, _C.ptr(bd), _C.ptr(alpha), act, ctypes.byref(yd), M, N, K,
                                                   _C.stream()), 'gcbf_linear_fwd_emit')
    torch.cuda.synchronize()
    hi, lo, amax = F16.split_tiled(y.cpu())
    assert torch.equal(yamax.view(torch.float32).cpu(), amax)
    assert torch.equal(ybuf[0, :, :N].cpu(), hi) and torch.equal(ybuf[1, :, :N].cpu(), lo)
