"""Data-grad epilogue of the wgmma GEMM (gcbf_linear_bwd_data_h) at the edges of the work it does after the mainloop: the ReLU mask
(loaded before the parked tile is touched, from either source), tile maxima, the emitted companion and the column sums.

Shapes put that work on its edges: contractions of one to eight k-blocks (half 1 of a 256-wide tile shorter than any slice of the
epilogue), ragged M with mask rows beyond M, output widths that are not a multiple of 256 (ragged column sums and mask loads) and
mask entries of +0.0 and -0.0.  Every launch runs twice and must give the same bits; the companion and tile maxima must be
split_tiled of the same launch's fp32 output, and the column sums the float32 sum of the masked output in the kernel's order (row
by row inside each 128-row tile from 0, then the tiles in order)."""
import ctypes
import math

import numpy as np
import pytest
import torch

import fp16x3_model as F16
from gcbf_b200 import _C, native
from helpers import per_tensor, tiled_buffers

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0') if torch.cuda.is_available() else None


def colsum_in_kernel_order(x):
    """float32 column sums of x [M, K]: each 128-row tile summed row by row from +0, then the tile partials added in order to +0."""
    x = x.numpy().astype(np.float32)
    total = np.zeros(x.shape[1], dtype=np.float32)
    for t0 in range(0, x.shape[0], 128):
        part = np.zeros(x.shape[1], dtype=np.float32)
        for r in range(t0, min(t0 + 128, x.shape[0])):
            part = part + x[r]
        total = total + part
    return torch.from_numpy(total)


def mask_source(M, K, g):
    """fp32 ReLU-mask source with about half its entries > 0 and whole columns and rows of +0.0 and -0.0 (both must mask)."""
    m = torch.randn(M, K, generator=g)
    m[:, 1::7] = 0.0
    m[:, 3::7] = -0.0
    m[5::11, :] = -0.0
    return m


def dgrad(products, DZ, W, alpha, mask_src, mask_h, M, N, K):
    """one launch: fp32 output AND emitted companion AND column sums, so the three can be checked against each other.
    mask_src: (fp32 tensor, pitch) or None; mask_h: companion descriptor or None"""
    dx = torch.full((M, K), float('nan'), device=DEV)
    dxd, dxbuf, dxamax = tiled_buffers(M, K)
    colsum = torch.zeros(K, device=DEV)
    rc = native.fn('gcbf_linear_bwd_data_h')(ctypes.byref(DZ), ctypes.byref(W), _C.ptr(alpha),
                                              _C.ptr(mask_src[0]) if mask_src else None, mask_src[1] if mask_src else 0,
                                              ctypes.byref(mask_h) if mask_h is not None else None, _C.ptr(dx), K, 0,
                                              ctypes.byref(dxd), _C.ptr(colsum), None, M, N, K, _C.stream(), products)
    native.check(rc, 'gcbf_linear_bwd_data_h')
    torch.cuda.synchronize()
    return dx.cpu(), dxbuf.cpu(), dxamax.cpu(), colsum.cpu()


# (M, N = contraction, K = output width): N of 32 / 64 / 256 are 1 / 2 / 8 k-blocks per 128-column half; M ragged in the last row
# tile (mask rows exist beyond M only in the source's allocation); K not a multiple of 256 (a ragged 256-wide tile, a 4-column group
# cut by the edge when K % 4 != 0)
SHAPES = [(300, 32, 2048), (300, 64, 520), (777, 256, 2048), (129, 256, 390), (520, 96, 1100), (1000, 2048, 2048)]


@pytest.mark.parametrize('products', [3, 1])
@pytest.mark.parametrize('source', ['fp32', 'hi'])
@pytest.mark.parametrize('M,N,K', SHAPES)
def test_data_grad_epilogue_edges(M, N, K, source, products):
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    dz = torch.randn(M, N, generator=g) * torch.logspace(-3, 0, M).unsqueeze(1)      # row tiles of different scale
    W = torch.randn(N, K, generator=g) / math.sqrt(N)
    # the mask source has rows beyond M: a launch must not take them (or anything past column K) into its mask
    src_full = mask_source(M + 200, K + 12, g)
    src = src_full[:M, :K]
    dzd, Wd = dz.to(DEV), W.to(DEV)
    alpha = torch.tensor([0.75], device=DEV)
    DZ, kz = per_tensor(dzd)
    Wh, kw = per_tensor(Wd)
    if source == 'fp32':
        # a strided view (pitch K + 12): 16-byte loads when K % 4 == 0, element loads otherwise
        src_dev = src_full.to(DEV)
        mask = src > 0
        run = lambda: dgrad(products, DZ, Wh, alpha, (src_dev, K + 12), None, M, N, K)
    else:
        Sh, ks = per_tensor(src.to(DEV))
        mask = (ks.buf[0, :, :K].float() > 0).cpu()
        run = lambda: dgrad(products, DZ, Wh, alpha, None, Sh, M, N, K)
    dx, buf, amax, colsum = run()
    dx2, buf2, amax2, colsum2 = run()
    assert torch.equal(dx, dx2) and torch.equal(buf, buf2) and torch.equal(amax, amax2) and torch.equal(colsum, colsum2)
    # masked entries are exact zeros; none of the output is left unwritten
    assert not torch.isnan(dx).any()
    assert bool((dx[~mask] == 0).all())
    # against float64: 3xFP16 within 1e-5 of the max, one fp16 product within its per-element bound (2^-10 + accumulation terms)
    want = 0.75 * (dz.double() @ W.double()) * mask
    err = (dx.double() - want).abs()
    if products == 3:
        assert (err.max() / want.abs().max()).item() < 1e-5
    else:
        bound = (2.0 ** -10 + (N + 40) * 2.0 ** -23) * 0.75 * (dz.double().abs() @ W.double().abs()) * mask + 1e-30
        assert bool((err <= bound).all()), (err / bound).max().item()
    # the emitted companion and the tile maxima are the tile-scaled split of this launch's own fp32 output
    hi, lo, tile_amax = F16.split_tiled(dx)
    assert torch.equal(amax.view(torch.float32), tile_amax)
    assert torch.equal(buf[0, :, :K], hi) and torch.equal(buf[1, :, :K], lo)
    # column sums: float32, in the kernel's order
    assert torch.equal(colsum, colsum_in_kernel_order(dx))
