"""TEST INFRASTRUCTURE ONLY -- CPU model of the arithmetic of the tensor-core linear layers (csrc/gemm_wgmma_f16.cu).

The product computes an fp32 GEMM as three fp16 tensor-core products of [hi | lo] companions.  This module restates that
arithmetic in plain torch so that (a) the companion format is pinned bit-for-bit (tests/test_kernels_gpu.py compares the
split kernel against `split`) and (b) the accuracy claims written in DESIGN.md section 5 are checked on the CPU, without a
GPU, against fp64 (tests/test_oracle_cpu.py::test_fp16x3_model_accuracy).  Only tests/ import it.
"""
import torch


def scale_for(amax: torch.Tensor) -> float:
    """Power of two s with amax * s in [2^14, 2^15) (1 for zero / denormal / non-finite amax); mirrors
    scale_bits_from_amax in csrc/gemm_wgmma_f16.cu."""
    bits = amax.reshape(1).float().view(torch.int32).item()
    e = (bits >> 23) & 0xff
    if e in (0, 255):
        return 1.0
    se = min(max(127 + 14 - (e - 127), 2), 252)
    return 2.0 ** (se - 127)


def split(x: torch.Tensor):
    """(hi, lo, s): x * s = hi + lo with hi = fp16(x * s), lo = fp16(x * s - hi), both round-to-nearest-even."""
    s = scale_for(x.abs().max())
    xs = x.float() * s
    hi = xs.half()
    lo = (xs - hi.float()).half()
    return hi, lo, s


def gemm(a: torch.Tensor, b: torch.Tensor, chunk: int = 128) -> torch.Tensor:
    """a [M, K] x b [N, K]^T with the kernel's arithmetic: three products hi*hi + lo*hi + hi*lo (lo*lo dropped), exact
    products of fp16 values, K consumed in chunks whose partial sums are promoted to fp32 with round-to-nearest (the
    in-chunk accumulation is modelled in fp64 and rounded once: the tensor core's own in-chunk error is bounded by
    tools/acc_probe.py on hardware), descaled by 1 / (s_a * s_b)."""
    ah, al, sa = split(a)
    bh, bl, sb = split(b)
    ah, al, bh, bl = ah.double(), al.double(), bh.double(), bl.double()
    acc = torch.zeros(a.shape[0], b.shape[0], dtype=torch.float32)
    for k0 in range(0, a.shape[1], chunk):
        sl = slice(k0, k0 + chunk)
        part = ah[:, sl] @ bh[:, sl].T + al[:, sl] @ bh[:, sl].T + ah[:, sl] @ bl[:, sl].T
        acc = acc + part.float()
    return acc * (1.0 / sa) * (1.0 / sb)


# ---- tile-scaled companions (round 2): what the GEMM epilogues emit -------------------------------------------------------------
TILE_ROWS, TILE_COLS = 128, 256


def split_tiled(x: torch.Tensor):
    """Companion with one power-of-two scale per (128-row, 256-column) tile -- the format the producing GEMM's epilogue writes
    (csrc/gemm_wgmma_f16.cu, EPI emit): every output tile knows its own max|y| exactly, so no pass over the tensor and no
    a-priori bound is needed.  Returns (hi, lo, tile_amax [ceil(rows/128), ceil(cols/256)] float32).  Per tile the arithmetic is
    `split` above (scale_for(tile max), hi = fp16(x s), lo = fp16(x s - hi))."""
    rows, cols = x.shape
    tr, tc = (rows + TILE_ROWS - 1) // TILE_ROWS, (cols + TILE_COLS - 1) // TILE_COLS
    hi = torch.zeros(rows, cols, dtype=torch.float16)
    lo = torch.zeros(rows, cols, dtype=torch.float16)
    amax = torch.zeros(tr, tc, dtype=torch.float32)
    for i in range(tr):
        for j in range(tc):
            r, c = slice(i * TILE_ROWS, (i + 1) * TILE_ROWS), slice(j * TILE_COLS, (j + 1) * TILE_COLS)
            t = x[r, c].float()
            amax[i, j] = t.abs().max() if t.numel() else 0.0
            s = scale_for(amax[i, j])
            ts = t * s
            h = ts.half()
            hi[r, c] = h
            lo[r, c] = (ts - h.float()).half()
    return hi, lo, amax


def _tile_scales(amax: torch.Tensor) -> torch.Tensor:
    return torch.tensor([[scale_for(a) for a in row] for row in amax], dtype=torch.float64)


def gemm_tiled_a(a: torch.Tensor, b: torch.Tensor, chunk: int = 128) -> torch.Tensor:
    """a [M, K] (tile-scaled companion, the K-major A operand of a forward / data-grad product) x b [N, K]^T (per-tensor
    companion, a weight): K consumed in `chunk`-wide pieces (a chunk never straddles a 256-column tile of `a`); each chunk sum is
    descaled by 1 / (s_a[row block, column tile] * s_b) -- powers of two, exact -- while it is added to the fp32 result with
    round-to-nearest, exactly what the kernel's promotion FFMA does."""
    assert TILE_COLS % chunk == 0
    ah, al, a_amax = split_tiled(a)
    bh, bl, sb = split(b)
    ah, al, bh, bl = ah.double(), al.double(), bh.double(), bl.double()
    sa = _tile_scales(a_amax)
    M = a.shape[0]
    acc = torch.zeros(M, b.shape[0], dtype=torch.float32)
    row_block = torch.arange(M) // TILE_ROWS
    for k0 in range(0, a.shape[1], chunk):
        sl = slice(k0, k0 + chunk)
        part = ah[:, sl] @ bh[:, sl].T + al[:, sl] @ bh[:, sl].T + ah[:, sl] @ bl[:, sl].T
        inv = (1.0 / (sa[row_block, k0 // TILE_COLS] * sb)).unsqueeze(1)
        acc = (acc.double() + part.float().double() * inv).float()          # fma(part, inv, acc): one rounding
    return acc


def gemm_tiled_wgrad(dz: torch.Tensor, x: torch.Tensor) -> torch.Tensor:
    """dW [N, K] = dz [M, N]^T x [M, K] with BOTH operands tile-scaled (MN-major operands of the weight-grad product): the
    contraction runs over rows in chunks of exactly one 128-row block, descaled per chunk by
    1 / (s_dz[block, n // 256] * s_x[block, k // 256])."""
    dh, dl, d_amax = split_tiled(dz)
    xh, xl, x_amax = split_tiled(x)
    dh, dl, xh, xl = dh.double(), dl.double(), xh.double(), xl.double()
    sd, sx = _tile_scales(d_amax), _tile_scales(x_amax)
    N, K = dz.shape[1], x.shape[1]
    acc = torch.zeros(N, K, dtype=torch.float32)
    nt, kt = torch.arange(N) // TILE_COLS, torch.arange(K) // TILE_COLS
    for blk, m0 in enumerate(range(0, dz.shape[0], TILE_ROWS)):
        sl = slice(m0, m0 + TILE_ROWS)
        part = dh[sl].T @ xh[sl] + dl[sl].T @ xh[sl] + dh[sl].T @ xl[sl]
        inv = 1.0 / (sd[blk, nt].unsqueeze(1) * sx[blk, kt].unsqueeze(0))
        acc = (acc.double() + part.float().double() * inv).float()
    return acc
