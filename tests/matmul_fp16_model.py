"""CPU model and error bound of the one-product tensor-core GEMM (params['matmul'] = 'fp16', gemm_h_kernel<..., P = 1>).

Arithmetic of the kernel: every fp32 operand element x is scaled by a power of two s (per tensor, or per (128-row, 256-column) tile
for companions an epilogue emitted) and rounded once, x_hat = fp16(x s) (round to nearest even, fp16 subnormals included); the
lo plane is not read.  The contraction is consumed in promotion chunks of L elements: inside a chunk the tensor core adds the exact
fp16 x fp16 products in fp32 with truncation; each chunk sum is then added to the fp32 result with one round-to-nearest FMA that also
applies the chunk's descale 1 / (s_a s_b).  Split-K slices are summed in fp32 in a fixed order, then the epilogue adds the bias
(as fl(b * fl(1 / alpha))) and multiplies by alpha.

Error bound (eps = 2^-11, u = 2^-24, gamma(n) = n u / (1 - n u), gamma_t(n) the same with the truncation unit 2^-23):
  representation   |x_hat / s - x| <= eps |x| + d,  d = 2^-25 / s (half the fp16 subnormal spacing, in the unscaled units), so per
                   product |a_hat b_hat - a b| / (s_a s_b) <= (2 eps + eps^2) |a||b| + (1 + eps)(d_a |b| + |a| d_b) + d_a d_b;
  accumulation     gamma_t(L + 1) of the chunk's absolute sum (L truncated additions plus the final normalisation), and
                   gamma(chunks + splits + 3) of the whole absolute sum for the promotion FMAs, the split pass and the epilogue,
so for C = alpha A B (+ bias) (+ prev)
  |c - c64| <= |alpha| [ (2^-10 + kappa 2^-23) (|A||B|)_ij + subnormal terms ] + gamma(4) |b_j| + gamma(chunks + splits + 4) |prev|
with kappa 2^-23 = 2^-22 + (1 + 2^-10) (gamma_t(L + 1) + gamma(chunks + splits + 3)), i.e. kappa ~= L + 3 + (chunks + splits + 3) / 2.
`bound` below evaluates it per element; tests/test_matmul_fp16_cpu.py checks `gemm_p1` (this arithmetic, with the in-chunk
accumulator truncated after every 16-element wgmma) against float64 with it -- also with exactly representable operands, where only
the accumulation terms are left -- and tests/test_matmul_fp16_gpu.py asserts it for the kernel against float64 of the original fp32
operands.
"""
import math

import numpy as np

EPS = 2.0 ** -11
U = 2.0 ** -24
SUB = 2.0 ** -25


def gamma(n):
    return n * U / (1.0 - n * U)


def gamma_t(n):
    return n * 2.0 ** -23 / (1.0 - n * 2.0 ** -23)


def scale_for(amax: float) -> float:
    """Power of two s with amax s in [2^14, 2^15); 1 for zero / subnormal / non-finite amax (scale_bits_from_amax)."""
    bits = int(np.array([amax], dtype=np.float32).view(np.uint32)[0])
    e = (bits >> 23) & 0xff
    if e in (0, 255):
        return 1.0
    se = min(max(127 + 14 - (e - 127), 2), 252)
    return 2.0 ** (se - 127)


def tile_scales(x: np.ndarray, tile_rows: int = 128, tile_cols: int = 256) -> np.ndarray:
    """Per-element scale of a tile-scaled companion of x (one power of two per (128-row, 256-column) tile)."""
    s = np.empty(x.shape, dtype=np.float64)
    for r in range(0, x.shape[0], tile_rows):
        for c in range(0, x.shape[1], tile_cols):
            t = x[r:r + tile_rows, c:c + tile_cols]
            s[r:r + tile_rows, c:c + tile_cols] = scale_for(float(np.abs(t).max()) if t.size else 0.0)
    return s


def tensor_scales(x: np.ndarray) -> np.ndarray:
    return np.full(x.shape, scale_for(float(np.abs(x).max()) if x.size else 0.0), dtype=np.float64)


def hi(x: np.ndarray, s: np.ndarray) -> np.ndarray:
    """fp16(x s) as float64 (scaled units)."""
    return (x.astype(np.float32) * s.astype(np.float32)).astype(np.float16).astype(np.float64)


def trunc32(x: np.ndarray) -> np.ndarray:
    """x rounded to fp32 toward zero (as float64)."""
    t = x.astype(np.float32)
    over = np.abs(t.astype(np.float64)) > np.abs(x)
    t[over] = np.nextafter(t[over], np.float32(0))
    return t.astype(np.float64)


WG_K = 16            # contraction elements per wgmma instruction


def gemm_p1(a, b, sa, sb, chunk):
    """a [M, K] x b [K, N] (fp32 values, per-element power-of-two scales sa / sb, constant over each chunk of the contraction) with
    the kernel's arithmetic: inside a chunk the accumulator is truncated to fp32 after each 16-element wgmma (the group's exact fp16
    products summed exactly, then added to the running fp32 value and truncated), then one round-to-nearest FMA per chunk."""
    ah, bh = hi(a, sa), hi(b, sb)
    M, K = a.shape
    acc = np.zeros((M, b.shape[1]), dtype=np.float32)
    for k0 in range(0, K, chunk):
        part = np.zeros((M, b.shape[1]), dtype=np.float64)
        for g0 in range(k0, min(K, k0 + chunk), WG_K):
            sl = slice(g0, min(K, g0 + WG_K))
            part = trunc32(part + ah[:, sl] @ bh[sl, :])
        inv = 1.0 / (sa[:, k0:k0 + 1] * sb[k0:k0 + 1, :])
        acc = (acc.astype(np.float64) + part * inv).astype(np.float32)          # one FMA: part * inv is exact (power of two)
    return acc


def bound(a, b, sa, sb, chunk, chunks=None, splits=1, alpha=1.0, bias=None, prev=None, exact_operands=False):
    """Per-element bound on |c - alpha a b (- bias) (- prev)| for the one-product GEMM (float64 [M, N]).  exact_operands: a s and b s
    are fp16 values already (no representation error): the accumulation terms alone."""
    A, B = np.abs(a.astype(np.float64)), np.abs(b.astype(np.float64))
    da, db = SUB / sa, SUB / sb
    P = A @ B
    rep = 0.0 * P if exact_operands else (2 * EPS + EPS * EPS) * P + (1 + EPS) * (da @ B + A @ db) + da @ db
    n = chunks if chunks is not None else math.ceil(a.shape[1] / chunk)
    acc = (gamma_t(chunk + 1) + gamma(n + splits + 3)) * (P + rep)
    out = abs(alpha) * (rep + acc)
    if bias is not None:
        out = out + gamma(4) * np.abs(bias.astype(np.float64))[None, :]
    if prev is not None:
        out = out + gamma(n + splits + 4) * np.abs(prev.astype(np.float64))
    return out


def kappa(chunk, chunks, splits=1):
    """kappa of the bound's (2^-10 + kappa 2^-23) |A||B| form (subnormal terms apart)."""
    g = gamma_t(chunk + 1) + gamma(chunks + splits + 3)
    return (EPS * EPS + g * (1 + 2 * EPS + EPS * EPS)) / 2.0 ** -23
