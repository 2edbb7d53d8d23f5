"""Every implementation of the linear-layer products against float64, element by element.

`gcbf_linear_fwd` / `gcbf_linear_bwd_data` / `gcbf_linear_bwd_weight` (csrc/linear.cu) pick one of five implementations by shape,
and ops.use_h sends the big layers to the wgmma 3xFP16 kernel (csrc/gemm_wgmma_f16.cu).  `expected_impl` below mirrors those
rules; every case asserts that the library routed its shape where the mirror says, so a rule change without its mirror fails here
(and tests/test_linear_paths_cpu.py then shows which cells of the dispatch table the case table still covers).

What each case checks, on two operand layouts (`LAYOUTS`):
  * all three products under the epilogue options (activation, bias, 1/sigma, ReLU mask, accumulation), each against a float64
    reference with a PER-ELEMENT bound (below), so a wrong result in a row that is small next to the tensor's max still fails;
  * every operand is a column slice of a NaN-filled buffer: an over-read poisons the result, an over-write changes the padding
    (compared bit for bit); the odd-pitch layout, one float off a 16-byte boundary, takes every float4 -> scalar fallback;
  * every call runs twice from the same state and must give the same bits (the library promises reproducible steps).

Error bounds (u = 2^-24, gamma(n) = n u / (1 - n u), the standard bound of an n-term dot product in any summation order, FMA or not):
  fp32 FFMA paths   |got - ref| <= gamma(C + 4) (|alpha| (|A| |B|)_ij + |b_j|)      C = contraction length; the 4 covers the alpha
                    product (applied per partial sum on split paths), the bias add and the partial-sum pass;
                    TANH adds the 2-ulp error of tanhf (CUDA programming guide): 2^-22 |y|.  Accumulation (data-grad `accumulate`,
                    weight-grad into out_w / out_b) treats the previous value as one more summand -- the ordered partial pass
                    (add_partials) starts from it -- so |prev| joins the absolute sum and C + 4 becomes C + 5.
  3xFP16 path       (a) the kernel against the float64 product of its own fp16 companions (oracle/fp16x3_model.py split):
                    inside a promotion chunk of L contraction elements the tensor core adds 3L exact fp16 products with
                    TRUNCATION (unit 2^-23, not 2^-24), every added product and the final normalisation losing < 1 ulp of the running
                    magnitude <= the chunk's absolute sum: gamma_t(3L + 1) with gamma_t built on 2^-23; each chunk is then promoted
                    with one round-to-nearest FMA, the split-K slices summed in fp32, and the epilogue adds the bias as
                    fl(b * fl(1 / alpha)) and multiplies by alpha: gamma(chunks + splits + 3) on the product, gamma(4) on |b|
                    (accumulation as above: gamma(chunks + splits + 4) on |alpha| S_abs + |prev|).
                    (b) that companion product against the exact float64 product: the representation error documented in the
                    kernel header -- per element |x - (hi + lo) / s| <= 2^-21 |x| + 2^-39 max|x| -- plus the dropped lo*lo term,
                    |lo| / s <= 2^-11 |x| + 2^-38 max|x|.
"""
import math
import os
import re

import pytest
import torch

from gcbf_b200 import _C, ops

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0') if torch.cuda.is_available() else None

NUM_SMS = 132            # kNumSMs (csrc/common.cuh): the split rules of the kernels are written for the H100 SXM
PRODUCTS = ('fwd', 'dgrad', 'wgrad')


# ---- the dispatch rule, mirrored --------------------------------------------------------------------------------------------------
def use_h_rule(M, N, K):
    """gcbf_linear_h_supported / ops.use_h with GEMM_IMPL = 0: the [M,K] x [N,K] layer runs on the wgmma kernel."""
    return M >= 256 and N >= 96 and K >= 96 and M * N * K >= (1 << 24)


def _skinny(M, N, K):
    return K <= 16 and N >= 64 and M >= 64


def _tiny(N, K):
    return N <= 32 and K <= 256


def _fewrows(M, N, K):
    return 1 <= M <= 64 and N >= 64 and K >= 32


def _narrow(M, N, K):
    return 1 <= M <= 64 and 1 <= K <= 32 and N >= 64


def _cdiv(a, b):
    return -(-a // b)


def _tc_kch(product):
    """k-blocks (32 K-elements each) per promotion chunk of the wgmma kernel: g_kch / g_kch_dgrad and their environment overrides."""
    kc, kd = os.environ.get('GCBF_TC_KCH'), os.environ.get('GCBF_TC_KCH_DGRAD')
    kch = int(kc) if kc and 1 <= int(kc) <= 8 else 4
    kch_d = int(kd) if kd and 1 <= int(kd) <= 8 else ((kch if kch > 4 else 8) if kc else 8)
    return kch_d if product == 'dgrad' else kch


def wgmma_wgrad_splits(M, N, K):
    """Contraction splits of the wgmma weight-grad (gcbf_linear_bwd_weight_h, then th::launch's chunk rounding)."""
    bn = 256 if K > 128 else 128
    tiles = _cdiv(N, 128) * _cdiv(K, bn)
    splits = max(1, min(_cdiv(M, 256), NUM_SMS // tiles)) if tiles < NUM_SMS else 1
    kblocks, kch = _cdiv(M, 32), _tc_kch('wgrad')
    kps = _cdiv(_cdiv(kblocks, splits), kch) * kch
    return _cdiv(kblocks, kps)


def expected_impl(product, M, N, K):
    """(gcbf_last_gemm_impl value, variant) of one product of the [M,K] x [N,K] layer; impl 2 = the wgmma kernel (ops.use_h)."""
    if use_h_rule(M, N, K):
        bn = 256 if (N if product == 'fwd' else K) > 128 else 128
        split = '-splitk' if product == 'wgrad' and wgmma_wgrad_splits(M, N, K) > 1 else ''
        return 2, f'bn{bn}{split}'
    if _skinny(M, N, K):
        return 3, ''
    if product == 'fwd':
        return (4, '') if _tiny(N, K) else ((5, 'fewrows') if _fewrows(M, N, K) else (1, ''))
    if product == 'dgrad':
        if _tiny(N, K):
            return 4, ''
        if _fewrows(M, K, N):              # output width K, contraction N
            return 5, 'fewrows'
        return (5, 'narrow') if _narrow(M, N, K) else (1, '')
    return (5, 'fewrows') if _fewrows(M, N, K) else (1, '')


LAYOUTS = ('aligned', 'odd')


def kernel_variant(product, M, N, K, layout):
    """(impl, variant, kernel-name fragment or None) for one layout.  Where two kernels of an implementation are chosen by operand
    alignment (few-rows tiled vs its fallback, skinny data-grad with W^T resident vs chunked) the kernel name tells them apart; the
    float4 / scalar branches inside the SIMT, skinny and tiny kernels are not observable from outside (`vec_ok` flags) and are only
    exercised, by the two layouts."""
    impl, var = expected_impl(product, M, N, K)
    aligned = layout == 'aligned'
    if impl == 2:
        return impl, var, f'gemm_h_kernel<{var[2:5]}'
    if impl == 5 and product == 'fwd':
        tiled = aligned and K % 4 == 0
        return impl, 'tiled' if tiled else 'fallback', 'fewrows_fwd_tiled_kernel' if tiled else 'fewrows_fwd_kernel'
    if impl == 5 and product == 'dgrad' and var == 'fewrows':
        tiled = aligned and K % 4 == 0 and N % 4 == 0
        return impl, 'tiled' if tiled else 'fallback', 'fewrows_dgrad_tiled_kernel' if tiled else 'fewrows_dgrad_kernel'
    if impl == 5:
        return impl, var, 'fewrows_dgrad_narrow_kernel' if var == 'narrow' else 'fewrows_wgrad_kernel'
    if impl == 3 and product == 'dgrad':
        full = aligned and N % 4 == 0 and N <= 3072 and M >= 4096
        return impl, 'full' if full else 'chunked', 'skinny_dgrad_full_kernel' if full else 'skinny_dgrad_kernel'
    return impl, var, None


# ---- the case table: shapes on both sides of every threshold of the dispatch rule (tests/test_linear_paths_cpu.py checks that) ----
CASES = [
    # skinny-K (K <= 16, N >= 64, M >= 64) and its W^T-resident data-grad (M >= 4096)
    (64, 64, 16), (64, 64, 17), (63, 64, 16), (64, 63, 16), (4096, 256, 13),
    # tiny-N (N <= 32, K <= 256)
    (300, 32, 256), (300, 33, 256), (300, 32, 257), (300, 1, 17),
    # few-rows (M <= 64, N >= 64, K >= 32): tiled cluster kernels (cluster split up to 8) and the unaligned fallback
    (1, 64, 32), (64, 64, 32), (65, 64, 32), (64, 63, 32), (64, 64, 31), (1, 256, 2048), (4, 256, 2048), (16, 2048, 2048),
    (44, 128, 1026),
    # few-rows data-grad (output width K >= 64, contraction N >= 32) and the narrow data-grad (K <= 32)
    (16, 256, 63), (16, 256, 64), (16, 31, 512), (16, 32, 512), (8, 256, 32), (8, 256, 33),
    # SIMT: ragged 128 x 128 tiles, split-K weight-grad
    (127, 130, 260), (129, 130, 260),
    # wgmma: M / N / K thresholds, M*N*K = 2^24 exactly and one row below, tile width 128 vs 256, split-K weight-grad
    (255, 512, 512), (256, 512, 512), (2048, 95, 96), (2048, 96, 96), (2048, 96, 95), (1023, 128, 128), (1024, 128, 128),
    (512, 128, 256), (512, 129, 256), (512, 256, 128), (512, 256, 129), (8192, 128, 128), (256, 512, 128),
]


# ---- error bounds -------------------------------------------------------------------------------------------------------------
U = 2.0 ** -24


def gamma(n):
    return n * U / (1.0 - n * U)


def gamma_t(n):
    """gamma with the unit roundoff of truncation (2^-23): the tensor core's in-chunk accumulation."""
    return n * 2.0 ** -23 / (1.0 - n * 2.0 ** -23)


TANH_ULP = 2.0 ** -22     # tanhf: 2 ulp (CUDA C programming guide, single-precision functions); 2 ulp(y) <= 2^-22 |y|


def _act64(z, act):
    return torch.relu(z) if act == ops.ACT_RELU else (torch.tanh(z) if act == ops.ACT_TANH else z)


def _act_bound(pre_bound, ref, act):
    """Bound after the activation: ReLU and tanh are 1-Lipschitz; tanhf adds its own 2 ulp."""
    return pre_bound + TANH_ULP * (ref.abs() + pre_bound) if act == ops.ACT_TANH else pre_bound


def assert_within(got, ref, bound, what):
    """Per-element |got - ref| <= bound; NaN (an over-read, an unwritten output) fails."""
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    if bool(bad.any()):
        i = int(bad.reshape(-1).nonzero()[0])
        idx = tuple(int(v) for v in torch.unravel_index(torch.tensor(i), tuple(got.shape)))
        raise AssertionError(f'{what}: {int(bad.sum())} of {got.numel()} elements outside the bound; first at {idx}: '
                             f'got {got.reshape(-1)[i].item()!r} want {ref.reshape(-1)[i].item()!r} bound {bound.reshape(-1)[i].item():.3e}')


def _split64(t):
    """(hi / s, lo / s) in float64 (exact: s is a power of two) of the fp16 companion the library makes of `t`."""
    import fp16x3_model as F16
    hi, lo, s = F16.split(t)
    return hi.double() / s, lo.double() / s


def _doc_repr(t):
    """Documented representation bounds of the companion of t: (|x - (hi+lo)/s| bound, |lo|/s bound), per element."""
    a, amax = t.double().abs(), t.double().abs().max()
    return 2.0 ** -21 * a + 2.0 ** -39 * amax, 2.0 ** -11 * a + 2.0 ** -38 * amax


class Product:
    """C = A @ B of one product in float64, with the operands as matrices: the fp32 sources and (3xFP16 path) their companions."""

    def __init__(self, A, B, A_src, A_T, B_src, B_T):
        # A_src / B_src: the tensors the library splits; A_T / B_T: whether A / B are their transposes
        self.A, self.B = A.double(), B.double()
        self.S = self.A @ self.B
        self.P = self.A.abs() @ self.B.abs()
        self.srcs = (A_src, A_T, B_src, B_T)

    def h_model(self):
        """(S_model, S_abs): the companion product hi*hi + lo*hi + hi*lo and its absolute sum, descaled."""
        A_src, A_T, B_src, B_T = self.srcs
        ah, al = _split64(A_src)
        bh, bl = _split64(B_src)
        if A_T:
            ah, al = ah.t(), al.t()
        if B_T:
            bh, bl = bh.t(), bl.t()
        S = ah @ bh + al @ bh + ah @ bl
        Sa = ah.abs() @ bh.abs() + al.abs() @ bh.abs() + ah.abs() @ bl.abs()
        return S, Sa

    def repr_bound(self):
        """(b): |S_model - S| from the documented per-element representation error and the dropped lo*lo term."""
        A_src, A_T, B_src, B_T = self.srcs
        (da, la), (db, lb) = _doc_repr(A_src), _doc_repr(B_src)
        if A_T:
            da, la = da.t(), la.t()
        if B_T:
            db, lb = db.t(), lb.t()
        return self.A.abs() @ db + da @ self.B.abs() + da @ db + la @ lb


# ---- operand buffers with NaN padding -----------------------------------------------------------------------------------------
class Buf:
    """A [rows, cols] operand as a column slice of a NaN-filled buffer with one extra padding row.  'aligned': pitch = 0 mod 4,
    16-byte aligned base; 'odd': odd pitch, base one float in."""

    def __init__(self, t, layout, fill=None):
        rows, cols = t.shape
        self.off = 0 if layout == 'aligned' else 1
        self.pitch = (cols + 3) // 4 * 4 + 4 if layout == 'aligned' else (cols + 1 if (cols + 1) % 2 else cols + 2)
        self.buf = torch.full((rows + 1, self.pitch), float('nan'), device=DEV)
        self.view = self.buf[:rows, self.off:self.off + cols]
        self.view.copy_(t if fill is None else torch.full_like(t, fill))
        self.shape = (rows, cols)
        self.init = self.buf.clone()

    def reset(self):
        self.buf.copy_(self.init)

    def pads_intact(self):
        inside = torch.zeros_like(self.buf, dtype=torch.bool)
        inside[:self.shape[0], self.off:self.off + self.shape[1]] = True
        return torch.equal(self.buf.view(torch.int32)[~inside], self.init.view(torch.int32)[~inside])

    def unchanged(self):
        return torch.equal(self.buf.view(torch.int32), self.init.view(torch.int32))


class Vec:
    """A [n] vector inside a NaN-filled buffer (one float in for the odd layout)."""

    def __init__(self, t, layout):
        n = t.numel()
        self.off = 0 if layout == 'aligned' else 1
        self.buf = torch.full((n + 2,), float('nan'), device=DEV)
        self.view = self.buf[self.off:self.off + n]
        self.view.copy_(t)
        self.init = self.buf.clone()

    def reset(self):
        self.buf.copy_(self.init)

    def pads_intact(self):
        inside = torch.zeros_like(self.buf, dtype=torch.bool)
        inside[self.off:self.off + self.view.numel()] = True
        return torch.equal(self.buf.view(torch.int32)[~inside], self.init.view(torch.int32)[~inside])

    def unchanged(self):
        return torch.equal(self.buf.view(torch.int32), self.init.view(torch.int32))


def _bits(t):
    return t.view(torch.int32).clone()


def run_twice(fn, outs):
    """fn() twice from the same output state: the bits must agree (fixed-order reductions: split-K, clusters, partial sums)."""
    fn()
    first = [_bits(o.buf) for o in outs]
    for o in outs:
        o.reset()
    fn()
    for o, f in zip(outs, first):
        assert torch.equal(_bits(o.buf), f), 'two identical calls gave different bits'


def kernels_launched(fn):
    """Names of the CUDA kernels fn launches (torch.profiler): distinguishes two kernels of one implementation."""
    from torch.profiler import ProfilerActivity, profile
    for _ in range(3):      # a session occasionally delivers no device records at all: observe again (fn is idempotent here)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            fn()
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        if names:
            return names
    raise AssertionError('the profiler saw no kernel')


# ---- inputs -------------------------------------------------------------------------------------------------------------------
def _g(seed):
    g = torch.Generator(device='cpu')
    g.manual_seed(seed)
    return g


def _spread(rows, cols, g, h):
    """Uniform(-1, 1) rows spread over six decades (torch.logspace), a whole zero row; for the 3xFP16 path the max is pinned to 1.5
    (scale 2^14) and a row holds values just below / above the fp16 normal threshold 2^-14 after scaling."""
    t = torch.rand(rows, cols, generator=g) * 2 - 1
    if rows > 1:
        t *= torch.logspace(0, -6, rows).unsqueeze(1)
    if rows > 2:
        t[rows // 2] = 0
    if h and rows > 2 and cols >= 4:
        t[0, 0] = 1.5
        t[1, :4] = torch.tensor([1 - 2.0 ** -6, 1 + 2.0 ** -6, -(1 - 2.0 ** -11), 1 + 2.0 ** -11]) * 2.0 ** -28
    return t


def _relu_src(M, K, g):
    """Mask source with exact +0.0 and -0.0 entries: both are 'off' (mask = src > 0)."""
    t = torch.randn(M, K, generator=g)
    flat = t.view(-1)
    flat[0::8] = 0.0
    flat[1::8] = -0.0
    return t


def _inputs(M, N, K, h):
    g = _g(M * 1000003 + N * 1009 + K)
    x, W, dz = _spread(M, K, g, h), _spread(N, K, g, h), _spread(M, N, g, h)
    b = torch.randn(N, generator=g)
    return dict(x=x.to(DEV), W=W.to(DEV), dz=dz.to(DEV), b=b.to(DEV), relu=_relu_src(M, K, g).to(DEV),
                prev_x=torch.randn(M, K, generator=g).to(DEV), prev_w=torch.randn(N, K, generator=g).to(DEV),
                prev_b=torch.randn(N, generator=g).to(DEV))


ALPHA = 0.7      # 1/sigma stand-in, deliberately not 1


def _alpha(on):
    return torch.tensor([ALPHA], device=DEV) if on else None


def _ld(v):
    return v.stride(0)


# ---- the three products -------------------------------------------------------------------------------------------------------
def _check_impl(product, M, N, K, layout, fn, check_kernel):
    """gcbf_last_gemm_impl (not set by the wgmma path, which ops.use_h selects) and, with check_kernel, the kernel that ran."""
    impl, var, kname = kernel_variant(product, M, N, K, layout)
    if impl != 2:
        assert _C.lib().gcbf_last_gemm_impl() == impl, (product, M, N, K, _C.lib().gcbf_last_gemm_impl(), impl)
    if check_kernel and kname is not None:
        names = [re.sub(r'\(int\)|\s', '', n) for n in kernels_launched(fn)]      # 'gemm_h_kernel<(int)256, ...' -> '<256,'
        assert any(kname in n for n in names), (product, M, N, K, layout, kname, names)


def check_fwd(c, layout, M, N, K, act, with_b, with_a, check_kernel):
    h = use_h_rule(M, N, K)
    x, W = Buf(c['x'], layout), Buf(c['W'], layout)
    b = Vec(c['b'], layout) if with_b else None
    y = Buf(torch.empty(M, N, device=DEV), layout, fill=float('nan'))
    am = Vec(torch.tensor([0x7f7fffff], dtype=torch.int32).view(torch.float32).to(DEV), layout)   # garbage: must be reset
    alpha = _alpha(with_a)

    def call():
        ops.linear_fwd(x.view, W.view, b.view if b else None, alpha, act, out=y.view, out_amax=am.view.view(torch.int32))
    run_twice(call, [y, am])
    _check_impl('fwd', M, N, K, layout, call, check_kernel)
    a = ALPHA if with_a else 1.0
    bias = c['b'].double() if with_b else torch.zeros(N, device=DEV, dtype=torch.float64)
    pr = Product(c['x'], c['W'].t(), c['x'], False, c['W'], True)
    what = f'fwd {M}x{N}x{K} {layout} act={act} bias={with_b} alpha={with_a}'
    if h:
        Sm, Sa = pr.h_model()
        L = 32 * _tc_kch('fwd')
        # the bias enters as fl(b * fl(1 / alpha)), is added and multiplied by alpha: four roundings
        pre = abs(a) * (gamma_t(3 * L + 1) + gamma(_cdiv(K, L) + 3)) * Sa + gamma(4) * bias.abs()
        ref = _act64(a * Sm + bias, act)
        assert_within(y.view, ref, _act_bound(pre, ref, act), what + ' (a) vs companion product')
        assert_within(Sm, pr.S, pr.repr_bound(), what + ' (b) companion product vs exact')
    else:
        ref = _act64(a * pr.S + bias, act)
        pre = gamma(K + 4) * (abs(a) * pr.P + bias.abs())
        assert_within(y.view, ref, _act_bound(pre, ref, act), what)
    # max|y| of the epilogue / amax pass, bit for bit
    assert am.view.view(torch.int32).item() == y.view.abs().max().view(torch.int32).item(), what + ' out_amax'
    assert y.pads_intact() and am.pads_intact() and x.unchanged() and W.unchanged() and (b is None or b.unchanged()), \
        what + ' padding / inputs'


def check_dgrad(c, layout, M, N, K, with_mask, acc, with_a, check_kernel):
    h = use_h_rule(M, N, K)
    dz, W = Buf(c['dz'], layout), Buf(c['W'], layout)
    rs = Buf(c['relu'], layout) if with_mask else None
    dx = Buf(c['prev_x'], layout) if acc else Buf(torch.empty(M, K, device=DEV), layout, fill=float('nan'))
    alpha = _alpha(with_a)

    def call():
        ops.linear_bwd_data(dz.view, W.view, alpha, rs.view if rs else None, out=dx.view, accumulate=acc)
    run_twice(call, [dx])
    _check_impl('dgrad', M, N, K, layout, call, check_kernel)
    a = ALPHA if with_a else 1.0
    what = f'dgrad {M}x{N}x{K} {layout} mask={with_mask} acc={acc} alpha={with_a}'
    pr = Product(c['dz'], c['W'], c['dz'], False, c['W'], False)
    mask = (c['relu'] > 0) if with_mask else torch.ones(M, K, dtype=torch.bool, device=DEV)
    prev = c['prev_x'].double() if acc else torch.zeros(M, K, device=DEV, dtype=torch.float64)
    # accumulation: the previous value is one more summand of the sum (the ordered partial pass starts from it), not a last add
    if h:
        Sm, Sa = pr.h_model()
        L = 32 * _tc_kch('dgrad')
        v_ref = a * Sm
        bound = abs(a) * gamma_t(3 * L + 1) * Sa * mask + gamma(_cdiv(N, L) + 4) * (abs(a) * Sa * mask + prev.abs())
        assert_within(Sm, pr.S, pr.repr_bound(), what + ' (b) companion product vs exact')
    else:
        v_ref = a * pr.S
        bound = gamma(N + 5) * (abs(a) * pr.P * mask + prev.abs())
    ref = prev + v_ref * mask
    assert_within(dx.view, ref, bound, what)
    # masked entries (src <= 0, including +-0.0) are exactly off: 0, or the untouched previous value
    off = ~mask
    assert torch.equal(dx.view[off], c['prev_x'][off] if acc else torch.zeros_like(dx.view[off])), what + ' masked entries'
    assert dx.pads_intact() and dz.unchanged() and W.unchanged() and (rs is None or rs.unchanged()), what + ' padding / inputs'


def check_wgrad(c, layout, M, N, K, acc, with_a, with_b, check_kernel):
    h = use_h_rule(M, N, K)
    dz, x = Buf(c['dz'], layout), Buf(c['x'], layout)
    dW = Buf(c['prev_w'], layout) if acc else Buf(torch.empty(N, K, device=DEV), layout, fill=float('nan'))
    db = (Vec(c['prev_b'], layout) if acc else Vec(torch.full((N,), float('nan'), device=DEV), layout)) if with_b else None
    alpha = _alpha(with_a)

    def call():
        if acc:
            ops.linear_bwd_weight(dz.view, x.view, alpha, need_bias=with_b, out_w=dW.view, out_b=db.view if db else None)
        elif h:
            dzh = ops.split_h(dz.view, colsum=db.view if db else None)
            ops.linear_bwd_weight_h(dzh, ops.split_h(x.view), alpha, out=dW.view, accumulate=False)
        else:
            _C.call('gcbf_linear_bwd_weight', _C.ptr(dz.view), _ld(dz.view), _C.ptr(x.view), _ld(x.view), _C.ptr(alpha), _C.ptr(dW.view),
                    _ld(dW.view), _C.ptr(db.view) if db else None, M, N, K, 0, 0)
    run_twice(call, [dW] + ([db] if db else []))
    _check_impl('wgrad', M, N, K, layout, call, check_kernel)
    a = ALPHA if with_a else 1.0
    what = f'wgrad {M}x{N}x{K} {layout} acc={acc} alpha={with_a} bias={with_b}'
    pr = Product(c['dz'].t(), c['x'], c['dz'], True, c['x'], False)
    prev = c['prev_w'].double() if acc else torch.zeros(N, K, device=DEV, dtype=torch.float64)
    if h:
        Sm, Sa = pr.h_model()
        L = 32 * _tc_kch('wgrad')
        splits = wgmma_wgrad_splits(M, N, K)
        v_ref = a * Sm
        bound = abs(a) * gamma_t(3 * L + 1) * Sa + gamma(_cdiv(M, L) + splits + 4) * (abs(a) * Sa + prev.abs())
        assert_within(Sm, pr.S, pr.repr_bound(), what + ' (b) companion product vs exact')
    else:
        v_ref = a * pr.S
        bound = gamma(M + 5) * (abs(a) * pr.P + prev.abs())
    assert_within(dW.view, prev + v_ref, bound, what)
    if db:
        dz64 = c['dz'].double()
        prev_b = c['prev_b'].double() if acc else torch.zeros(N, device=DEV, dtype=torch.float64)
        # column sums: M terms, the ordered partial pass, the previous value as one more summand
        assert_within(db.view, prev_b + dz64.sum(0), gamma(M + 3) * (dz64.abs().sum(0) + prev_b.abs()), what + ' db')
        assert db.pads_intact(), what + ' db padding'
    assert dW.pads_intact() and dz.unchanged() and x.unchanged(), what + ' padding / inputs'


# options: every one on every path in each layout, and the interacting combinations (mask + accumulate, bias + alpha + TANH)
def fwd_options(layout):
    flip = layout == 'odd'
    return [(ops.ACT_NONE, flip, not flip), (ops.ACT_RELU, not flip, flip), (ops.ACT_TANH, True, True)]


def dgrad_options(layout):
    flip = layout == 'odd'
    return [(True, False, not flip), (True, True, flip), (False, True, not flip), (False, False, flip)]


def wgrad_options(layout):
    flip = layout == 'odd'
    return [(False, not flip, not flip), (True, flip, True)]      # (accumulate, alpha, bias)


@pytest.fixture(autouse=True)
def _auto_dispatch():
    assert ops.GEMM_IMPL == 0 and ops.USE_WGMMA, 'these tests check the automatic dispatch'
    yield


@pytest.mark.parametrize('layout', LAYOUTS)
@pytest.mark.parametrize('M,N,K', CASES)
def test_linear_paths(M, N, K, layout):
    h = use_h_rule(M, N, K)
    assert ops.use_h(M, N, K) == h and bool(_C.lib().gcbf_linear_h_supported(M, N, K)) == h, 'dispatch mirror out of date'
    if h and not _C.lib().gcbf_has_wgmma():
        pytest.fail('library built without the wgmma path')
    c = _inputs(M, N, K, h)
    for i, (act, with_b, with_a) in enumerate(fwd_options(layout)):
        check_fwd(c, layout, M, N, K, act, with_b, with_a, check_kernel=i == 0)
    for i, (mask, acc, with_a) in enumerate(dgrad_options(layout)):
        check_dgrad(c, layout, M, N, K, mask, acc, with_a, check_kernel=i == 0)
    for i, (acc, with_a, with_b) in enumerate(wgrad_options(layout)):
        check_wgrad(c, layout, M, N, K, acc, with_a, with_b, check_kernel=i == 0)


@pytest.mark.parametrize('N,K', [(64, 16), (32, 128), (256, 2048), (130, 260)])
def test_linear_zero_rows(N, K):
    """M = 0: the forward resets out_amax to 0; the weight-grad zeroes dW / db unless it accumulates, then leaves them alone; the
    data-grad writes nothing.  (Skinny, tiny, few-rows-width and SIMT-width layers; the dispatcher returns before choosing.)"""
    x, dz = torch.empty(0, K, device=DEV), torch.empty(0, N, device=DEV)
    W = Buf(torch.randn(N, K, device=DEV), 'odd')
    am = torch.tensor([12345], dtype=torch.int32, device=DEV)
    y = ops.linear_fwd(x, W.view, torch.randn(N, device=DEV), _alpha(True), ops.ACT_TANH, out_amax=am)
    assert y.shape == (0, N) and am.item() == 0
    dx = ops.linear_bwd_data(dz, W.view, _alpha(True), None)
    assert dx.shape == (0, K)
    for acc in (False, True):
        dW = Buf(torch.randn(N, K, device=DEV), 'odd')
        db = Vec(torch.randn(N, device=DEV), 'odd')
        _C.call('gcbf_linear_bwd_weight', None, N, None, K, None, _C.ptr(dW.view), _ld(dW.view), _C.ptr(db.view), 0, N, K, int(acc), 0)
        if acc:
            assert dW.unchanged() and db.unchanged()
        else:
            assert torch.equal(dW.view, torch.zeros(N, K, device=DEV)) and torch.equal(db.view, torch.zeros(N, device=DEV))
            assert dW.pads_intact() and db.pads_intact()
    assert W.unchanged()


@pytest.mark.parametrize('zero', ['x', 'W', 'dz'])
def test_wgmma_zero_operand(zero):
    """An all-zero operand has amax 0, so its companion scale is 1 (and all planes zero): the products must be exact zeros (plus the
    bias, through the epilogue's (v + b / alpha) * alpha: three roundings)."""
    M, N, K = 512, 256, 256
    assert use_h_rule(M, N, K)
    c = _inputs(M, N, K, True)
    c[zero].zero_()
    for act, with_b, with_a in fwd_options('aligned'):
        check_fwd(c, 'aligned', M, N, K, act, with_b, with_a, check_kernel=False)
    for mask, acc, with_a in dgrad_options('aligned'):
        check_dgrad(c, 'aligned', M, N, K, mask, acc, with_a, check_kernel=False)
    for acc, with_a, with_b in wgrad_options('aligned'):
        check_wgrad(c, 'aligned', M, N, K, acc, with_a, with_b, check_kernel=False)


# ---- spectral norm ------------------------------------------------------------------------------------------------------------
SN_SHAPES = [(2048, 13), (2048, 2048), (256, 2048), (128, 256), (1, 128), (2, 128)]


def _normalize_bound(t, e):
    """Per-element bound on fl(t / ||t||) when t carries the per-element error e: first order |e_k| / ||t|| + |v_k| (||e|| / ||t|| +
    gamma(n + 3)) (the norm's n fused squares, the sqrt, the division), times 1.01 for the second-order terms."""
    nrm = t.norm()
    return 1.01 * (e / nrm + (t / nrm).abs() * (e.norm() / nrm + gamma(t.numel() + 3)))


@pytest.mark.parametrize('batched', [False, True])
def test_sn_power_iter_float64(batched):
    """One power iteration (v = normalize(W^T u0), u = normalize(W v), 1/sigma = 1 / (u . W v)) of the layers the nets use,
    against float64.  v is compared with the float64 step from u0; u and 1/sigma with the float64 step from the kernel's v, so each
    half is checked at its own rounding bound: gamma(n) for the n-term products W^T u (n = N) and W v (n = K)."""
    g = _g(77)
    specs, u0s = [], []
    for N, K in SN_SHAPES:
        W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(DEV)
        u0 = torch.nn.functional.normalize(torch.randn(N, generator=g), dim=0).to(DEV)
        v0 = torch.nn.functional.normalize(torch.randn(K, generator=g), dim=0).to(DEV)
        specs.append(ops.LinearSpec(W, torch.zeros(N, device=DEV), u0.clone(), v0.clone()))
        u0s.append(u0)
    if batched:
        invs, _ = ops.sn_power_iter_batched(specs)
    else:
        invs = [ops.sn_power_iter(L.W, L.u, L.v) for L in specs]
    for L, u0, inv in zip(specs, u0s, invs):
        N, K = L.W.shape
        W64 = L.W.double()
        t = W64.t() @ u0.double()
        assert_within(L.v, t / t.norm(), _normalize_bound(t, gamma(N) * (W64.abs().t() @ u0.double().abs())), f'v {N}x{K}')
        s = W64 @ L.v.double()
        e_s = gamma(K) * (W64.abs() @ L.v.double().abs())
        assert_within(L.u, s / s.norm(), _normalize_bound(s, e_s), f'u {N}x{K}')
        # sigma = sum_n u_n s_n = ||s~||^2 / fl(||s~||): |sigma - ||s||| <= ||e_s|| + ||s|| gamma(2N + 2) (the norm, the N-term dot
        # product and the divisions); 1/sigma adds one rounding
        sig, sig_b = s.norm(), e_s.norm() + s.norm() * gamma(2 * N + 2)
        inv_ref = 1.0 / sig
        assert_within(inv.reshape(1), inv_ref.reshape(1), (inv_ref * (sig_b / (sig - sig_b) + U) * 1.01).reshape(1), f'1/sigma {N}x{K}')


@pytest.mark.parametrize('N,K', SN_SHAPES)
@pytest.mark.parametrize('into_acc', [False, True])
def test_sn_grad_fixup_float64(N, K, into_acc):
    """dW - <dW, W> (1/sigma) u v^T against float64 with the kernel's own u, v, 1/sigma: the check is on the fix-up alone.  Bound:
    the float64 inner product (|err| <= NK 2^-53 sum|dW W|) rounded to fp32 and multiplied by 1/sigma (2 roundings), the two products
    with u_r and v_c and the subtraction: gamma(5) |c u_r v_c| + u |g|; the acc variant adds u |acc + g|.  A coefficient off by 1 %
    moves every element by 1e-2 |c u_r v_c|, far outside."""
    g = _g(N * 7 + K)
    W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(DEV)
    u = torch.nn.functional.normalize(torch.randn(N, generator=g), dim=0).to(DEV)
    v = torch.nn.functional.normalize(torch.randn(K, generator=g), dim=0).to(DEV)
    inv = ops.sn_power_iter(W, u, v)
    # a gradient with a large component along W (a sizeable correction) plus noise
    G = (torch.randn(N, K, generator=g).to(DEV) * 0.1 + 3.0 * W).contiguous()
    dW = G.clone()
    acc0 = torch.randn(N, K, generator=g).to(DEV)
    acc = acc0.clone() if into_acc else None
    ops.sn_grad_fixup(dW, W, u, v, inv, acc=acc)
    G64, W64 = G.double(), W.double()
    inner = (G64 * W64).sum()
    inner_err = N * K * 2.0 ** -53 * (G64 * W64).abs().sum()
    inv64 = inv.double()
    cuv = (inner * inv64) * torch.outer(u.double(), v.double())
    ref = G64 - cuv
    bound = gamma(5) * cuv.abs() + inner_err * inv64.abs() * torch.outer(u.double(), v.double()).abs() + U * ref.abs()
    assert cuv.abs().max() > 1e-3 * G64.abs().max(), 'the correction must be visible next to the gradient'
    if into_acc:
        ref_acc = acc0.double() + ref
        assert_within(acc, ref_acc, bound * (1 + U) + U * ref_acc.abs(), f'fixup acc {N}x{K}')
        assert torch.equal(dW, G), 'the acc variant must leave dW alone'
    else:
        assert_within(dW, ref, bound, f'fixup {N}x{K}')
