"""Host-side orchestration of the sm_90a kernels: raw op wrappers (one C-ABI call each) and the two
autograd.Functions the nn.Modules are built from.

    GNNNetFunction   edge-MLP phi -> attention aggregation -> node-MLP gamma [-> row select -> head MLP]
                     = CBFGNNLayer / ControllerGNNLayer (reference gcbf/nn/gnn.py:14-36, 56-73), optionally fused
                     with CBFGNN.forward / GNNController.forward (gcbf/algo/gcbf.py:37-55,
                     gcbf/controller/gnn_controller.py:29-48)
    MLPFunction      gcbf.nn.MLP.forward (gcbf/nn/mlp.py:44-47)

torch is used for device memory (torch.empty / zeros), streams and autograd bookkeeping only; every
arithmetic step is a kernel of libgcbf_b200.so.  No CPU fallback: CPU tensors raise.
"""
import ctypes
import os
from dataclasses import dataclass, field
from typing import List, Optional, Sequence, Tuple

import torch

from . import _C, native
from .arena import ARENA, empty as _empty, zeros as _zeros
from ._C import call, ptr

ACT_NONE, ACT_RELU, ACT_TANH = 0, 1, 2
# GCBF_NATIVE=0 keeps the per-kernel Python sequencing of round 1 (net_forward / net_backward below) instead of the chain-level
# entry points of the library (csrc/net.cu, csrc/step.cu): same kernels, same order -- an A/B switch for debugging only.
NATIVE = os.environ.get('GCBF_NATIVE', '1') != '0'
ENV_IDS = {'SimpleCar': 0, 'DubinsCar': 1, 'SimpleDrone': 2}
GEMM_IMPL = 0   # 0 auto, 1 force fp32 SIMT, 2 force wgmma (tests flip this)


class _GemmTimer:
    """Optional CUDA-event timing of every linear-layer launch (bench.py's roofline numbers).  Events are recorded
    on the launching stream around each C-ABI GEMM call; summary() synchronises and adds them up.  Operand preparation
    of the tensor-core path (amax + fp16 [hi|lo] split, shared by the GEMMs a matrix takes part in) is timed separately."""

    def __init__(self):
        self.on = False
        self.records = []
        self.prep = []

    def enable(self):
        self.on, self.records, self.prep = True, [], []
        native.fn('gcbf_timing_enable')(1)

    def disable(self):
        self.on, self.records, self.prep = False, [], []
        native.fn('gcbf_timing_enable')(0)

    def _collect_native(self):
        """(ms, flops, kind, M, N, K) records of the launches the chain-level entry points made (csrc/net.cu `Timed`)."""
        cap = 1 << 16
        buf = (native.TimeRec * cap)()
        cnt = ctypes.c_int(0)
        native.check(native.fn('gcbf_timing_collect')(buf, cap, ctypes.byref(cnt)), 'gcbf_timing_collect')
        return [(buf[i].ms, buf[i].flops, buf[i].kind, buf[i].M, buf[i].N, buf[i].K) for i in range(min(cnt.value, cap))]

    def run(self, flops, fn, impl=None, tag=None):
        if not self.on:
            return fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        self.records.append((e0, e1, flops, impl if impl is not None else _C.lib().gcbf_last_gemm_impl(), tag))

    def run_prep(self, fn):
        if not self.on:
            return fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        self.prep.append((e0, e1))

    def summary(self):
        torch.cuda.synchronize()
        by = {1: [0.0, 0.0, 0], 2: [0.0, 0.0, 0]}
        shapes = {}
        for e0, e1, flops, impl, tag in self.records:
            b = by.get(impl, by[1])
            ms = e0.elapsed_time(e1)
            b[0] += ms
            b[1] += flops
            b[2] += 1
            if tag is not None and impl == 2:
                t = shapes.setdefault(tag, [0.0, 0.0, 0])
                t[0] += ms
                t[1] += flops
                t[2] += 1
        prep_ms = sum(e0.elapsed_time(e1) for e0, e1 in self.prep)
        nprep = len(self.prep)
        for ms, flops, kind, M, N, K in self._collect_native():
            if kind == 4:
                prep_ms += ms
                nprep += 1
                continue
            b = by[2] if kind in (0, 1, 2) else by[1]
            b[0] += ms
            b[1] += flops
            b[2] += 1
            if kind in (0, 1, 2):
                t = shapes.setdefault((('forward', 'data-grad', 'weight-grad')[kind], M, N, K), [0.0, 0.0, 0])
                t[0] += ms
                t[1] += flops
                t[2] += 1
        tensor = by[2][1] > by[1][1]
        ms, flops, n = by[2] if tensor else by[1]
        dominant = None
        if shapes:
            tag, (tms, tfl, tn) = max(shapes.items(), key=lambda kv: kv[1][0])
            dominant = dict(product=tag[0], M=tag[1], N=tag[2], K=tag[3], launches=tn, ms_per_launch=tms / tn, flops_per_launch=tfl / tn)
        return dict(kernel='gemm_wgmma_3xfp16' if tensor else 'gemm_simt_kernel', ms=ms, flops=flops, launches=n, tensor=tensor,
                    prep_ms=prep_ms, prep_launches=nprep, dominant=dominant,
                    other_ms=(by[1] if tensor else by[2])[0], other_flops=(by[1] if tensor else by[2])[1])


GEMM_TIMER = _GemmTimer()


def _mat(t: torch.Tensor) -> Tuple[torch.Tensor, int]:
    """2-D fp32 row-major view with unit inner stride; returns (tensor_keeping_storage_alive, ld)."""
    if t.dim() == 2 and t.dtype == torch.float32 and t.is_contiguous():
        return t, t.shape[1]                     # the common case: a dense arena / parameter matrix
    if t.dim() == 1:
        t = t.unsqueeze(1)
    if t.dtype != torch.float32:
        raise TypeError(f'expected float32, got {t.dtype}')
    if t.stride(1) != 1 or (t.shape[0] > 1 and t.stride(0) < t.shape[1]):
        t = t.contiguous()
    ld = t.stride(0) if t.shape[0] > 1 else max(t.shape[1], t.stride(0))
    return t, ld


# ----------------------------------------------------------------------------------------------------
# raw ops (each = one C-ABI entry point)
# ----------------------------------------------------------------------------------------------------
USE_WGMMA = True     # set False to keep every layer on the fp32 SIMT kernel
WEIGHT_EPOCH = 0       # bumped whenever a raw kernel rewrites parameters (GCBF.optim_step): invalidates weight companions


@dataclass
class H16:
    """fp16 [hi | lo] companion of an fp32 matrix (same row-major layout, pitch `ld` halves): x * s = hi + lo with the
    per-tensor power-of-two scale s derived from `amax` (device int32 = float bits of max|x|).  One companion serves
    every GEMM the matrix takes part in (K-major or MN-major operand, csrc/gemm_wgmma_f16.cu).  Non-zero amax strides: `amax`
    is an array of per-(128 x 256)-tile maxima instead (what the GEMM epilogues emit)."""
    buf: torch.Tensor
    amax: torch.Tensor
    rows: int
    cols: int
    ld: int
    amax_row_stride: int = 0
    amax_col_stride: int = 0

    def desc(self) -> native.H16Desc:
        """the `gcbf_h16` the tensor-core entry points take (valid while this object keeps the tensors alive)"""
        return native.H16Desc(ptr(self.buf), ptr(self.amax), self.ld, self.rows, self.cols, self.amax_row_stride, self.amax_col_stride, 0)


def use_h(M: int, N: int, K: int) -> bool:
    """Does the [M,K] x [N,K] layer (forward, data-grad and weight-grad alike) run on the wgmma 3xFP16 kernel?"""
    if not USE_WGMMA or GEMM_IMPL == 1:
        return False
    if GEMM_IMPL == 2:
        return True
    return M >= 256 and N >= 96 and K >= 96 and M * N * K >= (1 << 24)     # == gcbf_linear_h_supported (tested)


_AMAX_POOL = {'epoch': -1, 'buf': None, 'next': 0}


def amax_slot(device) -> torch.Tensor:
    """One int32 device word for a tensor's max|x| (float bits).  Inside a train step the words come from one pooled arena
    allocation (a 1-element view each) instead of ~150 separate allocations."""
    if not ARENA.active or torch.device(device) != ARENA.device:
        return torch.empty(1, device=device, dtype=torch.int32)
    p = _AMAX_POOL
    if p['epoch'] != ARENA.epoch or p['next'] >= 1024:
        p['buf'], p['epoch'], p['next'] = _empty(1024, device=device, dtype=torch.int32), ARENA.epoch, 0
    i = p['next']
    p['next'] = i + 1
    return p['buf'][i:i + 1]


def split_h(t: torch.Tensor, amax: Optional[torch.Tensor] = None, colsum: Optional[torch.Tensor] = None,
            persistent: bool = False, into: Optional[H16] = None, colsum_accumulate: bool = False) -> H16:
    """amax (unless the producer already supplied it) + fp16 [hi|lo] split; `colsum` (fp32 [cols]) optionally receives
    the column sums of t (the bias gradient when t = dZ)."""
    m, ld = _mat(t)
    rows, cols = m.shape
    ld_h = (cols + 7) // 8 * 8
    if into is not None and into.rows == rows and into.cols == cols:
        buf, own_amax = into.buf, into.amax
    else:
        alloc = torch.empty if persistent else _empty
        buf = alloc(2, rows, ld_h, device=m.device, dtype=torch.float16)
        own_amax = torch.empty(1, device=m.device, dtype=torch.int32) if persistent else amax_slot(m.device)

    def go():
        nonlocal amax
        if amax is None:
            amax = own_amax
            call('gcbf_amax_f32', ptr(m), ld, rows, cols, ptr(amax), 0)
        call('gcbf_split_f16', ptr(m), ld, rows, cols, ptr(amax), ptr(buf), ld_h, ptr(colsum), 1 if colsum_accumulate else 0)
    GEMM_TIMER.run_prep(go)
    return H16(buf, amax, rows, cols, ld_h)


def weight_h(W: torch.Tensor) -> H16:
    """Companion of a weight matrix, re-made only when the weights changed (optimizer step / in-place update).  The
    cache entry lives on the tensor object itself, so it can never outlive the weights it was made from."""
    stamp = (WEIGHT_EPOCH, W._version, W.data_ptr(), tuple(W.shape))
    ent = getattr(W, '_gcbf_h16', None)
    if ent is not None and ent[0] == stamp:
        return ent[1]
    h = split_h(W.detach(), persistent=True, into=ent[1] if ent is not None else None)
    W._gcbf_h16 = (stamp, h)
    return h


def prepare_weights(jobs) -> None:
    """Refresh the stale companions of several weight matrices in two launches (instead of a memset + amax + split each).
    `jobs`: iterable of (LinearSpec, M) -- the layers about to run with M rows; layers that do not qualify for the tensor
    core or whose companion is current are skipped.  Bit-identical to weight_h() layer by layer."""
    stale = []
    for L, M in jobs:
        W = L.W
        N, K = W.shape
        if not use_h(M, N, K):
            continue
        stamp = (WEIGHT_EPOCH, W._version, W.data_ptr(), tuple(W.shape))
        ent = getattr(W, '_gcbf_h16', None)
        if ent is not None and ent[0] == stamp:
            continue
        if any(W is w for w, _, _ in stale):
            continue
        if ent is not None and ent[1].rows == N and ent[1].cols == K:
            h = ent[1]
        else:
            ld_h = (K + 7) // 8 * 8
            h = H16(torch.empty(2, N, ld_h, device=W.device, dtype=torch.float16),
                    torch.empty(1, device=W.device, dtype=torch.int32), N, K, ld_h)
        stale.append((W, stamp, h))
    if not stale:
        return
    arr = (_C.SplitDesc * len(stale))()
    keep = []
    for i, (W, _, h) in enumerate(stale):
        Wm, ldw = _mat(W.detach())
        keep.append(Wm)
        a = arr[i]
        a.src, a.ld, a.rows, a.cols, a.ld_h, a.amax_slot, a.dst = ptr(Wm), ldw, h.rows, h.cols, h.ld, ptr(h.amax), ptr(h.buf)
    GEMM_TIMER.run_prep(lambda: call('gcbf_amax_split_batched', arr, len(stale)))
    for W, stamp, h in stale:
        W._gcbf_h16 = (stamp, h)


def linear_fwd_h(xh: H16, wh: H16, b, inv_sigma, act, out=None, out_amax=None):
    M, K, N = xh.rows, xh.cols, wh.rows
    assert wh.cols == K, (M, K, wh.rows, wh.cols)
    if out is None:
        out = _empty(M, N, device=xh.buf.device, dtype=torch.float32)
    y, ldy = _mat(out)
    assert y.data_ptr() == out.data_ptr()
    GEMM_TIMER.run(2.0 * M * N * K, lambda: call('gcbf_linear_fwd_h', xh.desc(), wh.desc(), ptr(b), ptr(inv_sigma), act, ptr(y), ldy, None,
                                                 ptr(out_amax), M, N, K, tail=(3,)), impl=2, tag=('forward', M, N, K))
    return out


def linear_bwd_data_h(dzh: H16, wh: H16, inv_sigma, relu_src, out=None, accumulate=False, out_amax=None):
    M, N, K = dzh.rows, dzh.cols, wh.cols
    assert wh.rows == N
    if out is None:
        assert not accumulate
        out = _empty(M, K, device=dzh.buf.device, dtype=torch.float32)
    o, ldo = _mat(out)
    assert o.data_ptr() == out.data_ptr()
    rs, ldr = (None, 0)
    if relu_src is not None:
        rs, ldr = _mat(relu_src)
    GEMM_TIMER.run(2.0 * M * N * K, lambda: call('gcbf_linear_bwd_data_h', dzh.desc(), wh.desc(), ptr(inv_sigma), ptr(rs), ldr, None, ptr(o), ldo,
                                                 1 if accumulate else 0, None, None, ptr(out_amax), M, N, K, tail=(3,)), impl=2,
                   tag=('data-grad', M, N, K))
    return out


def linear_bwd_weight_h(dzh: H16, xh: H16, inv_sigma, out=None, accumulate=False):
    M, N, K = dzh.rows, dzh.cols, xh.cols
    assert xh.rows == M
    if out is None:
        assert not accumulate
        out = _empty(N, K, device=dzh.buf.device, dtype=torch.float32)
    o, ldo = _mat(out)
    assert o.data_ptr() == out.data_ptr() and tuple(o.shape) == (N, K)
    GEMM_TIMER.run(2.0 * M * N * K, lambda: call('gcbf_linear_bwd_weight_h', dzh.desc(), xh.desc(), ptr(inv_sigma), ptr(o), ldo,
                                                 1 if accumulate else 0, M, N, K, tail=(3,)), impl=2, tag=('weight-grad', M, N, K))
    return out


def linear_fwd(x, W, b, inv_sigma, act, out=None, out_amax=None):
    x, ldx = _mat(x)
    W, ldw = _mat(W)
    M, K = x.shape
    N = W.shape[0]
    assert W.shape[1] == K, (x.shape, W.shape)
    if use_h(M, N, K):
        return linear_fwd_h(split_h(x), weight_h(W), b, inv_sigma, act, out=out, out_amax=out_amax)
    if out is None:
        out = _empty(M, N, device=x.device, dtype=torch.float32)
    y, ldy = _mat(out)
    assert y.data_ptr() == out.data_ptr()
    GEMM_TIMER.run(2.0 * M * N * K, lambda: call('gcbf_linear_fwd', ptr(x), ldx, ptr(W), ldw, ptr(b), ptr(inv_sigma), ptr(y), ldy,
                                                 M, N, K, act, GEMM_IMPL, ptr(out_amax)))
    return out


def linear_bwd_data(dz, W, inv_sigma, relu_src, out=None, accumulate=False):
    dz, lddz = _mat(dz)
    W, ldw = _mat(W)
    M, N = dz.shape
    K = W.shape[1]
    assert W.shape[0] == N
    if use_h(M, N, K):
        return linear_bwd_data_h(split_h(dz), weight_h(W), inv_sigma, relu_src, out=out, accumulate=accumulate)
    if out is None:
        assert not accumulate
        out = _empty(M, K, device=dz.device, dtype=torch.float32)
    o, ldo = _mat(out)
    assert o.data_ptr() == out.data_ptr()
    rs, ldr = (None, 0)
    if relu_src is not None:
        rs, ldr = _mat(relu_src)
    GEMM_TIMER.run(2.0 * M * N * K, lambda: call('gcbf_linear_bwd_data', ptr(dz), lddz, ptr(W), ldw, ptr(inv_sigma), ptr(rs), ldr,
                                                 ptr(o), ldo, M, N, K, 1 if accumulate else 0, GEMM_IMPL))
    return out


def linear_bwd_weight(dz, x, inv_sigma, need_bias=True, out_w=None, out_b=None):
    """dW, db of one layer.  `out_w` / `out_b`: accumulate INTO these tensors (e.g. the parameters' .grad views) instead of
    returning fresh ones."""
    dz, lddz = _mat(dz)
    x, ldx = _mat(x)
    M, N = dz.shape
    K = x.shape[1]
    if use_h(M, N, K):
        db = out_b if out_b is not None else (_empty(N, device=dz.device, dtype=torch.float32) if need_bias else None)
        dzh = split_h(dz, colsum=db, colsum_accumulate=out_b is not None)
        return linear_bwd_weight_h(dzh, split_h(x), inv_sigma, out=out_w, accumulate=out_w is not None), db
    assert (out_w is None) == (out_b is None) or not need_bias
    acc = out_w is not None
    dW = out_w if acc else _empty(N, K, device=dz.device, dtype=torch.float32)
    db = (out_b if acc else _empty(N, device=dz.device, dtype=torch.float32)) if need_bias else None
    dWm, lddw = _mat(dW)
    assert dWm.data_ptr() == dW.data_ptr()
    GEMM_TIMER.run(2.0 * M * N * K, lambda: call('gcbf_linear_bwd_weight', ptr(dz), lddz, ptr(x), ldx, ptr(inv_sigma), ptr(dW), lddw,
                                                 ptr(db), M, N, K, 1 if acc else 0, GEMM_IMPL))
    return dW, db


def act_bwd(dy, y, act):
    dy = dy.contiguous()
    y = y.contiguous()
    out = _empty(dy.shape, device=dy.device, dtype=dy.dtype)
    call('gcbf_act_bwd', ptr(dy), ptr(y), ptr(out), dy.numel(), act)
    return out


_SN_WS = {}


def _sn_workspace(device, N, K):
    need = int(_C.lib().gcbf_sn_workspace_floats(N, K))
    ws = _SN_WS.get(device)
    if ws is None or ws.numel() < need:
        ws = torch.empty(max(need, 1 << 16), device=device, dtype=torch.float32)
        _SN_WS[device] = ws
    return ws


def sn_power_iter(W, u, v):
    """In-place power iteration on the module buffers u, v; returns the device scalar 1/sigma."""
    Wm, ldw = _mat(W)
    N, K = Wm.shape
    inv_sigma = torch.empty(1, device=W.device, dtype=torch.float32)
    call('gcbf_sn_power_iter', ptr(Wm), ldw, N, K, ptr(u), ptr(v), ptr(inv_sigma), ptr(_sn_workspace(W.device, N, K)))
    return inv_sigma


_SN_ORDER = {}     # id(first u buffer of a net) -> CUDA event recorded after the net's latest power iteration (+ u/v snapshots)


def sn_power_iter_batched(layers, snapshot: bool = False):
    """One power iteration on every spectral-normalised LinearSpec of `layers` in four launches (instead of four per
    layer).  Returns (inv_sigmas, uvs): per-layer 1/sigma device scalars (None for layers without spectral norm) and, with
    `snapshot`, per-layer (u, v) copies taken right after the iteration (the backward's sigma-gradient needs the vectors of
    ITS forward).  The iterations of one net are chained through a CUDA event, so forwards of the same net issued on
    different streams still advance u, v in program order (and never overwrite them under a snapshot in flight)."""
    sn = [L for L in layers if L.sn]
    if not sn:
        return [None] * len(layers), [None] * len(layers)
    dev = sn[0].W.device
    key = id(sn[0].u)
    prev = _SN_ORDER.get(key)
    if prev is not None:
        torch.cuda.current_stream(dev).wait_event(prev)
    inv = torch.empty(len(sn), device=dev, dtype=torch.float32)
    arr = (_C.SnLayer * len(sn))()
    need = 0
    keep = []
    for i, L in enumerate(sn):
        Wm, ldw = _mat(L.W)
        keep.append(Wm)
        N, K = Wm.shape
        a = arr[i]
        a.W, a.ldw, a.N, a.K, a.u, a.v, a.inv_sigma = ptr(Wm), ldw, N, K, ptr(L.u), ptr(L.v), inv.data_ptr() + 4 * i
        need += int(_C.lib().gcbf_sn_workspace_floats(N, K))
    stream_key = (dev, 'batched', _C.stream())          # one workspace per stream: two forwards may be in flight
    ws = _SN_WS.get(stream_key)
    if ws is None or ws.numel() < need:
        ws = _SN_WS[stream_key] = torch.empty(max(need, 1 << 18), device=dev, dtype=torch.float32)
    call('gcbf_sn_power_iter_batched', arr, len(sn), ptr(ws), ws.numel())
    snaps = [(L.u.clone(), L.v.clone()) for L in sn] if snapshot else [None] * len(sn)
    ev = torch.cuda.Event()
    ev.record()
    _SN_ORDER[key] = ev
    out, uvs, i = [], [], 0
    for L in layers:
        if L.sn:
            out.append(inv[i:i + 1])
            uvs.append(snaps[i])
            i += 1
        else:
            out.append(None)
            uvs.append(None)
    return out, uvs


def sn_grad_fixup(dW, W, u, v, inv_sigma, acc=None):
    """Gradient through sigma of the spectral norm.  acc=None: dW corrected in place; else the corrected gradient is added
    to `acc` (the parameter's .grad view)."""
    Wm, ldw = _mat(W)
    N, K = Wm.shape
    am, lda = (None, 0)
    if acc is not None:
        am, lda = _mat(acc)
        assert am.data_ptr() == acc.data_ptr()
    call('gcbf_sn_grad_fixup', ptr(dW), K, ptr(Wm), ldw, N, K, ptr(u), ptr(v), ptr(inv_sigma),
         ptr(_sn_workspace(W.device, N, K)), ptr(am), lda)
    return dW


def copy2d(src, dst, rows, cols):
    s, lds = _mat(src)
    d, ldd = _mat(dst)
    assert d.data_ptr() == dst.data_ptr()
    call('gcbf_copy2d', ptr(s), lds, ptr(d), ldd, rows, cols)


def rows_gather(src, idx, out):
    s, lds = _mat(src)
    o, ldo = _mat(out)
    assert o.data_ptr() == out.data_ptr()
    call('gcbf_rows_gather', ptr(s), lds, ptr(idx), ptr(o), ldo, idx.numel(), out.shape[1])
    return out


def rows_scatter(src, idx, out):
    s, lds = _mat(src)
    o, ldo = _mat(out)
    assert o.data_ptr() == out.data_ptr()
    call('gcbf_rows_scatter', ptr(s), lds, ptr(idx), ptr(o), ldo, idx.numel(), src.shape[1])
    return out


def rowptr_from_edge_index(edge_index: torch.Tensor, num_nodes: int, check_sorted: bool = True) -> torch.Tensor:
    """CSR row pointer (int32, num_nodes+1) over target nodes of a target-sorted edge_index."""
    _C.require_cuda(edge_index)
    ei = edge_index.contiguous()
    E = ei.shape[1]
    rowptr = torch.empty(num_nodes + 1, device=ei.device, dtype=torch.int32)
    flag = torch.empty(1, device=ei.device, dtype=torch.int32)
    dst = ei[1]
    call('gcbf_rowptr_from_targets', dst.data_ptr() if E else None, E, num_nodes, ptr(rowptr), ptr(flag))
    if check_sorted and int(flag.item()) != 0:
        raise ValueError('edge_index[1] (targets) must be in range and sorted ascending: every reference call site '
                         '(RadiusGraph / nonzero / Batch.from_data_list) produces target-sorted edges')
    return rowptr


def radius_graph(states: torch.Tensor, pos_dim: int, num_graphs: int, nodes_per_graph: int, num_agents: int,
                 radius: float, metric: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """K1: returns (edge_index int64 [2,E] sorted (target, source), rowptr int32 over agents)."""
    _C.require_cuda(states)
    st, ld = _mat(states)
    na = num_graphs * num_agents
    rowptr = torch.empty(na + 1, device=st.device, dtype=torch.int32)
    call('gcbf_radius_graph_count', ptr(st), ld, pos_dim, num_graphs, nodes_per_graph, num_agents, float(radius),
         metric, ptr(rowptr))
    E = int(rowptr[-1].item())          # the one host sync: output size is data dependent
    ei = torch.empty(2, E, device=st.device, dtype=torch.int64)
    call('gcbf_radius_graph_fill', ptr(st), ld, pos_dim, num_graphs, nodes_per_graph, num_agents, float(radius),
         metric, ptr(rowptr), ptr(ei) if E else None, E)
    return ei, rowptr


def radius_graph_topk(states: torch.Tensor, pos_dim: int, num_graphs: int, nodes_per_graph: int, num_agents: int,
                      radius: float, metric: int, max_neighbors: int) -> Tuple[torch.Tensor, torch.Tensor]:
    """K1 with the top-k neighbour filter of an env built with `max_neighbors` (MACBF; reference dubins_car.py:736-740,
    simple_drone.py:322-326, simple_car.py:32-33): same protocol and output order as radius_graph."""
    _C.require_cuda(states)
    st, ld = _mat(states)
    na = num_graphs * num_agents
    rowptr = torch.empty(na + 1, device=st.device, dtype=torch.int32)
    call('gcbf_radius_graph_topk_count', ptr(st), ld, pos_dim, num_graphs, nodes_per_graph, num_agents, float(radius), metric,
         int(max_neighbors), ptr(rowptr))
    E = int(rowptr[-1].item())
    ei = torch.empty(2, E, device=st.device, dtype=torch.int64)
    call('gcbf_radius_graph_topk_fill', ptr(st), ld, pos_dim, num_graphs, nodes_per_graph, num_agents, float(radius), metric,
         int(max_neighbors), ptr(rowptr), ptr(ei) if E else None, E)
    return ei, rowptr


def edge_masks(edge_attr: torch.Tensor, pos_dim: int, agent_radius: float) -> torch.Tensor:
    """(safe, unsafe) per EDGE as a [2, E] bool tensor: env.safe_mask / unsafe_mask(data, return_edge=True)."""
    _C.require_cuda(edge_attr)
    ea, ld = _mat(edge_attr.detach())
    E = int(ea.shape[0])
    out = torch.empty(2, E, device=ea.device, dtype=torch.uint8)
    call('gcbf_edge_masks', ptr(ea) if E else None, ld, pos_dim, E, float(agent_radius), ptr(out[0]) if E else None,
         ptr(out[1]) if E else None)
    return out.view(torch.bool)


class EdgeInputFunction(torch.autograd.Function):
    """cat[x_i, x_j, e_ij] per edge (the `message` input of every layer in gcbf/nn/gnn.py); x is the node-type indicator and
    carries no gradient, d edge_attr is the last `edge_dim` columns of the incoming gradient."""

    @staticmethod
    def forward(ctx, x, edge_attr, edge_index):
        _C.require_cuda(x, edge_attr, edge_index)
        xc, ea, ei = x.detach().contiguous(), edge_attr.detach().contiguous(), edge_index.contiguous()
        E, nd, ed = int(ei.shape[1]), int(xc.shape[1]), int(ea.shape[1])
        out = torch.empty(E, 2 * nd + ed, device=xc.device, dtype=torch.float32)
        call('gcbf_edge_input_fwd', ptr(xc), nd, ptr(ea) if E else None, ed, ptr(ei) if E else None, E, ptr(out) if E else None,
             2 * nd + ed)
        ctx.dims = (nd, ed)
        return out

    @staticmethod
    def backward(ctx, d_out):
        nd, ed = ctx.dims
        d_ea = None
        if ctx.needs_input_grad[1]:
            E = int(d_out.shape[0])
            d_ea = torch.empty(E, ed, device=d_out.device, dtype=torch.float32)
            if E:
                copy2d(d_out[:, 2 * nd:], d_ea, E, ed)
        return None, d_ea, None


class SegMaxFunction(torch.autograd.Function):
    """MessagePassing(aggr='max') (gcbf/nn/gnn.py:116-119): per-target maximum of the incoming messages over the CSR of the
    target-sorted edge list, 0 for nodes without incoming edges; the gradient goes to the arg-max edge of every (node, channel)."""

    @staticmethod
    def forward(ctx, msg, rowptr, num_nodes):
        _C.require_cuda(msg, rowptr)
        m, ld = _mat(msg.detach())
        E, C = int(m.shape[0]), int(m.shape[1])
        out = torch.empty(num_nodes, C, device=m.device, dtype=torch.float32)
        arg = torch.empty(num_nodes, C, device=m.device, dtype=torch.int32)
        call('gcbf_seg_max_fwd', ptr(m) if E else None, ld, ptr(rowptr), num_nodes, C, ptr(out), C, ptr(arg))
        ctx.save_for_backward(arg)
        ctx.dims = (E, C, num_nodes)
        return out

    @staticmethod
    def backward(ctx, d_out):
        (arg,) = ctx.saved_tensors
        E, C, num_nodes = ctx.dims
        d, ld = _mat(d_out)
        d_msg = torch.empty(E, C, device=d_out.device, dtype=torch.float32)
        call('gcbf_seg_max_bwd', ptr(d), ld, ptr(arg), num_nodes, C, ptr(d_msg) if E else None, C, E)
        return d_msg, None, None


class GatherCatFunction(torch.autograd.Function):
    """cat([feat[agent_mask], extra], dim=1) (gcbf/controller/macbf_controller.py:44-46): row gather (identity when row_index is
    None) + column concatenation in one output buffer; backward scatters the feature columns back to the selected rows."""

    @staticmethod
    def forward(ctx, feat, row_index, extra):
        _C.require_cuda(feat, extra)
        f = feat.detach()
        R = int(row_index.numel()) if row_index is not None else int(f.shape[0])
        F, X = int(f.shape[1]), int(extra.shape[1])
        out = torch.empty(R, F + X, device=f.device, dtype=torch.float32)
        if R:
            if row_index is not None:
                rows_gather(f, row_index, out[:, :F])
            else:
                copy2d(f, out[:, :F], R, F)
            copy2d(extra.detach().contiguous(), out[:, F:], R, X)
        ctx.dims = (int(f.shape[0]), F)
        ctx.row_index = row_index
        return out

    @staticmethod
    def backward(ctx, d_out):
        Nn, F = ctx.dims
        if not ctx.needs_input_grad[0]:
            return None, None, None
        R = int(d_out.shape[0])
        if ctx.row_index is not None:
            d_feat = torch.zeros(Nn, F, device=d_out.device, dtype=torch.float32)
            if R:
                rows_scatter(d_out[:, :F], ctx.row_index, d_feat)
        else:
            d_feat = torch.empty(Nn, F, device=d_out.device, dtype=torch.float32)
            if R:
                copy2d(d_out[:, :F], d_feat, R, F)
        return d_feat, None, None


def edge_attr_fwd(env_id: int, states, edge_index):
    st, ld = _mat(states)
    ei = edge_index.contiguous()
    E = ei.shape[1]
    ed = {0: 4, 1: 5, 2: 6}[env_id]
    out = _empty(E, ed, device=st.device, dtype=torch.float32)
    call('gcbf_edge_attr_fwd', env_id, ptr(st), ld, ptr(ei) if E else None, E, ptr(out) if E else None)
    return out


def edge_attr_bwd(env_id: int, states, edge_index, d_edge_attr):
    st, ld = _mat(states)
    ei = edge_index.contiguous()
    E = ei.shape[1]
    d_states = _zeros(st.shape[0], ld, device=st.device, dtype=torch.float32)
    d_ea = d_edge_attr.contiguous()
    call('gcbf_edge_attr_bwd', env_id, ptr(st), ld, ptr(ei) if E else None, E, ptr(d_ea) if E else None, ptr(d_states))
    return d_states[:, :st.shape[1]]


class EdgeAttrFunction(torch.autograd.Function):
    """env.edge_attr(state, edge_index): reference simple_car.py:246-247, dubins_car.py:724-728,
    simple_drone.py:313-314."""

    @staticmethod
    def forward(ctx, states, edge_index, env_id):
        _C.require_cuda(states, edge_index)
        ctx.env_id = env_id
        ctx.save_for_backward(states, edge_index)
        return edge_attr_fwd(env_id, states, edge_index)

    @staticmethod
    def backward(ctx, d_out):
        states, edge_index = ctx.saved_tensors
        return edge_attr_bwd(ctx.env_id, states, edge_index, d_out), None, None


# ----------------------------------------------------------------------------------------------------
# MLP chain
# ----------------------------------------------------------------------------------------------------
@dataclass
class LinearSpec:
    W: torch.Tensor                      # [N, K]  (weight, or weight_orig when spectral-normalised)
    b: torch.Tensor                      # [N]
    u: Optional[torch.Tensor] = None     # spectral-norm buffers (updated in place on every forward)
    v: Optional[torch.Tensor] = None
    act: int = ACT_NONE

    @property
    def sn(self) -> bool:
        return self.u is not None


@dataclass
class MLPCtx:
    acts: List[torch.Tensor] = field(default_factory=list)      # acts[0] = input, acts[l] = output of layer l
    inv_sigma: List[Optional[torch.Tensor]] = field(default_factory=list)
    uv: List[Optional[Tuple[torch.Tensor, torch.Tensor]]] = field(default_factory=list)
    acts_h: List[Optional[H16]] = field(default_factory=list)  # acts_h[l] = fp16 companion of acts[l] when layer l is on the wgmma kernel
    out_amax: Optional[torch.Tensor] = None                   # amax slot of the MLP's output when the caller asked for it


def mlp_forward(x: torch.Tensor, layers: Sequence[LinearSpec], save: bool, x_amax: Optional[torch.Tensor] = None,
                next_width: int = 0, inv_sigmas: Optional[list] = None, uvs: Optional[list] = None):
    """Returns (y, ctx, y_amax).  `x_amax`: amax slot of x when its producer already reduced it.  `next_width` > 0: the
    output feeds a linear layer of that many out-features next (possibly in another MLP); if that layer runs on the tensor
    cores the last layer's epilogue reduces max|y| and the slot is returned as y_amax (else None)."""
    ctx = MLPCtx() if save else None
    if save:
        ctx.acts.append(x)
    for l, L in enumerate(layers):
        inv_sigma = None
        if L.sn:
            # old-style torch spectral_norm in training mode: one power iteration per forward, even under
            # no_grad (the reference never calls .eval(); SURVEY 3.5); batched per net by the caller when possible
            inv_sigma = inv_sigmas[l] if inv_sigmas is not None else sn_power_iter(L.W, L.u, L.v)
        M, K = x.shape
        N = L.W.shape[0]
        nxt_n = layers[l + 1].W.shape[0] if l + 1 < len(layers) else next_width
        y_amax = amax_slot(x.device) if (nxt_n > 0 and use_h(M, nxt_n, N)) else None
        xh = None
        if use_h(M, N, K):
            xh = split_h(x, amax=x_amax)
            x = linear_fwd_h(xh, weight_h(L.W), L.b, inv_sigma, L.act, out_amax=y_amax)
        else:
            x = linear_fwd(x, L.W, L.b, inv_sigma, L.act, out_amax=y_amax)
        x_amax = y_amax
        if save:
            ctx.acts.append(x)
            ctx.acts_h.append(xh)
            ctx.inv_sigma.append(inv_sigma)
            ctx.uv.append((uvs[l] if uvs is not None else (L.u.clone(), L.v.clone())) if L.sn else None)
    return x, ctx, x_amax


SKIP_WGRAD = False   # set by GCBF.apply: only input gradients are needed there, weight-gradient GEMMs are skipped
GRAD_INTO_PARAM = False   # set by GCBF.train_step: weight / bias gradients are accumulated straight into the parameters'
#                           .grad views (the flat gradient bucket) by the kernels; autograd then sees None for them


def _grad_targets(L):
    if not GRAD_INTO_PARAM:
        return None, None
    gW, gb = getattr(L.W, 'grad', None), getattr(L.b, 'grad', None)
    if gW is None or gb is None or not gW.is_contiguous() or not gb.is_contiguous():
        return None, None
    return gW, gb


def mlp_backward(ctx: MLPCtx, layers: Sequence[LinearSpec], dy: torch.Tensor, need_dx: bool,
                 dx_out: Optional[torch.Tensor] = None, dx_accumulate: bool = False, dy_amax: Optional[torch.Tensor] = None,
                 dx_amax: Optional[torch.Tensor] = None, mask_acts: Optional[List[torch.Tensor]] = None, bias_grad: bool = True,
                 dy_is_preact: bool = False):
    """Returns (dx or None, [(dW, db) per layer]).  `dy_amax`: amax slot of dy when its producer reduced it (only valid if
    the output layer has no activation).  `dx_amax`: slot that receives max|dx| when the input-gradient GEMM runs on the
    tensor cores (the caller checks `dx_amax_valid`).
    The backward of a tangent pass (gcbf_b200/jvp.py) runs this on the tangent's layer inputs (ctx.acts) with: `mask_acts` the
    PRIMAL activations the hidden ReLU masks come from, `bias_grad=False` (the tangent layers have no bias) and `dy_is_preact`
    (dy is already the gradient of the output layer's pre-activation)."""
    grads = [None] * len(layers)
    dz = dy
    last = len(layers) - 1
    if dy_is_preact:
        pass
    elif layers[last].act == ACT_TANH:
        dz = act_bwd(dz, ctx.acts[last + 1], ACT_TANH)
    elif layers[last].act == ACT_RELU:
        dz = act_bwd(dz, ctx.acts[last + 1], ACT_RELU)
    # amax of dz when the producing data-grad epilogue already reduced it
    dz_amax = dy_amax if (dy_is_preact or layers[last].act == ACT_NONE) else None
    mlp_backward.dx_amax_valid = False
    for l in range(last, -1, -1):
        L = layers[l]
        x_in = ctx.acts[l]
        inv_sigma = ctx.inv_sigma[l]
        M, N = dz.shape
        K = x_in.shape[1]
        if use_h(M, N, K):
            # one fp16 companion of dz serves the weight-grad (MN-major A) and the data-grad (K-major A); the bias
            # gradient (column sums of dz) is fused into the split
            gW, gb = (None, None) if SKIP_WGRAD else _grad_targets(L)
            if not bias_grad:
                gb = None
            db = None if (SKIP_WGRAD or not bias_grad) else (gb if gb is not None else _empty(N, device=dz.device, dtype=torch.float32))
            dzh = split_h(dz, amax=dz_amax, colsum=db, colsum_accumulate=gb is not None)
            if SKIP_WGRAD:
                grads[l] = (None, None)
            else:
                xh = ctx.acts_h[l] if ctx.acts_h[l] is not None else split_h(x_in)
                if L.sn:
                    dW = linear_bwd_weight_h(dzh, xh, inv_sigma)
                    u, v = ctx.uv[l]
                    sn_grad_fixup(dW, L.W, u, v, inv_sigma, acc=gW)
                else:
                    dW = linear_bwd_weight_h(dzh, xh, inv_sigma, out=gW, accumulate=gW is not None)
                grads[l] = (None if gW is not None else dW, None if gb is not None else db)
            wh = weight_h(L.W)
            if l > 0:
                assert layers[l - 1].act == ACT_RELU
                Kp = ctx.acts[l - 1].shape[1]
                dz_amax = amax_slot(dz.device) if use_h(M, K, Kp) else None
                dz = linear_bwd_data_h(dzh, wh, inv_sigma, x_in if mask_acts is None else mask_acts[l], out_amax=dz_amax)
            elif need_dx:
                dz = linear_bwd_data_h(dzh, wh, inv_sigma, None, out=dx_out, accumulate=dx_accumulate, out_amax=dx_amax)
                mlp_backward.dx_amax_valid = dx_amax is not None
            else:
                dz = None
            continue
        dz_amax = None
        if SKIP_WGRAD:
            grads[l] = (None, None)
        else:
            gW, gb = _grad_targets(L)
            if not bias_grad:
                gb = None
            if L.sn:
                dW, db = linear_bwd_weight(dz, x_in, inv_sigma, need_bias=bias_grad)
                u, v = ctx.uv[l]
                sn_grad_fixup(dW, L.W, u, v, inv_sigma, acc=gW)
                if gb is not None:
                    gb.add_(db)
            else:
                dW, db = linear_bwd_weight(dz, x_in, inv_sigma, need_bias=bias_grad, out_w=gW, out_b=gb)
            grads[l] = (None if gW is not None else dW, None if gb is not None else db)
        if l > 0:
            # hidden ReLU of layer l-1 folded into the epilogue: dz_{l-1} = (dz_l W_l) * (y_{l-1} > 0)
            assert layers[l - 1].act == ACT_RELU
            dz = linear_bwd_data(dz, L.W, inv_sigma, x_in if mask_acts is None else mask_acts[l])
        elif need_dx:
            dz = linear_bwd_data(dz, L.W, inv_sigma, None, out=dx_out, accumulate=dx_accumulate)
        else:
            dz = None
    return dz, grads


def _flatten_specs(specs: Sequence[LinearSpec]) -> List[torch.Tensor]:
    out = []
    for s in specs:
        out += [s.W, s.b]
    return out


def _linear_array(layers, grads, views=None):
    arr = (native.LinearDesc * len(layers))()
    for l, L in enumerate(layers):
        native.fill_linear(arr[l], L, views[l] if grads == 'tensors' else grads, GEMM_IMPL == 2)
    return arr


def native_mlp_forward(x, layers, save):
    sync_gemm_impl()
    xm, ldx = _mat(x)
    M = int(xm.shape[0])
    arr = _linear_array(layers, None)
    out = torch.empty(M, layers[-1].W.shape[0], device=xm.device, dtype=torch.float32)
    nbytes = native.fn('gcbf_mlp_forward_workspace_bytes')(arr, len(layers), M, 1 if save else 0)
    ws = native.workspace(nbytes, xm.device)
    mctx = native.MlpCtx() if save else None
    rc = native.fn('gcbf_mlp_forward')(arr, len(layers), 1 if native._weights_stale(layers) else 0, ptr(xm), ldx, M, ptr(out), out.shape[1],
                                       ptr(ws), ws.numel(), ctypes.byref(mctx) if save else None, _C.stream())
    native.check(rc, 'gcbf_mlp_forward')
    native._mark_fresh(layers)
    return out, ((mctx, ws, xm, M) if save else None)


def native_mlp_backward(layers, state, dy, need_dx):
    mctx, ws, xm, M = state
    sync_gemm_impl()
    views = None
    if SKIP_WGRAD:
        arr = _linear_array(layers, None)
    elif GRAD_INTO_PARAM:
        arr = _linear_array(layers, 'param')
    else:
        views = _grad_views(layers, dy.device)
        arr = _linear_array(layers, 'tensors', views)
    dym, lddy = _mat(dy)
    dx = torch.empty(M, layers[0].W.shape[1], device=dy.device, dtype=torch.float32) if need_dx else None
    nbytes = native.fn('gcbf_mlp_backward_workspace_bytes')(arr, len(layers), M)
    ws2 = native.workspace(nbytes, dy.device)
    rc = native.fn('gcbf_mlp_backward')(arr, len(layers), ctypes.byref(mctx), ptr(dym), lddy, ptr(dx), 1 if SKIP_WGRAD else 0, ptr(ws2),
                                        ws2.numel(), _C.stream())
    native.check(rc, 'gcbf_mlp_backward')
    return dx, (views if views is not None else [(None, None)] * len(layers))


class MLPFunction(torch.autograd.Function):
    """gcbf.nn.MLP.forward.  apply(x, layers, *flat_params) where flat_params = [W0, b0, W1, b1, ...]."""

    @staticmethod
    def forward(ctx, x, layers, *params):
        _C.require_cuda(x)
        need = any(ctx.needs_input_grad)      # (grad mode is always off inside Function.forward)
        ctx.layers = layers
        ctx.need_dx = ctx.needs_input_grad[0]
        if NATIVE and len(layers) <= native.MAX_LAYERS:
            y, ctx.mctx = native_mlp_forward(x.detach(), layers, need)
            ctx.native = True
            return y
        ctx.native = False
        y, mctx, _ = mlp_forward(x.detach(), layers, need)
        ctx.mctx = mctx
        return y

    @staticmethod
    def backward(ctx, dy):
        if ctx.native:
            dx, grads = native_mlp_backward(ctx.layers, ctx.mctx, dy, ctx.need_dx)
        else:
            dx, grads = mlp_backward(ctx.mctx, ctx.layers, dy, ctx.need_dx)
        flat = []
        for dW, db in grads:
            flat += [dW, db]
        return (dx, None, *flat)


# ----------------------------------------------------------------------------------------------------
# GNN layer (+ optional fused head)
# ----------------------------------------------------------------------------------------------------
# GCBF.params['matmul'] -> fp16 products per k-slice of the wgmma GEMM (gcbf_net_desc.tc_products): 'fp32' = 3xFP16 (fp32-grade, the
# default), 'fp16' = one fp16 product (about 2^-10 relative per product, up to three times the tensor rate)
MATMUL_PRODUCTS = {'fp32': 3, 'fp16': 1}


@dataclass
class NetSpec:
    phi: List[LinearSpec]
    gate: List[LinearSpec]
    gamma: List[LinearSpec]
    head: Optional[List[LinearSpec]] = None
    node_dim: int = 4
    edge_dim: int = 4
    phi_dim: int = 256
    tc_products: int = 3        # fp16 products per k-slice of the tensor-core layers (MATMUL_PRODUCTS); library-sequenced passes only

    def all_layers(self):
        return self.phi + self.gate + self.gamma + (self.head or [])


def net_forward(spec: NetSpec, x, edge_attr, edge_index, rowptr, row_index, head_extra, save, sigma=None):
    """phi -> attention aggregation -> gamma (on `row_index` rows only when given) -> head.
    Returns (out, ctx-tuple).  sigma: (inv_sigmas, uvs) of an earlier sn_power_iter_batched(spec.all_layers()) to use instead of a
    new power iteration (passes that share one spectral-norm step, e.g. the chunks of one field call)."""
    if spec.tc_products != 3:
        raise ValueError("the fp16 matmul mode runs in the library-sequenced passes only (GCBF_NATIVE=1); this pass is "
                         "sequenced in Python at 3xFP16")
    dev = x.device
    E = edge_index.shape[1]
    Nn = x.shape[0]
    kin = 2 * spec.node_dim + spec.edge_dim
    ei = edge_index.contiguous()
    xc = x.contiguous()
    ea = edge_attr.contiguous()
    ein = _empty(E, kin, device=dev, dtype=torch.float32)
    call('gcbf_edge_input_fwd', ptr(xc), spec.node_dim, ptr(ea) if E else None, spec.edge_dim, ptr(ei) if E else None,
         E, ptr(ein) if E else None, kin)
    # the power iterations depend on the weights only: all spectral-normalised layers of the net in one batched call
    n_phi, n_gate, n_gamma = len(spec.phi), len(spec.gate), len(spec.gamma)
    isg, uvs = sn_power_iter_batched(spec.all_layers(), snapshot=save) if sigma is None else sigma
    R = row_index.numel() if row_index is not None else Nn
    prepare_weights([(L, E) for L in spec.phi + spec.gate] + [(L, R) for L in spec.gamma + (spec.head or [])])
    isg_phi, isg_gate = isg[:n_phi], isg[n_phi:n_phi + n_gate]
    isg_gamma, isg_head = isg[n_phi + n_gate:n_phi + n_gate + n_gamma], isg[n_phi + n_gate + n_gamma:]
    uv_phi, uv_gate = uvs[:n_phi], uvs[n_phi:n_phi + n_gate]
    uv_gamma, uv_head = uvs[n_phi + n_gate:n_phi + n_gate + n_gamma], uvs[n_phi + n_gate + n_gamma:]
    msg, c_phi, msg_amax = mlp_forward(ein, spec.phi, save, next_width=spec.gate[0].W.shape[0], inv_sigmas=isg_phi, uvs=uv_phi)   # gnn.py:30-32
    gate, c_gate, _ = mlp_forward(msg, spec.gate, save, x_amax=msg_amax, inv_sigmas=isg_gate, uvs=uv_gate)  # AttentionalAggregation.gate_nn
    C = spec.phi_dim
    gin_all = _empty(Nn, C + spec.node_dim, device=dev, dtype=torch.float32)
    att = _empty(E, device=dev, dtype=torch.float32)
    call('gcbf_attn_aggr_fwd', ptr(msg) if E else None, C, ptr(gate) if E else None, ptr(rowptr), Nn, C,
         ptr(att) if E else None, ptr(gin_all), C + spec.node_dim)
    copy2d(xc, gin_all[:, C:], Nn, spec.node_dim)                        # cat([aggr_out, x])  gnn.py:35
    if row_index is not None:
        gin = _empty(row_index.numel(), C + spec.node_dim, device=dev, dtype=torch.float32)
        rows_gather(gin_all, row_index, gin)
    else:
        gin = gin_all
    chain_head = spec.head is not None and head_extra is None            # the head reads gamma's output in place
    feat, c_gamma, feat_amax = mlp_forward(gin, spec.gamma, save,
                                           next_width=spec.head[0].W.shape[0] if chain_head else 0, inv_sigmas=isg_gamma,
                                           uvs=uv_gamma)   # gnn.py:34-36
    c_head = None
    out = feat
    hin = None
    if spec.head is not None:
        if head_extra is not None:                                       # cat([x, data.u_ref])  gnn_controller.py:46
            R, F = feat.shape
            hin = _empty(R, F + head_extra.shape[1], device=dev, dtype=torch.float32)
            copy2d(feat, hin, R, F)
            copy2d(head_extra.contiguous(), hin[:, F:], R, head_extra.shape[1])
        else:
            hin = feat
        out, c_head, _ = mlp_forward(hin, spec.head, save, x_amax=feat_amax if chain_head else None, inv_sigmas=isg_head, uvs=uv_head)
    ctx = (c_phi, c_gate, c_gamma, c_head, msg, att, Nn, E) if save else None
    return out, ctx


def net_backward(spec: NetSpec, ctx, d_out, rowptr, row_index, need_d_edge_attr):
    c_phi, c_gate, c_gamma, c_head, msg, att, Nn, E = ctx
    dev = d_out.device
    C = spec.phi_dim
    g_head = []
    d_feat = d_out
    d_feat_amax = None
    if spec.head is not None:
        slot = amax_slot(dev)
        d_hin, g_head = mlp_backward(c_head, spec.head, d_out, True, dx_amax=slot)
        F = spec.gamma[-1].W.shape[0]
        d_feat = d_hin[:, :F] if d_hin.shape[1] != F else d_hin           # strided view: kernels take ld
        if mlp_backward.dx_amax_valid:       # max over all of d_hin >= max over the d_feat columns: a valid (pow2) scale bound
            d_feat_amax = slot
    d_gin, g_gamma = mlp_backward(c_gamma, spec.gamma, d_feat, True, dy_amax=d_feat_amax)
    if row_index is not None:
        d_gin_all = _zeros(Nn, C + spec.node_dim, device=dev, dtype=torch.float32)
        rows_scatter(d_gin, row_index, d_gin_all)
    else:
        d_gin_all = d_gin
    d_msg = _empty(E, C, device=dev, dtype=torch.float32)
    d_gate = _empty(E, 1, device=dev, dtype=torch.float32)
    call('gcbf_attn_aggr_bwd', ptr(msg) if E else None, C, ptr(att) if E else None, ptr(rowptr), Nn, C, ptr(d_gin_all),
         C + spec.node_dim, ptr(d_msg) if E else None, C, ptr(d_gate) if E else None, 0)
    # gate MLP backward; its input gradient is accumulated onto the aggregation's d_msg
    slot = amax_slot(dev)
    _, g_gate = mlp_backward(c_gate, spec.gate, d_gate, True, dx_out=d_msg, dx_accumulate=True, dx_amax=slot)
    d_msg_amax = slot if mlp_backward.dx_amax_valid else None            # epilogue max of the accumulated d_msg
    d_ein, g_phi = mlp_backward(c_phi, spec.phi, d_msg, need_d_edge_attr, dy_amax=d_msg_amax)
    d_edge_attr = None
    if need_d_edge_attr:
        d_edge_attr = d_ein[:, 2 * spec.node_dim:]
    return d_edge_attr, g_phi + g_gate + g_gamma + g_head


def sync_gemm_impl():
    """Tell the library which linear-layer implementation the chain-level calls may use (tests flip ops.GEMM_IMPL)."""
    native.fn('gcbf_set_gemm_impl')(1 if (not USE_WGMMA or GEMM_IMPL == 1) else (2 if GEMM_IMPL == 2 else 0))


def _grad_views(specs, device):
    """One zeroed flat buffer with (gW, gb) views per layer: where gcbf_net_backward / gcbf_mlp_backward accumulate when the
    gradients go back to autograd as tensors (outside GCBF.train_step)."""
    total = sum(L.W.numel() + L.b.numel() for L in specs)
    flat = torch.zeros(total, device=device, dtype=torch.float32)
    views, off = [], 0
    for L in specs:
        nw, nb = L.W.numel(), L.b.numel()
        views.append((flat[off:off + nw].view(L.W.shape), flat[off + nw:off + nw + nb]))
        off += nw + nb
    return views


def native_net_forward(spec, x, edge_attr, edge_index, rowptr, row_index, head_extra, save):
    """One gcbf_net_forward call.  Returns (out, state) -- state holds the library's context, the workspace it points into and
    every tensor the context references."""
    sync_gemm_impl()
    specs = spec.all_layers()
    dev = x.device
    xc, ea, ei = x.contiguous(), edge_attr.contiguous(), edge_index.contiguous()
    he = head_extra.contiguous() if head_extra is not None else None
    E, Nn = int(ei.shape[1]), int(xc.shape[0])
    R = int(row_index.numel()) if row_index is not None else Nn
    nd = native.make_net_desc(spec, he.shape[1] if he is not None else 0, None, GEMM_IMPL == 2)
    nd.refresh_weights = 1 if native._weights_stale(specs) else 0
    out_dim = (spec.head or spec.gamma)[-1].W.shape[0]
    out = torch.empty(R, out_dim, device=dev, dtype=torch.float32)
    nbytes = native.fn('gcbf_net_forward_workspace_bytes')(ctypes.byref(nd), E, Nn, R, 1 if save else 0)
    if save:
        ws = native.workspace(nbytes, dev)           # lives in the autograd state until the backward has run
    else:
        # inference (rollouts: one actor forward per env step, a different edge count every step): a fresh torch allocation per call
        # sends the caching allocator into cudaMalloc for every new size (measured: 10 ms steps with 80 ms stalls); one grow-only
        # buffer per (device, stream) instead -- calls on a stream are ordered, so the next call may overwrite it
        key = (dev.index, _C.stream())
        gb = _INFER_WS.get(key)
        if gb is None:
            gb = _INFER_WS[key] = native.GrowBuffer()
        ws = gb.get(nbytes, dev)
    nctx = native.NetCtx() if save else None
    rc = native.fn('gcbf_net_forward')(ctypes.byref(nd), ptr(xc), ptr(ea) if E else None, ptr(ei) if E else None, ptr(rowptr), E, Nn,
                                       ptr(row_index), R, ptr(he), ptr(out), out_dim, ptr(ws), ws.numel(),
                                       ctypes.byref(nctx) if save else None, _C.stream())
    native.check(rc, 'gcbf_net_forward')
    native._mark_fresh(specs)
    state = (nctx, ws, (xc, ea, ei, rowptr, row_index, he), (E, Nn, R)) if save else None
    return out, state


_INFER_WS = {}


def native_net_backward(spec, state, d_out, need_d_edge_attr):
    nctx, ws, keep, (E, Nn, R) = state
    sync_gemm_impl()
    specs = spec.all_layers()
    dev = d_out.device
    he = keep[5]
    views = None
    if SKIP_WGRAD:
        nd = native.make_net_desc(spec, he.shape[1] if he is not None else 0, None, GEMM_IMPL == 2)
    elif GRAD_INTO_PARAM:
        nd = native.make_net_desc(spec, he.shape[1] if he is not None else 0, 'param', GEMM_IMPL == 2)
    else:
        views = _grad_views(specs, dev)
        nd = native.make_net_desc(spec, he.shape[1] if he is not None else 0, 'tensors', GEMM_IMPL == 2, grad_tensors=views)
    d_out = d_out if d_out.stride(-1) == 1 else d_out.contiguous()
    d_ea = torch.empty(E, spec.edge_dim, device=dev, dtype=torch.float32) if need_d_edge_attr else None
    nbytes = native.fn('gcbf_net_backward_workspace_bytes')(ctypes.byref(nd), E, Nn, R, 1 if need_d_edge_attr else 0)
    ws2 = native.workspace(nbytes, dev)
    rc = native.fn('gcbf_net_backward')(ctypes.byref(nd), ctypes.byref(nctx), ptr(d_out), d_out.stride(0) if d_out.dim() == 2 else 1,
                                        ptr(d_ea), 1 if SKIP_WGRAD else 0, ptr(ws2), ws2.numel(), _C.stream())
    native.check(rc, 'gcbf_net_backward')
    if views is None:
        return d_ea, [(None, None)] * len(specs)
    return d_ea, views


class GNNNetFunction(torch.autograd.Function):
    """apply(x, edge_attr, edge_index, rowptr, row_index, head_extra, spec, *flat_params)."""

    @staticmethod
    def forward(ctx, x, edge_attr, edge_index, rowptr, row_index, head_extra, spec, *params):
        _C.require_cuda(x, edge_attr, edge_index)
        if x.requires_grad:
            raise NotImplementedError('gradient w.r.t. node features x is not part of the reference hot path '
                                      '(x is a constant type indicator, simple_car.py:132)')
        need = any(ctx.needs_input_grad)      # (grad mode is always off inside Function.forward)
        he = head_extra.detach() if head_extra is not None else None
        fwd = native_net_forward if NATIVE else net_forward
        out, nctx = fwd(spec, x.detach(), edge_attr.detach(), edge_index, rowptr, row_index, he, need)
        ctx.spec, ctx.nctx = spec, nctx
        ctx.rowptr, ctx.row_index = rowptr, row_index
        ctx.need_dea = ctx.needs_input_grad[1]
        return out

    @staticmethod
    def backward(ctx, d_out):
        if NATIVE:
            d_ea, grads = native_net_backward(ctx.spec, ctx.nctx, d_out, ctx.need_dea)
        else:
            d_ea, grads = net_backward(ctx.spec, ctx.nctx, d_out.contiguous(), ctx.rowptr, ctx.row_index, ctx.need_dea)
        flat = []
        for dW, db in grads:
            flat += [dW, db]
        return (None, d_ea, None, None, None, None, None, *flat)
