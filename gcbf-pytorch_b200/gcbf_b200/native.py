"""Binding of the chain-level C ABI (include/gcbf_b200.h, "ABI v3"): one ctypes call per GNN pass (`gcbf_net_forward` /
`gcbf_net_backward`), per bare MLP, and per phase of the train step (`gcbf_step_forward` / `_relink` / `_backward`).

The kernel sequencing the reference does with ~250 ATen calls per forward (gcbf/nn/gnn.py:27-36, gcbf/nn/mlp.py:44-47,
gcbf/algo/gcbf.py:158-226) lives in the library (csrc/net.cu, csrc/step.cu); Python only describes the networks (pointers to
the nn.Parameters, their .grad views and their persistent fp16 weight companions) and owns the memory: torch tensors serve as
the workspaces the library bump-allocates in.  No arithmetic happens here.
"""
import ctypes
from ctypes import POINTER, c_double, c_float, c_int, c_int32, c_int64, c_longlong, c_size_t, c_uint64, c_void_p
from typing import List, Optional, Sequence

import torch

from . import _C

P = c_void_p
MAX_LAYERS = 4
E_WORKSPACE = -4


class LinearDesc(ctypes.Structure):
    """mirror of `gcbf_linear_desc`"""
    _fields_ = [('W', P), ('b', P), ('u', P), ('v', P), ('gW', P), ('gb', P), ('Wh', P), ('w_amax', P),
                ('ldw', c_int32), ('ldgw', c_int32), ('ldwh', c_int32), ('N', c_int32), ('K', c_int32), ('act', c_int32)]


class NetDesc(ctypes.Structure):
    """mirror of `gcbf_net_desc`"""
    _fields_ = [('phi', LinearDesc * MAX_LAYERS), ('gate', LinearDesc * MAX_LAYERS), ('gamma', LinearDesc * MAX_LAYERS),
                ('head', LinearDesc * MAX_LAYERS), ('n_phi', c_int32), ('n_gate', c_int32), ('n_gamma', c_int32), ('n_head', c_int32),
                ('node_dim', c_int32), ('edge_dim', c_int32), ('phi_dim', c_int32), ('head_extra_dim', c_int32),
                ('refresh_weights', c_int32), ('tc_products', c_int32)]


class NetCtx(ctypes.Structure):
    _fields_ = [('opaque', c_uint64 * 208)]


class MlpCtx(ctypes.Structure):
    _fields_ = [('opaque', c_uint64 * 64)]


class StepDesc(ctypes.Structure):
    """mirror of `gcbf_step_desc`"""
    _fields_ = [('cbf', NetDesc), ('actor', NetDesc), ('env', _C.EnvCfg), ('goal', P), ('lqr_gain', P),
                ('ld_goal', c_int32), ('state_dim', c_int32), ('pos_dim', c_int32), ('action_dim', c_int32),
                ('graph_metric', c_int32), ('comm_radius', c_float),
                ('alpha', c_float), ('eps', c_float), ('coef_unsafe', c_float), ('coef_safe', c_float), ('coef_hdot', c_float),
                ('coef_action', c_float), ('grad_bucket', P), ('grad_bucket_floats', c_int64), ('goal_per_graph', c_int32), ('pad_', c_int32)]


class StepBatch(ctypes.Structure):
    """mirror of `gcbf_step_batch`"""
    _fields_ = [('states', P), ('ld_state', c_int32), ('x', P), ('edge_attr', P), ('edge_index', P), ('rowptr', P), ('u_ref', P),
                ('row_index', P), ('num_edges', c_int64), ('num_nodes', c_int32), ('num_agents_total', c_int32)]


class StepOut(ctypes.Structure):
    """mirror of `gcbf_step_out`"""
    _fields_ = [('h', P), ('actions', P), ('h_next', P), ('h_next_new', P), ('hdot', P), ('scalars', P), ('safe', P), ('unsafe', P),
                ('partial', P), ('edge_index_new', P), ('num_edges_new', c_int64)]


class StepCtx(ctypes.Structure):
    _fields_ = [('opaque', c_uint64 * 800)]


class H16Desc(ctypes.Structure):
    """mirror of `gcbf_h16`: fp16 [hi|lo] companion with a per-tensor (strides 0) or per-(128 x 256)-tile scale"""
    _fields_ = [('buf', P), ('amax', P), ('ld', c_int32), ('rows', c_int32), ('cols', c_int32), ('amax_row_stride', c_int32),
                ('amax_col_stride', c_int32), ('pad_', c_int32)]


class FieldDesc(ctypes.Structure):
    """mirror of `gcbf_field_desc`"""
    _fields_ = [('cbf', NetDesc), ('env', _C.EnvCfg), ('states', P), ('x', P), ('edge_index', P), ('rowptr', P), ('num_edges', c_int64),
                ('agents', P), ('xs', P), ('ys', P), ('max_edges', c_int64), ('ld_state', c_int32), ('state_dim', c_int32),
                ('pos_dim', c_int32), ('graph_metric', c_int32), ('comm_radius', c_float), ('relink', c_int32),
                ('num_probe_agents', c_int32), ('x_dim', c_int32), ('y_dim', c_int32), ('nx', c_int32), ('ny', c_int32),
                ('max_probes', c_int32)]


class TimeRec(ctypes.Structure):
    """mirror of `gcbf_time_rec`"""
    _fields_ = [('ms', c_double), ('flops', c_double), ('kind', c_int32), ('M', c_int32), ('N', c_int32), ('K', c_int32)]


SIGS = {
    'gcbf_net_forward_workspace_bytes': (c_size_t, [POINTER(NetDesc), c_int64, c_int, c_int, c_int]),
    'gcbf_net_backward_workspace_bytes': (c_size_t, [POINTER(NetDesc), c_int64, c_int, c_int, c_int]),
    'gcbf_net_forward': (c_int, [POINTER(NetDesc), P, P, P, P, c_int64, c_int, P, c_int, P, P, c_int, P, c_size_t, POINTER(NetCtx), P]),
    'gcbf_net_backward': (c_int, [POINTER(NetDesc), POINTER(NetCtx), P, c_int, P, c_int, P, c_size_t, P]),
    'gcbf_mlp_forward_workspace_bytes': (c_size_t, [POINTER(LinearDesc), c_int, c_int, c_int]),
    'gcbf_mlp_backward_workspace_bytes': (c_size_t, [POINTER(LinearDesc), c_int, c_int]),
    'gcbf_mlp_forward': (c_int, [POINTER(LinearDesc), c_int, c_int, P, c_int, c_int, P, c_int, P, c_size_t, POINTER(MlpCtx), P]),
    'gcbf_mlp_backward': (c_int, [POINTER(LinearDesc), c_int, POINTER(MlpCtx), P, c_int, P, c_int, P, c_size_t, P]),
    'gcbf_step_workspace_bytes': (c_size_t, [POINTER(StepDesc), POINTER(StepBatch)]),
    'gcbf_step_relink_workspace_bytes': (c_size_t, [POINTER(StepDesc), POINTER(StepBatch), c_int64]),
    'gcbf_step_forward': (c_int, [POINTER(StepDesc), POINTER(StepBatch), P, c_size_t, POINTER(StepCtx), POINTER(StepOut), P, P]),
    'gcbf_step_relink': (c_int, [POINTER(StepDesc), POINTER(StepBatch), POINTER(StepCtx), P, c_size_t, POINTER(c_size_t),
                                 POINTER(StepOut), P, P]),
    'gcbf_step_backward': (c_int, [POINTER(StepDesc), POINTER(StepBatch), POINTER(StepCtx), POINTER(StepOut), POINTER(c_void_p), P, P]),
    'gcbf_apply_workspace_bytes': (c_size_t, [POINTER(StepDesc), POINTER(StepBatch)]),
    'gcbf_apply': (c_int, [POINTER(StepDesc), POINTER(StepBatch), c_float, c_float, P, c_int, P, c_int, POINTER(c_int), P, c_size_t, P]),
    'gcbf_apply_batch_workspace_bytes': (c_size_t, [POINTER(StepDesc), POINTER(StepBatch)]),
    'gcbf_apply_batch': (c_int, [POINTER(StepDesc), POINTER(StepBatch), c_float, c_float, P, c_int, P, c_int, P, POINTER(c_int), P, c_size_t,
                                 P]),
    'gcbf_cbf_field_workspace_bytes': (c_size_t, [POINTER(FieldDesc)]),
    'gcbf_cbf_field': (c_int, [POINTER(FieldDesc), P, POINTER(c_int64), P, c_size_t, P]),
    'gcbf_cbf_field_probe_count': (c_int, [POINTER(FieldDesc), P, P]),
    'gcbf_cbf_field_probe_fill': (c_int, [POINTER(FieldDesc), P, P, c_int64, P, P]),
    'gcbf_cbf_condition_probe_count': (c_int, [POINTER(FieldDesc), P, P]),
    'gcbf_cbf_condition_probe_fill': (c_int, [POINTER(FieldDesc), P, c_int, c_int, c_int, c_int64, c_int, P, c_int64, P, P, P, P, P, c_int64,
                                              P, P]),
    'gcbf_linear_fwd_h': (c_int, [POINTER(H16Desc), POINTER(H16Desc), P, P, c_int, P, c_int, POINTER(H16Desc), P, c_int, c_int, c_int, P, c_int]),
    'gcbf_linear_bwd_data_h': (c_int, [POINTER(H16Desc), POINTER(H16Desc), P, P, c_int, POINTER(H16Desc), P, c_int, c_int, POINTER(H16Desc), P, P,
                                       c_int, c_int, c_int, P, c_int]),
    'gcbf_linear_bwd_weight_h': (c_int, [POINTER(H16Desc), POINTER(H16Desc), P, P, c_int, c_int, c_int, c_int, c_int, P, c_int]),
    'gcbf_linear_fwd_emit': (c_int, [P, c_int, P, c_int, P, P, c_int, POINTER(H16Desc), c_int, c_int, c_int, P]),
    'gcbf_launch_count': (c_longlong, [c_int]),
    'gcbf_tc_launch_count': (c_longlong, [c_int, c_int]),
    'gcbf_timing_enable': (c_int, [c_int]),
    'gcbf_timing_collect': (c_int, [POINTER(TimeRec), c_int, POINTER(c_int)]),
    'gcbf_set_gemm_impl': (c_int, [c_int]),
}
_C.register(SIGS)


def fn(name):
    return getattr(_C.lib(), name)


def check(rc: int, what: str):
    if rc != 0:
        _C.check(rc, what)


# ---- weight companions ---------------------------------------------------------------------------------------------------------
WEIGHT_EPOCH = 0          # bumped whenever a raw kernel rewrites parameters behind torch's back (GCBF.optim_step)


def _companion(W: torch.Tensor):
    """Persistent fp16 [hi|lo] companion buffer + amax word of a weight matrix, kept on the tensor object (so it can never
    outlive the weights).  Only matrices a tensor-core layer can use get one (both dims >= 96, gcbf_linear_h_supported)."""
    ent = getattr(W, '_gcbf_wh', None)
    N, K = W.shape
    if ent is None or ent[0].device != W.device:
        ld_h = (K + 7) // 8 * 8
        ent = (torch.empty(2, N, ld_h, device=W.device, dtype=torch.float16), torch.zeros(1, device=W.device, dtype=torch.int32), ld_h)
        W._gcbf_wh = ent
    return ent


def _weights_stale(specs) -> bool:
    stale = False
    for L in specs:
        W = L.W
        stamp = (WEIGHT_EPOCH, W._version, W.data_ptr())
        if getattr(W, '_gcbf_wh_stamp', None) != stamp:
            stale = True
    return stale


def _mark_fresh(specs):
    for L in specs:
        W = L.W
        W._gcbf_wh_stamp = (WEIGHT_EPOCH, W._version, W.data_ptr())


def fill_linear(d: LinearDesc, L, grads, force_h: bool):
    """L: ops.LinearSpec.  grads: None (no weight gradients), 'param' (accumulate into the parameters' .grad views) or a
    (gW, gb) pair of tensors."""
    W = L.W
    if W.dim() != 2 or W.dtype != torch.float32 or W.stride(1) != 1:
        raise TypeError('weights must be 2-D float32 with unit inner stride')
    N, K = W.shape
    d.W, d.b = W.data_ptr(), L.b.data_ptr()
    d.ldw = W.stride(0) if N > 1 else K
    d.u, d.v = (L.u.data_ptr(), L.v.data_ptr()) if L.sn else (None, None)
    d.N, d.K, d.act = N, K, L.act
    gW = gb = None
    if grads == 'param':
        gW, gb = W.grad, L.b.grad
        if gW is None or gb is None or not gW.is_contiguous():
            raise RuntimeError('parameters need dense .grad buffers for in-place gradient accumulation')
    elif grads is not None:
        gW, gb = grads
    d.gW, d.gb = (gW.data_ptr(), gb.data_ptr()) if gW is not None else (None, None)
    d.ldgw = K
    if force_h or (N >= 96 and K >= 96):
        buf, amax, ld_h = _companion(W)
        d.Wh, d.w_amax, d.ldwh = buf.data_ptr(), amax.data_ptr(), ld_h
    else:
        d.Wh, d.w_amax, d.ldwh = None, None, 0


def make_net_desc(spec, head_extra_dim: int, grads, force_h: bool = False, grad_tensors=None) -> NetDesc:
    """spec: ops.NetSpec.  grad_tensors: per-layer (gW, gb) list in all_layers() order when grads == 'tensors'."""
    nd = NetDesc()
    i = 0
    for name, layers in (('phi', spec.phi), ('gate', spec.gate), ('gamma', spec.gamma), ('head', spec.head or [])):
        if len(layers) > MAX_LAYERS:
            raise NotImplementedError(f'{name}: at most {MAX_LAYERS} linear layers per MLP')
        arr = getattr(nd, name)
        for l, L in enumerate(layers):
            g = grads
            if grads == 'tensors':
                g = grad_tensors[i]
            fill_linear(arr[l], L, g, force_h)
            i += 1
        setattr(nd, 'n_' + name, len(layers))
    nd.node_dim, nd.edge_dim, nd.phi_dim = spec.node_dim, spec.edge_dim, spec.phi_dim
    nd.head_extra_dim = head_extra_dim if spec.head else 0
    nd.tc_products = spec.tc_products
    return nd


# ---- workspaces ---------------------------------------------------------------------------------------------------------------
def workspace(nbytes: int, device) -> torch.Tensor:
    """256-byte aligned uint8 device buffer (torch's caching allocator hands out 512-byte aligned blocks)."""
    t = torch.empty(max(int(nbytes), 256), device=device, dtype=torch.uint8)
    assert t.data_ptr() % 256 == 0
    return t


class GrowBuffer:
    """Grow-only workspace: the train step's activations have a different size every step (the re-linked graph changes its edge
    count), which made torch's caching allocator fall into cudaMalloc storms; one persistent buffer per role, regrown with
    head-room when a step needs more."""

    def __init__(self):
        self.buf: Optional[torch.Tensor] = None

    def get(self, nbytes: int, device) -> torch.Tensor:
        if self.buf is None or self.buf.device != torch.device(device) or self.buf.numel() < nbytes:
            self.buf = None                    # release before regrowing
            self.buf = workspace(int(nbytes * 1.2) + (1 << 20), device)
        return self.buf


def view(ws: torch.Tensor, ptr: int, shape, dtype) -> torch.Tensor:
    """Typed view of the region of `ws` the library reported at device address `ptr`."""
    off = ptr - ws.data_ptr()
    n = 1
    for s in shape:
        n *= s
    nbytes = n * torch.empty(0, dtype=dtype).element_size()
    assert 0 <= off and off + nbytes <= ws.numel(), (off, nbytes, ws.numel())
    return ws[off:off + nbytes].view(dtype).view(shape)


def launch_count(reset: bool = False) -> int:
    return int(fn('gcbf_launch_count')(1 if reset else 0))


def tc_launch_count(products: int, reset: bool = False) -> int:
    """wgmma launches so far with `products` (3 or 1) fp16 products per k-slice."""
    return int(fn('gcbf_tc_launch_count')(products, 1 if reset else 0))
