"""CBFGNNLayer / ControllerGNNLayer (reference gcbf/nn/gnn.py:14-79) on the sm_90a kernels.

One message-passing layer:  m_ij = phi(cat[x_i, x_j, e_ij]);  a = softmax_i(gate_nn(m));  aggr_i = sum_j a_ij m_ij;
out_i = gamma(cat[aggr_i, x_i]).  Signature, attribute names (`phi`, `gamma`, `aggr_module.gate_nn`) and
state-dict keys follow the reference; torch_geometric is not needed -- the gather / segment-softmax /
scatter are CSR kernels on the target-sorted edge list every reference call site produces.
"""
import weakref
from typing import Optional

import torch
import torch.nn as nn
from torch import Tensor

from .. import _C, ops
from .mlp import MLP


class AttentionalAggregation(nn.Module):
    """Holder with torch_geometric's attribute name (`gate_nn`) so that checkpoints keep their keys."""

    def __init__(self, gate_nn: nn.Module, nn: Optional[nn.Module] = None):
        super().__init__()
        self.gate_nn = gate_nn
        if nn is not None:
            raise NotImplementedError('AttentionalAggregation(nn=...) is not used by the reference')


class GraphSequential(nn.Module):
    """Stand-in for torch_geometric.nn.Sequential('x, edge_attr, edge_index', [(layer, '... -> x')]):
    children are named module_{i} (state-dict key contract, reference gcbf/algo/gcbf.py:26-29)."""

    def __init__(self, *layers: nn.Module):
        super().__init__()
        for i, layer in enumerate(layers):
            self.add_module(f'module_{i}', layer)

    def forward(self, x: Tensor, edge_attr: Tensor, edge_index: Tensor) -> Tensor:
        for layer in self.children():
            x = layer(x, edge_attr, edge_index)
        return x


_ROWPTR_CACHE = {}


def cached_rowptr(edge_index: Tensor, num_nodes: int) -> Tensor:
    """CSR row pointer of a target-sorted edge_index, cached per edge_index tensor object."""
    key = (id(edge_index), edge_index.data_ptr(), edge_index.shape[1], edge_index._version, num_nodes)
    hit = _ROWPTR_CACHE.get(key)
    if hit is not None and hit[0]() is edge_index:
        return hit[1]
    rowptr = ops.rowptr_from_edge_index(edge_index, num_nodes)
    if len(_ROWPTR_CACHE) > 64:
        _ROWPTR_CACHE.clear()
    _ROWPTR_CACHE[key] = (weakref.ref(edge_index), rowptr)
    return rowptr


def prime_rowptr(edge_index: Tensor, num_nodes: int) -> Tensor:
    """CSR row pointer for an edge_index the kernels just produced (radius graph: target-sorted by construction), entered into
    the cache WITHOUT the sortedness check -- the check reads a device flag back, i.e. costs a host sync per new graph."""
    rowptr = ops.rowptr_from_edge_index(edge_index, num_nodes, check_sorted=False)
    if len(_ROWPTR_CACHE) > 64:
        _ROWPTR_CACHE.clear()
    key = (id(edge_index), edge_index.data_ptr(), edge_index.shape[1], edge_index._version, num_nodes)
    _ROWPTR_CACHE[key] = (weakref.ref(edge_index), rowptr)
    return rowptr


class _GNNLayerBase(nn.Module):
    limit_lip = False

    def __init__(self, node_dim: int, edge_dim: int, output_dim: int, phi_dim: int):
        super().__init__()
        # construction order (gate, phi, gamma) = the reference's, so a seeded init draws the same numbers
        self.aggr_module = AttentionalAggregation(
            gate_nn=MLP(in_channels=phi_dim, out_channels=1, hidden_layers=(128, 128), limit_lip=False))
        self.phi = MLP(in_channels=2 * node_dim + edge_dim, out_channels=phi_dim, hidden_layers=(2048, 2048),
                       limit_lip=self.limit_lip)
        self.gamma = MLP(in_channels=phi_dim + node_dim, out_channels=output_dim, hidden_layers=(2048, 2048),
                         limit_lip=self.limit_lip)
        self._dims = (node_dim, edge_dim, phi_dim)

    def net_spec(self, head: Optional[MLP] = None) -> ops.NetSpec:
        nd, ed, pd = self._dims
        return ops.NetSpec(self.phi.specs(), self.aggr_module.gate_nn.specs(), self.gamma.specs(),
                           head.specs() if head is not None else None, nd, ed, pd)

    def run(self, x: Tensor, edge_attr: Tensor, edge_index: Tensor, row_index: Optional[Tensor] = None,
            head: Optional[MLP] = None, head_extra: Optional[Tensor] = None) -> Tensor:
        """Layer (+ optional row selection and fused head MLP)."""
        spec = self.net_spec(head)
        rowptr = cached_rowptr(edge_index, x.shape[0])
        params = MLP.flat_params(spec.all_layers())
        if not torch.is_grad_enabled():
            # inference (rollouts, evaluation under no_grad): nothing is saved for a backward.  (Inside Function.forward grad mode is
            # always off and needs_input_grad ignores it, so the autograd path would keep the whole forward workspace alive per call.)
            _C.require_cuda(x, edge_attr, edge_index)
            fwd = ops.native_net_forward if ops.NATIVE else ops.net_forward
            return fwd(spec, x, edge_attr, edge_index, rowptr, row_index, head_extra, False)[0]
        return ops.GNNNetFunction.apply(x, edge_attr, edge_index, rowptr, row_index, head_extra, spec, *params)

    def forward(self, x: Tensor, edge_attr: Tensor, edge_index: Tensor) -> Tensor:
        return self.run(x, edge_attr, edge_index)

    def attention(self, data) -> Tensor:
        """Attention weights [E, 1] (reference gnn.py:44-53); inference helper, no autograd."""
        spec = self.net_spec()
        with torch.no_grad():
            E = data.edge_index.shape[1]
            ein = torch.empty(E, 2 * spec.node_dim + spec.edge_dim, device=data.x.device)
            xc, eac, eic = data.x.contiguous(), data.edge_attr.contiguous(), data.edge_index.contiguous()
            ops.call('gcbf_edge_input_fwd', ops.ptr(xc), spec.node_dim, ops.ptr(eac), spec.edge_dim, ops.ptr(eic), E,
                     ops.ptr(ein), ein.shape[1])
            msg, _, _ = ops.mlp_forward(ein, spec.phi, False)
            gate, _, _ = ops.mlp_forward(msg, spec.gate, False)
            rowptr = cached_rowptr(data.edge_index, data.x.shape[0])
            att = torch.empty(E, device=ein.device)
            scratch = torch.empty(data.x.shape[0], spec.phi_dim, device=ein.device)
            ops.call('gcbf_attn_aggr_fwd', ops.ptr(msg), spec.phi_dim, ops.ptr(gate), ops.ptr(rowptr),
                     data.x.shape[0], spec.phi_dim, ops.ptr(att), ops.ptr(scratch), spec.phi_dim)
        return att.unsqueeze(1)


class CBFGNNLayer(_GNNLayerBase):
    """phi / gamma spectral-normalised (limit_lip=True), reference gnn.py:14-36."""
    limit_lip = True


class ControllerGNNLayer(_GNNLayerBase):
    """reference gnn.py:56-73."""
    limit_lip = False


# ---- MACBF baseline layers (reference gcbf/nn/gnn.py:82-135; SURVEY 8f-4) -------------------------------------------------------
class CBFNetLayer(nn.Module):
    """Per-EDGE CBF value h_ij = phi(cat[x_i, x_j, e_ij]) -- `propagate` without aggregation (reference gnn.py:82-113).  The MLP
    (widths 64 / 128 / 64) runs on the linear kernels of the narrow ends of the GCBF MLPs (csrc/net.cu `mlp_forward` dispatch)."""

    def __init__(self, node_dim: int, edge_dim: int, output_dim: int):
        super().__init__()
        self.phi = MLP(in_channels=2 * node_dim + edge_dim, out_channels=output_dim, hidden_layers=(64, 128, 64), limit_lip=False)

    def forward(self, x: Tensor, edge_attr: Tensor, edge_index: Tensor) -> Tensor:
        return self.phi(ops.EdgeInputFunction.apply(x, edge_attr, edge_index))


class MACBFControllerLayer(nn.Module):
    """m_ij = phi(cat[x_i, x_j, e_ij]); aggr_i = max_j m_ij (0 without incoming edges); out_i = gamma(aggr_i) -- reference
    gnn.py:116-135 (`MessagePassing(aggr='max')`).  The maximum is a CSR kernel over the target-sorted edge list that also records
    the arg-max edge of every (node, channel) for the backward (csrc/macbf.cu)."""

    def __init__(self, node_dim: int, edge_dim: int, output_dim: int, phi_dim: int):
        super().__init__()
        self.phi = MLP(in_channels=2 * node_dim + edge_dim, out_channels=phi_dim, hidden_layers=(64,))
        self.gamma = MLP(in_channels=phi_dim, out_channels=output_dim, hidden_layers=(64, 128, 64))

    def forward(self, x: Tensor, edge_attr: Tensor, edge_index: Tensor) -> Tensor:
        msg = self.phi(ops.EdgeInputFunction.apply(x, edge_attr, edge_index))
        num_nodes = int(x.shape[0])
        aggr = ops.SegMaxFunction.apply(msg, cached_rowptr(edge_index, num_nodes), num_nodes)
        return self.gamma(aggr)
