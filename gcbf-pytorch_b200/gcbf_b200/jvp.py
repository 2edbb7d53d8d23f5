"""Analytic h_dot (SURVEY 8f-3): the directional derivative of the CBF along the closed-loop dynamics with the graph held fixed,

    h_dot_i = sum_k (dh_i / ds_k) . f(s_k, clamp(u_k + u_ref(s_k))),

as ONE forward-mode (tangent) pass next to the primal forward -- an additive alternative to the finite difference
(h(x + dt f) - h(x)) / dt the reference's loss uses (gcbf/algo/gcbf.py:193-207), used for evaluation and diagnostics, and by the
opt-in training loss of GCBF.params['h_dot'] = 'analytic' (the default keeps the finite difference: parity with the reference).

The primal pass is the Python-sequenced GNN forward (ops.net_forward, which keeps every layer's activations); the tangent pass walks
the same layers: each linear layer is the SAME forward GEMM kernel applied to the tangent (no bias, no activation, the forward's
1/sigma), each activation multiplies by its derivative at the primal output (gcbf_act_bwd), the attention aggregation and the
two ends (state derivative, edge-feature tangent) have their own kernels (csrc/jvp.cu).  No torch arithmetic.

The backward of (h, h_dot) (cbf_backward) walks head -> gamma -> attention -> gate -> phi for the primal and the tangent at once: the
linear layers reuse ops.mlp_backward (on the tangent's layer inputs, with the primal ReLU masks and no bias), the activations with a
second-order term (tanh) and the attention aggregation have backward kernels of their own, and the edge-feature / state-derivative ends
are VJPs in closed form (gcbf_edge_attr_bwd_ordered, gcbf_state_dot_bwd)."""
import ctypes
from typing import Optional, Tuple

import torch
from torch import Tensor

from . import _C, ops
from ._C import call, ptr


def state_dot(env, data, action: Tensor, freeze: Optional[bool] = None) -> Tensor:
    """f(x, clamp(action + u_ref(x))) for every node of the batch: [B * N, state_dim].  freeze: the single-graph reach-freeze of
    the reference's dynamics(); default = what forward_graph does (a batch of exactly one graph)."""
    _C.require_cuda(data.states, action)
    B = env._num_graphs_of(data)
    freeze = (B == 1) if freeze is None else bool(freeze)
    st, ld = ops._mat(data.states.detach())
    act = action.detach().contiguous()
    uref = env.u_ref(data)
    goal_pg = getattr(data, 'goal', None) if hasattr(data, 'goal') else None
    goal, ldg = ops._mat((goal_pg if goal_pg is not None else env._goal).contiguous())
    out = torch.empty(st.shape[0], env.state_dim, device=st.device, dtype=torch.float32)
    cfg = env._cfg(B)
    call('gcbf_state_dot', ctypes.byref(cfg), ptr(st), ld, ptr(act), ptr(uref), ptr(goal), ldg, 1 if goal_pg is not None else 0,
         1 if freeze else 0, ptr(out), env.state_dim)
    return out


def edge_attr_tangent(env, states: Tensor, sdot: Tensor, edge_index: Tensor) -> Tensor:
    st, ld = ops._mat(states.detach())
    sd, ldsd = ops._mat(sdot)
    ei = edge_index.contiguous()
    E = int(ei.shape[1])
    out = torch.empty(E, env.edge_dim, device=st.device, dtype=torch.float32)
    call('gcbf_edge_attr_tangent', ops.ENV_IDS[env.ENV_NAME], ptr(st), ld, ptr(sd), ldsd, ptr(ei) if E else None, E, ptr(out) if E else None)
    return out


def state_dot_bwd(env, data, action: Tensor, d_sdot: Tensor, d_action: Tensor, freeze: Optional[bool] = None) -> Tensor:
    """d_action += (d state_dot / d action)^T d_sdot: the VJP of state_dot (same arguments) through the clamp and the reach-freeze."""
    B = env._num_graphs_of(data)
    freeze = (B == 1) if freeze is None else bool(freeze)
    st, ld = ops._mat(data.states.detach())
    act = action.detach().contiguous()
    uref = env.u_ref(data)
    goal_pg = getattr(data, 'goal', None) if hasattr(data, 'goal') else None
    goal, ldg = ops._mat((goal_pg if goal_pg is not None else env._goal).contiguous())
    ds, ldd = ops._mat(d_sdot)
    cfg = env._cfg(B)
    call('gcbf_state_dot_bwd', ctypes.byref(cfg), ptr(st), ld, ptr(act), ptr(uref), ptr(goal), ldg, 1 if goal_pg is not None else 0,
         1 if freeze else 0, ptr(ds), ldd, ptr(d_action), 1)
    return d_action


def edge_attr_bwd_ordered(env, states: Tensor, edge_index: Tensor, d_edge_attr: Tensor) -> Tensor:
    """d states [nodes, state_dim] of sum(d_edge_attr * edge_attr(states)): the deterministic edge-feature VJP, which is also the VJP of
    edge_attr_tangent with respect to s_dot (the tangent is linear in s_dot with the same Jacobian)."""
    st, ld = ops._mat(states.detach())
    ei = edge_index.contiguous()
    E = int(ei.shape[1])
    d_states = torch.zeros(st.shape[0], ld, device=st.device, dtype=torch.float32)
    d_ea = d_edge_attr.contiguous()
    call('gcbf_edge_attr_bwd_ordered', ops.ENV_IDS[env.ENV_NAME], ptr(st), ld, ptr(ei) if E else None, E, int(st.shape[0]),
         ptr(d_ea) if E else None, ptr(d_states))
    return d_states[:, :env.state_dim]


def mlp_tangent(ctx: ops.MLPCtx, layers, t: Tensor, keep: bool = False):
    """Tangent of an MLP at the primal activations kept in `ctx` (ops.mlp_forward(..., save=True)).  keep: also return what the backward
    needs -- (t, tctx, tz): tctx an ops.MLPCtx whose acts are the tangent's layer inputs (with their own fp16 companions where a layer
    runs on the tensor cores) and whose 1/sigma and u, v are the primal's; tz the output layer's pre-activation tangent."""
    if t.shape[0] == 0:                                   # a graph without edges: nothing to propagate through the edge MLPs
        out = torch.empty(0, int(layers[-1].W.shape[0]), device=t.device, dtype=torch.float32)
        return (out, None, None) if keep else out
    tctx = ops.MLPCtx(inv_sigma=ctx.inv_sigma, uv=ctx.uv) if keep else None
    tz = None
    for l, L in enumerate(layers):
        N = int(L.W.shape[0])
        lin = ops.LinearSpec(L.W, torch.zeros(N, device=t.device, dtype=torch.float32), L.u, L.v, ops.ACT_NONE)
        t_in = t
        t, c1, _ = ops.mlp_forward(t, [lin], keep, inv_sigmas=[ctx.inv_sigma[l]], uvs=[None])   # the forward's sigma: no new power iteration
        if keep:
            tctx.acts.append(t_in)
            tctx.acts_h.append(c1.acts_h[0])
        tz = t
        if L.act != ops.ACT_NONE:
            t = ops.act_bwd(t, ctx.acts[l + 1], L.act)                                   # t * act'(y) from the primal output y
    return (t, tctx, tz) if keep else t


def net_tangent(spec: ops.NetSpec, ctx, t_edge_attr: Tensor, rowptr: Tensor, row_index: Optional[Tensor], keep: bool = False):
    """Tangent of ops.net_forward's output for a tangent of edge_attr (node features x are constants).  keep: returns (t, tstate), tstate
    what cbf_backward needs."""
    c_phi, c_gate, c_gamma, c_head, msg, att, Nn, E = ctx
    dev = t_edge_attr.device
    C, nd, ed = spec.phi_dim, spec.node_dim, spec.edge_dim
    t_in = torch.zeros(E, 2 * nd + ed, device=dev, dtype=torch.float32)                 # d cat[x_i, x_j, e] = [0, 0, de]
    if E:
        ops.copy2d(t_edge_attr.contiguous(), t_in[:, 2 * nd:], E, ed)
    st = {}

    def run(name, c, layers, t):
        if not keep:
            return mlp_tangent(c, layers, t)
        t, tctx, tz = mlp_tangent(c, layers, t, True)
        st[name] = (tctx, tz)
        return t
    t_msg = run('phi', c_phi, spec.phi, t_in)
    t_gate = run('gate', c_gate, spec.gate, t_msg)
    t_gin_all = torch.zeros(Nn, C + nd, device=dev, dtype=torch.float32)                # d cat[aggr, x] = [d aggr, 0]
    call('gcbf_attn_aggr_tangent', ptr(msg) if E else None, C, ptr(t_msg) if E else None, C, ptr(att) if E else None,
         ptr(t_gate) if E else None, ptr(rowptr), Nn, C, ptr(t_gin_all), C + nd)
    if row_index is not None:
        t_gin = torch.empty(row_index.numel(), C + nd, device=dev, dtype=torch.float32)
        ops.rows_gather(t_gin_all, row_index, t_gin)
    else:
        t_gin = t_gin_all
    t = run('gamma', c_gamma, spec.gamma, t_gin)
    if spec.head is not None:
        t = run('head', c_head, spec.head, t)
    if not keep:
        return t
    st['t_msg'], st['t_gate'] = t_msg, t_gate
    return t, st


def _mlp_pair_backward(c: ops.MLPCtx, tc: ops.MLPCtx, tz: Tensor, layers, dy: Tensor, dty: Tensor, need_dx: bool, need_dtx: bool,
                       dx_out: Optional[Tensor] = None, dtx_out: Optional[Tensor] = None):
    """Backward of one MLP for the primal and its tangent: (dL/dx, dL/dx_dot).  Weight gradients of both go to the layers' .grad (under
    ops.GRAD_INTO_PARAM); the bias gradient comes from the primal only."""
    act = layers[-1].act
    if act != ops.ACT_NONE:
        dy, dty = dy.contiguous(), dty.contiguous()
        dz, dtz = torch.empty_like(dy), torch.empty_like(dty)
        call('gcbf_act_tangent_bwd', ptr(dy), ptr(dty), ptr(c.acts[-1].contiguous()), ptr(tz.contiguous()) if act == ops.ACT_TANH else None,
             dy.numel(), act, ptr(dz), ptr(dtz))
    else:
        dz, dtz = dy, dty
    dx, _ = ops.mlp_backward(c, layers, dz, need_dx, dx_out=dx_out, dx_accumulate=dx_out is not None, dy_is_preact=True)
    dtx, _ = ops.mlp_backward(tc, layers, dtz, need_dtx, dx_out=dtx_out, dx_accumulate=dtx_out is not None, mask_acts=c.acts,
                              bias_grad=False, dy_is_preact=True)
    return dx, dtx


def net_backward_hdot(spec: ops.NetSpec, ctx, tstate, d_out: Tensor, d_tout: Tensor, rowptr: Tensor, row_index: Optional[Tensor]):
    """Backward of (net_forward, net_tangent) given dL/d out and dL/d out_dot: parameter gradients into the layers' .grad (ops.GRAD_INTO_PARAM)
    and returns dL/d t_edge_attr [E, edge_dim] (None for a graph without edges)."""
    c_phi, c_gate, c_gamma, c_head, msg, att, Nn, E = ctx
    dev = d_out.device
    C, nd = spec.phi_dim, spec.node_dim
    d_feat, d_tfeat = d_out, d_tout
    if spec.head is not None:
        d_feat, d_tfeat = _mlp_pair_backward(c_head, *tstate['head'], spec.head, d_out, d_tout, True, True)
    d_gin, d_tgin = _mlp_pair_backward(c_gamma, *tstate['gamma'], spec.gamma, d_feat, d_tfeat, True, True)
    if E == 0:
        return None                                      # phi / gate saw no rows: no gradient for them, h_dot does not depend on the states
    if row_index is not None:
        d_gin_all = torch.zeros(Nn, C + nd, device=dev, dtype=torch.float32)
        d_tgin_all = torch.zeros(Nn, C + nd, device=dev, dtype=torch.float32)
        ops.rows_scatter(d_gin, row_index, d_gin_all)
        ops.rows_scatter(d_tgin, row_index, d_tgin_all)
    else:
        d_gin_all, d_tgin_all = d_gin, d_tgin
    t_msg, t_gate = tstate['t_msg'], tstate['t_gate']
    d_msg = torch.empty(E, C, device=dev, dtype=torch.float32)
    d_gate = torch.empty(E, 1, device=dev, dtype=torch.float32)
    d_tmsg = torch.empty(E, C, device=dev, dtype=torch.float32)
    d_tgate = torch.empty(E, 1, device=dev, dtype=torch.float32)
    call('gcbf_attn_aggr_bwd', ptr(msg), C, ptr(att), ptr(rowptr), Nn, C, ptr(d_gin_all), C + nd, ptr(d_msg), C, ptr(d_gate), 0)
    call('gcbf_attn_aggr_tangent_bwd', ptr(msg), C, ptr(t_msg), C, ptr(att), ptr(t_gate), ptr(rowptr), Nn, C, ptr(d_tgin_all), C + nd,
         ptr(d_tmsg), C, ptr(d_tgate), ptr(d_msg), C, ptr(d_gate), 1)
    _mlp_pair_backward(c_gate, *tstate['gate'], spec.gate, d_gate, d_tgate, True, True, dx_out=d_msg, dtx_out=d_tmsg)
    _, d_tein = _mlp_pair_backward(c_phi, *tstate['phi'], spec.phi, d_msg, d_tmsg, False, True)
    return d_tein[:, 2 * nd:]


def cbf_forward_saved(cbf, data):
    """h = cbf(data) through ops.net_forward with every activation kept: (h [B * n, 1], state for h_dot_tangent / cbf_backward)."""
    from .data import agent_row_index
    from .nn.gnn import cached_rowptr
    _C.require_cuda(data.states, data.edge_attr, data.edge_index)
    layer = cbf.feat_transformer.module_0
    spec = layer.net_spec(cbf.feat_2_CBF)
    x, ea, ei = data.x.contiguous(), data.edge_attr.detach().contiguous(), data.edge_index.contiguous()
    rowptr = cached_rowptr(data.edge_index, int(x.shape[0]))
    rows = agent_row_index(data)
    with torch.no_grad():
        h, ctx = ops.net_forward(spec, x, ea, ei, rowptr, rows, None, True)
    return h, dict(spec=spec, ctx=ctx, ei=ei, rowptr=rowptr, rows=rows)


def h_dot_tangent(env, data, action: Tensor, state: dict, freeze: Optional[bool] = None, keep: bool = False) -> Tensor:
    """h_dot [B * n, 1] at the forward kept in `state` (cbf_forward_saved) along x_dot = f(x, clamp(action + u_ref)); keep: also keep what
    cbf_backward needs (in `state`)."""
    _C.require_cuda(action)
    with torch.no_grad():
        sdot = state_dot(env, data, action, freeze)
        t_ea = edge_attr_tangent(env, data.states, sdot, state['ei'])
        if not keep:
            return net_tangent(state['spec'], state['ctx'], t_ea, state['rowptr'], state['rows'])
        h_dot, state['tangent'] = net_tangent(state['spec'], state['ctx'], t_ea, state['rowptr'], state['rows'], keep=True)
    return h_dot


def cbf_backward(env, data, action: Tensor, state: dict, d_h: Tensor, d_hdot: Tensor, d_action: Tensor, freeze: Optional[bool] = None):
    """Backward of (h, h_dot) = (cbf_forward_saved, h_dot_tangent(..., keep=True)): the CBF's parameter gradients go to its .grad (run under
    ops.GRAD_INTO_PARAM), dL/d action through h_dot -> x_dot -> clamp is ADDED onto d_action [B * n, action_dim]."""
    with torch.no_grad():
        d_t_ea = net_backward_hdot(state['spec'], state['ctx'], state['tangent'], d_h, d_hdot, state['rowptr'], state['rows'])
        if d_t_ea is None:
            return d_action
        d_sdot = edge_attr_bwd_ordered(env, data.states, state['ei'], d_t_ea)
        return state_dot_bwd(env, data, action, d_sdot, d_action, freeze)


def cbf_value_and_h_dot(cbf, env, data, action: Tensor, freeze: Optional[bool] = None) -> Tuple[Tensor, Tensor]:
    """(h, h_dot) of a CBFGNN on a batch: h [B * n, 1] exactly as cbf(data) (one spectral-norm power iteration, like every forward of
    the reference), h_dot [B * n, 1] = dh/dt along x_dot = f(x, clamp(action + u_ref)) with the edges of `data` held fixed."""
    _C.require_cuda(data.states, data.edge_attr, data.edge_index, action)
    h, state = cbf_forward_saved(cbf, data)
    return h, h_dot_tangent(env, data, action, state, freeze)
