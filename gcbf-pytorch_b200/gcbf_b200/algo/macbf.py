"""MACBF, the paper's baseline algorithm (reference gcbf/algo/macbf.py:20-239; SURVEY 8f-4), on the sm_90a kernels.

Differences from GCBF that matter for the kernels: the CBF is a per-EDGE value h_ij (an MLP on cat[x_i, x_j, e_ij], no aggregation),
the actor aggregates with a per-target MAX, the safe / unsafe sets are per-edge distance tests, the h_dot condition uses the
retained edges only (no re-linked graph), the env is built with `max_neighbors = 12` (top-k filtered radius graph), and the
accuracies are plain element-wise means.  The train step is sequenced from Python over autograd Functions whose forward / backward
are C-ABI calls (ops.py: EdgeInputFunction, MLPFunction -> gcbf_mlp_forward / gcbf_mlp_backward, SegMaxFunction, GatherCatFunction,
EdgeAttrFunction, the env's step Function); the losses, their gradients w.r.t. (h, h_next, actions) and the accuracies come from
gcbf_macbf_loss_partials / gcbf_macbf_loss_grads with the optional all-reduce of the partial sums in between (environment-parallel
ranks reproduce the single-process means), clip + Adam are the fused kernels of the GCBF path on the flat parameter bucket.
"""
from typing import Dict, Optional

import numpy as np
import torch
import torch.nn as nn
from torch import Tensor

from .. import _C, ops
from ..controller import MACBFController
from ..data import Batch
from ..nn import CBFNetLayer, GraphSequential
from .gcbf import GCBF


class CBFNet(nn.Module):
    """Pair-wise CBF values for the (top-k filtered) edges of the graph: [E, 1] (reference macbf.py:20-51; the reference does not
    restrict the result to agent rows either -- every edge already ends in an agent)."""

    def __init__(self, num_agents: int, node_dim: int, edge_dim: int):
        super().__init__()
        self._num_agents = num_agents
        self._top_k = 12
        self.net = GraphSequential(CBFNetLayer(node_dim=node_dim, edge_dim=edge_dim, output_dim=1))

    def forward(self, data) -> Tensor:
        return self.net(data.x, data.edge_attr, data.edge_index)


class MACBF(GCBF):
    GRAD_INTO_PARAM = True      # False: the MLP weight gradients travel back through autograd (A/B switch, tests run both)

    def __init__(self, env, num_agents: int, node_dim: int, edge_dim: int, action_dim: int, device: torch.device,
                 batch_size: int = 500, params: Optional[dict] = None, reference_rng: bool = True):
        """reference_rng: the reference constructs GCBF's two 12 M-parameter networks first (macbf.py:65-72: `super().__init__`) and
        then replaces them, so its MACBF networks are initialised from the RNG stream AFTER those draws.  True (default) does the same
        on the CPU generator and discards the result: seeded runs start from the reference's weights.  False skips it (a checkpoint is
        loaded anyway, or the exact initial weights do not matter)."""
        self._reference_rng = bool(reference_rng)
        super().__init__(env=env, num_agents=num_agents, node_dim=node_dim, edge_dim=edge_dim, action_dim=action_dim, device=device)
        self.lr_cbf, self.lr_actor = 3e-4, 1e-3            # macbf.py:84-85
        self.batch_size = batch_size
        self.params = params if params is not None else {
            'alpha': 1.0, 'eps': 0.02, 'inner_iter': 10, 'loss_action_coef': 0.001, 'loss_unsafe_coef': 1., 'loss_safe_coef': 1.,
            'loss_h_dot_coef': 0.1}

    def _build_networks(self, num_agents: int, node_dim: int, edge_dim: int, action_dim: int, device):
        if self._reference_rng:
            super()._build_networks(num_agents, node_dim, edge_dim, action_dim, torch.device('cpu'))      # RNG draws only
        self.cbf = CBFNet(num_agents=num_agents, node_dim=node_dim, edge_dim=edge_dim).to(device)
        self.actor = MACBFController(num_agents=num_agents, node_dim=node_dim, edge_dim=edge_dim, phi_dim=128,
                                     action_dim=action_dim).to(device)

    # ---- rollout-time API (macbf.py:105-118) ----------------------------------------------------------------------------------
    @torch.no_grad()
    def step(self, data, prob: float) -> Tensor:
        action = self.actor(data)
        prob = max(prob, 0.5)
        if np.random.rand() < prob:
            action = torch.zeros_like(action)
        is_safe = not bool(torch.any(self._env.unsafe_mask(data)))
        self.buffer.append(data, is_safe)
        return action

    def use_device_replay(self, capacity: int = 4096):
        raise NotImplementedError('the device replay ring re-links sampled graphs with the unfiltered radius graph; MACBF keeps the list buffer')

    # ---- the train step -------------------------------------------------------------------------------------------------------
    def train_step(self, graphs, apply_optim: bool = True, compute_acc_h_dot: bool = True) -> Dict[str, Tensor]:
        """One inner iteration of MACBF.update (macbf.py:135-186) on a collated batch.  Returns device tensors (no host sync):
        'scalars' = [loss_unsafe, loss_safe, loss_h_dot, loss_action, acc_unsafe, acc_safe, total_loss, acc_derivative], plus
        h / h_next (per edge), actions, the per-edge masks."""
        env, hp = self._env, self.params
        bucket = self._ensure_bucket()
        red = self._reducer()
        dev = graphs.states.device
        h = self.cbf(graphs)                                             # macbf.py:137  [E, 1]
        actions = self.actor(graphs)                                     # macbf.py:138
        masks = env.edge_masks(graphs)                                   # macbf.py:144, 156 -- one launch
        graphs_next = env.forward_graph(graphs, actions)                 # macbf.py:167 (retained edges)
        h_next = self.cbf(graphs_next)                                   # macbf.py:168
        E, M, a_dim = int(h.shape[0]), int(actions.shape[0]), self.action_dim
        hd, hnd, actd = h.detach(), h_next.detach(), actions.detach()
        safe_u8, unsafe_u8 = masks[0].view(torch.uint8), masks[1].view(torch.uint8)
        partial = torch.empty(16, device=dev, dtype=torch.float64)
        dt = float(env.dt)
        _C.call('gcbf_macbf_loss_partials', _C.ptr(hd), _C.ptr(hnd), _C.ptr(safe_u8), _C.ptr(unsafe_u8), E, _C.ptr(actd), a_dim, M,
                float(hp['alpha']), float(hp['eps']), dt, _C.ptr(partial))
        red.sum_(partial)                                                # global counts => global means
        d_h, d_hn, d_act = torch.empty_like(hd), torch.empty_like(hnd), torch.empty_like(actd)
        scalars = torch.empty(8, device=dev, dtype=torch.float32)
        _C.call('gcbf_macbf_loss_grads', _C.ptr(hd), _C.ptr(hnd), _C.ptr(safe_u8), _C.ptr(unsafe_u8), E, _C.ptr(actd), a_dim, M,
                float(hp['alpha']), float(hp['eps']), dt, float(hp['loss_unsafe_coef']), float(hp['loss_safe_coef']),
                float(hp['loss_h_dot_coef']), float(hp['loss_action_coef']), _C.ptr(partial), _C.ptr(d_h), _C.ptr(d_hn), _C.ptr(d_act),
                _C.ptr(scalars))
        bucket.zero_grad()                                               # macbf.py:179-180
        # the parameters' .grad are views into the flat bucket.  GRAD_INTO_PARAM: the weight-grad kernels of gcbf_mlp_backward accumulate
        # straight into them and autograd sees no parameter gradients (otherwise autograd adds each returned gradient with an ATen
        # kernel: 37 extra launches per step)
        ops.GRAD_INTO_PARAM = self.GRAD_INTO_PARAM
        try:
            if E:
                torch.autograd.backward([h, h_next, actions], [d_h, d_hn, d_act])      # macbf.py:181
            else:
                torch.autograd.backward([actions], [d_act])
        finally:
            ops.GRAD_INTO_PARAM = False
        red.sum_(bucket.grad)
        if apply_optim:
            self.optim_step()                                            # macbf.py:182-186: clip(1e-3) per net + Adam, fused
        return dict(scalars=scalars, h=hd, actions=actd, h_next=hnd, safe_mask=masks[0], unsafe_mask=masks[1],
                    acc_h_dot=scalars[7].to(torch.float64))

    def update(self, step: int, writer=None) -> dict:
        """Reference-shaped update loop (macbf.py:120-207): same sampling as GCBF.update, `inner_iter` train steps."""
        seg_len = 3
        info = {}
        for i_inner in range(self.params['inner_iter']):
            if self.memory.size == 0:
                graph_list = self.buffer.sample(self.batch_size // 5, seg_len)
            else:
                graph_list = (self.buffer.sample(self.batch_size // 10, seg_len, True) +
                              self.memory.sample(self.batch_size // 5 - self.batch_size // 10, seg_len, True))
            res = self.train_step(Batch.from_data_list(graph_list))
            s = res['scalars'].tolist()                                  # the one host sync per inner iteration
            info = {'acc/safe': s[5], 'acc/unsafe': s[4], 'acc/derivative': s[7]}
            if writer is not None:
                it = step * self.params['inner_iter'] + i_inner
                for tag, val in (('loss/unsafe', s[0]), ('loss/safe', s[1]), ('loss/derivative', s[2]), ('loss/action', s[3]),
                                 ('acc/unsafe', s[4]), ('acc/safe', s[5]), ('acc/derivative', s[7])):
                    writer.add_scalar(tag, val, it)
        self.memory.merge(self.buffer)
        self.buffer.clear()
        return info

    def apply(self, data, rand: Optional[float] = 0, max_iter: int = 30) -> Tensor:
        """Reference macbf.py:209-239.  The reference hands `action = self.actor(data).detach()` to Adam(lr = 1) and back-propagates
        mean(relu(-h_dot - alpha h)) -- but that leaf does not require grad, so it never receives a gradient, `Adam.step()` skips it
        and the loop only evaluates the CBF up to 32 times: the returned action IS the actor's output (pinned by the fixtures'
        `apply_action`, generated by the reference's own apply).  This method returns it without the idle CBF evaluations."""
        with torch.no_grad():
            return self.actor(data)
