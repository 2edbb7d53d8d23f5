"""GCBF: CBF network + actor + the train step of reference gcbf/algo/gcbf.py:64-309 on the sm_90a kernels.

What changes relative to the reference's `update` body (results identical, see tests/test_parity_gpu.py):
  * safe/unsafe masks and the re-linked radius graphs are ONE kernel launch over the whole batch instead of
    per-graph Python loops (gcbf.py:168, 180, 195-199);
  * the four losses, their gradients w.r.t. (h, h_next, actions) and the accuracies come from two small
    kernels (ops: gcbf_loss_partials / gcbf_loss_grads) with an optional all-reduce of the 9 partial sums in
    between, so environment-parallel ranks reproduce the single-process masked means;
  * parameters and gradients of both nets live in ONE flat fp32 bucket: a single NCCL all-reduce, then
    global-norm clip + Adam as one fused kernel per net (gcbf.py:220-226);
  * the M x M broadcast of `acc/derivative` (gcbf.py:209) is an exact pair count, not an M x M temporary.
"""
import ctypes
import os
import weakref
from typing import Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn
from torch import Tensor

from .. import _C, ops
from ..controller import GNNController
from ..data import Batch, Data, agent_row_index
from ..nn import MLP, CBFGNNLayer, GraphSequential
from .base import Algorithm
from .buffer import Buffer


class CBFGNN(nn.Module):
    """h(x): CBFGNNLayer(out=1024) -> agent rows -> MLP(1024 -> 512,128,32 -> 1, Tanh); reference gcbf.py:21-61."""

    def __init__(self, num_agents: int, node_dim: int, edge_dim: int, phi_dim: int):
        super().__init__()
        self.num_agents = num_agents
        self.feat_transformer = GraphSequential(
            CBFGNNLayer(node_dim=node_dim, edge_dim=edge_dim, output_dim=1024, phi_dim=phi_dim))
        self.feat_2_CBF = MLP(in_channels=1024, out_channels=1, hidden_layers=(512, 128, 32),
                              output_activation=nn.Tanh())

    def forward(self, data) -> Tensor:
        layer = self.feat_transformer.module_0
        return layer.run(data.x, data.edge_attr, data.edge_index, row_index=agent_row_index(data), head=self.feat_2_CBF)

    def attention(self, data) -> Tensor:
        return self.feat_transformer.module_0.attention(data)


class _FlatBucket:
    """All parameters of a list of modules re-homed into one flat fp32 buffer (and their .grad into a second
    one), so the gradient all-reduce is a single collective and clip+Adam a single pass per net."""

    ALIGN = 64          # floats: every parameter starts on a 256-byte boundary (16-byte vector loads / cp.async / TMA of the weight
                        # matrices; without it the 1-element bias of the gate's last layer shifts every later matrix by 4 bytes)

    def __init__(self, modules: List[nn.Module], device):
        up = lambda n: (n + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        self.ranges, self.tail_start = [], []
        params, offsets = [], []
        off = 0
        for m in modules:
            start, tail = off, None
            for name, p in m.named_parameters():
                # where the [gamma + head] parameters of the net start (parameters() order: gate_nn, phi, gamma, head): that tail of
                # a net's range is final before the E-row phi / gate backward has run, so its all-reduce can start early
                if '.gamma.' in name and tail is None:
                    tail = off
                params.append(p)
                offsets.append(off)
                off += up(p.numel())
            self.ranges.append((start, off))
            self.tail_start.append(off if tail is None else tail)
        total = off
        self.flat = torch.zeros(total, device=device, dtype=torch.float32)      # the padding stays zero: zero gradient, zero Adam update
        self.grad = torch.zeros(total, device=device, dtype=torch.float32)
        self.exp_avg = torch.zeros(total, device=device, dtype=torch.float32)
        self.exp_avg_sq = torch.zeros(total, device=device, dtype=torch.float32)
        for p, o in zip(params, offsets):
            n = p.numel()
            self.flat[o:o + n].copy_(p.data.reshape(-1))
            p.data = self.flat[o:o + n].view(p.shape)
            p.grad = self.grad[o:o + n].view(p.shape)
        self.params, self.offsets = params, offsets
        self.sumsq = torch.zeros(len(modules), device=device, dtype=torch.float64)
        self.step = 0

    def zero_grad(self):
        self.grad.zero_()


class GCBF(Algorithm):

    def __init__(self, env, num_agents: int, node_dim: int, edge_dim: int, action_dim: int, device: torch.device,
                 batch_size: int = 500, params: Optional[dict] = None):
        super().__init__(env=env, num_agents=num_agents, node_dim=node_dim, edge_dim=edge_dim, action_dim=action_dim,
                         device=device)
        self._build_networks(num_agents, node_dim, edge_dim, action_dim, device)
        self.lr_cbf, self.lr_actor = 3e-4, 1e-3            # gcbf.py:102-103
        self.max_grad_norm = 1e-3                          # gcbf.py:223-224
        self._bucket: Optional[_FlatBucket] = None
        self.buffer = Buffer()
        self.memory = Buffer()
        self.device_replay = False                         # use_device_replay() swaps the two lists for device rings
        self.batch_size = batch_size
        self.params = params if params is not None else {
            'alpha': 1.0, 'eps': 0.02, 'inner_iter': 10, 'loss_action_coef': 0.001, 'loss_unsafe_coef': 1.,
            'loss_safe_coef': 1., 'loss_h_dot_coef': 0.1}
        self.process_group = None   # set to a torch.distributed group for data-parallel training
        self._matmul_mode()         # validates params['matmul'] and puts the mode on the two modules

    def _build_networks(self, num_agents: int, node_dim: int, edge_dim: int, action_dim: int, device):
        # models: same construction order as the reference (gcbf.py:87-100) => same seeded initialisation
        self.cbf = CBFGNN(num_agents=num_agents, node_dim=node_dim, edge_dim=edge_dim, phi_dim=256).to(device)
        self.actor = GNNController(num_agents=num_agents, node_dim=node_dim, edge_dim=edge_dim, phi_dim=256,
                                   action_dim=action_dim).to(device)

    # ---- rollout-time API ---------------------------------------------------------------------------
    @torch.no_grad()
    def act(self, data) -> Tensor:
        self._matmul_mode()
        return self.actor(data)

    @torch.no_grad()
    def step(self, data, prob: float) -> Tensor:
        self._matmul_mode()
        action = self.actor(data)
        if np.random.rand() < prob:
            action = torch.zeros_like(action)
        is_safe = not bool(torch.any(self._env.unsafe_mask(data)))
        self.buffer.append(data, is_safe)
        return action

    def is_update(self, step: int) -> bool:
        return step % self.batch_size == 0

    def use_device_replay(self, capacity: int = 4096):
        """Keep visited graphs as device-resident (states, u_ref) rings and collate sampled batches on the GPU
        (algo/device_buffer.py) instead of Python lists of `Data` + `Batch.from_data_list`.  Same sampling semantics."""
        from .device_buffer import DeviceReplay
        assert self.buffer.size == 0 and self.memory.size == 0, 'switch before collecting data'
        self.buffer, self.memory = DeviceReplay(self.device, capacity), DeviceReplay(self.device, capacity)
        self.device_replay = True
        return self

    # ---- the train step -----------------------------------------------------------------------------
    def _ensure_bucket(self) -> _FlatBucket:
        if self._bucket is None:
            self._bucket = _FlatBucket([self.cbf, self.actor], self.device)
        return self._bucket

    def _reducer(self):
        from ..distributed import Reducer
        red = getattr(self, '_red', None)
        if red is None or red.group is not self.process_group:
            red = self._red = Reducer(self.process_group)
        return red

    def _side_stream(self, dev, num_edges: int = 0):
        """Second CUDA stream for the actor / re-linked passes.  GCBF_TWO_STREAMS: 1 = always, 0 = never, unset = only while
        the batch is small enough for the overlap to pay (measured: -12 % step time at 24 k edges per step, +8 % at 206 k,
        where the GPU is already at its power limit and the two working sets evict each other from L2)."""
        mode = os.environ.get('GCBF_TWO_STREAMS', 'auto')
        if mode == '0' or (mode != '1' and num_edges > 100_000):
            return None
        st = getattr(self, '_side', None)
        if st is None:
            st = self._side = torch.cuda.Stream(device=dev, priority=int(os.environ.get('GCBF_SIDE_PRIORITY', '0')))
        return st

    def train_step(self, graphs, apply_optim: bool = True, compute_acc_h_dot: bool = True) -> Dict[str, Tensor]:
        """One inner iteration of GCBF.update (gcbf.py:158-226) on a collated batch.  Returns device tensors
        (no host sync): 'scalars' = [loss_unsafe, loss_safe, loss_h_dot, loss_action, acc_unsafe, acc_safe,
        total_loss, num_agents], 'acc_h_dot', plus h / actions / h_next / h_next_new for inspection (views into the step's
        workspace: valid until the next train_step of this object).
        params['h_dot'] selects the CBF-condition loss: 'finite_difference' (the default, the reference's) or 'analytic'
        (_train_step_analytic)."""
        self._matmul_mode()
        if self._h_dot_mode() == 'analytic':
            self._refuse_fp16("params['h_dot'] = 'analytic' training")
            return self._train_step_analytic(graphs, apply_optim, compute_acc_h_dot)
        if ops.NATIVE:
            return self._train_step_native(graphs, apply_optim, compute_acc_h_dot)
        from ..arena import ARENA
        ARENA.begin(graphs.states.device)      # every activation / gradient below is a view into the step arena
        try:
            return self._train_step(graphs, apply_optim, compute_acc_h_dot)
        finally:
            ARENA.end()

    H_DOT_MODES = ('finite_difference', 'analytic')
    MATMUL_MODES = ('fp32', 'fp16')

    def _matmul_mode(self) -> str:
        """params['matmul']: 'fp32' (default; 3xFP16 tensor-core products, fp32-grade) or 'fp16' (one fp16 product per k-slice in
        the 2048-wide layers: faster, with the accuracy contract of DESIGN section 5).  The two modules read the key at every pass
        (their layers hold a weak reference to this object), so self.cbf(data) / self.actor(data) -- rollouts, VectorRollout, the
        Trainer -- run in the mode the key has at that moment.  Only the library-sequenced passes have the fp16 kernels: with
        GCBF_NATIVE=0 'fp16' is refused."""
        mode = self.params.get('matmul', 'fp32')
        if mode not in self.MATMUL_MODES:
            raise ValueError(f"params['matmul'] must be one of {self.MATMUL_MODES}, got {mode!r}")
        if mode == 'fp16' and not ops.NATIVE:
            raise ValueError("params['matmul'] = 'fp16' needs the library-sequenced passes (GCBF_NATIVE=1)")
        for m in (self.cbf, self.actor):
            layer = m.feat_transformer.module_0
            if layer._matmul_owner is None or layer._matmul_owner() is not self:
                layer._matmul_owner = weakref.ref(self)
        return mode

    def _matmul_products(self) -> int:
        return ops.MATMUL_PRODUCTS[self._matmul_mode()]

    def set_matmul(self, mode: str):
        """Switch the tensor-core precision ('fp32' or 'fp16') of every later pass of both nets."""
        old = self.params.get('matmul', 'fp32')
        self.params['matmul'] = mode
        try:
            self._matmul_mode()
        except ValueError:
            self.params['matmul'] = old
            raise
        return self

    def _refuse_fp16(self, what: str):
        if self._matmul_mode() == 'fp16':
            raise ValueError(f"{what} is sequenced in Python on the 3xFP16 kernels and does not run in params['matmul'] = 'fp16'")

    def _h_dot_mode(self) -> str:
        mode = self.params.get('h_dot', 'finite_difference')
        if mode not in self.H_DOT_MODES:
            raise ValueError(f"params['h_dot'] must be one of {self.H_DOT_MODES}, got {mode!r}")
        return mode

    def _train_step_analytic(self, graphs, apply_optim: bool, compute_acc_h_dot: bool) -> Dict[str, Tensor]:
        """One inner iteration with the analytic h_dot in the CBF-condition loss (params['h_dot'] = 'analytic'): the losses, masked
        means and accuracies of gcbf.py:164-218 with h_dot = J_h(s) . f(s, clamp(actions + u_ref(s))) (gcbf_b200/jvp.py: the edges
        of `graphs` held fixed, the same 1/sigma and u, v as h -- ONE power iteration, where the finite-difference step does three) in
        place of the finite difference, differentiated through: the CBF gets gradients through h and h_dot (incl. the second-order
        terms of the attention softmax, the head's tanh and sigma), the actor through loss_action and h_dot -> x_dot -> clamp -> actions.
        No h_next, no re-linked graph.  Python-sequenced on the current stream."""
        from .. import jvp
        env, hp = self._env, self.params
        bucket = self._ensure_bucket()
        dev = graphs.states.device
        red = self._reducer()
        M = graphs.u_ref.shape[0]
        a_dim = self.action_dim

        h, state = jvp.cbf_forward_saved(self.cbf, graphs)               # gcbf.py:161  (the one power iteration)
        actions = self.actor(graphs)                                     # gcbf.py:162
        masks = env._masks(graphs)                                       # gcbf.py:168, 180
        actd = actions.detach()
        hdot = jvp.h_dot_tangent(env, graphs, actd, state, keep=True)    # [M, 1]

        partial = torch.empty(16, device=dev, dtype=torch.float64)
        safe_u8, unsafe_u8 = masks[0].view(torch.uint8), masks[1].view(torch.uint8)
        _C.call('gcbf_loss_partials_hdot', _C.ptr(h), _C.ptr(hdot), _C.ptr(actd), a_dim, _C.ptr(safe_u8), _C.ptr(unsafe_u8), M,
                float(hp['alpha']), float(hp['eps']), _C.ptr(partial))
        red.sum_(partial)                                                # global counts => global masked means
        d_h, d_hdot, d_act = torch.empty_like(h), torch.empty_like(hdot), torch.empty_like(actd)
        scalars = torch.empty(8, device=dev, dtype=torch.float32)
        _C.call('gcbf_loss_grads_hdot', _C.ptr(h), _C.ptr(hdot), _C.ptr(actd), a_dim, _C.ptr(safe_u8), _C.ptr(unsafe_u8), M,
                float(hp['alpha']), float(hp['eps']), float(hp['loss_unsafe_coef']), float(hp['loss_safe_coef']),
                float(hp['loss_h_dot_coef']), float(hp['loss_action_coef']), _C.ptr(partial), _C.ptr(d_h), _C.ptr(d_hdot),
                _C.ptr(d_act), _C.ptr(scalars))

        bucket.zero_grad()
        ops.GRAD_INTO_PARAM = True     # weight-grad kernels accumulate straight into the bucket's .grad views
        try:
            jvp.cbf_backward(env, graphs, actd, state, d_h, d_hdot, d_act)   # CBF gradients; d_act += the h_dot path
            torch.autograd.backward(actions, d_act)
        finally:
            ops.GRAD_INTO_PARAM = False

        hdot = hdot.reshape(-1)
        out = dict(scalars=scalars, h=h, actions=actd.clone(), safe_mask=masks[0], unsafe_mask=masks[1], hdot=hdot)
        if compute_acc_h_dot:                                            # gcbf.py:209 (M x M broadcast mean)
            out['acc_h_dot'] = self._acc_h_dot(red, hdot, h, M, dev)
        red.sum_(bucket.grad)                                            # the ONE gradient collective
        if apply_optim:
            self.optim_step()
        return out

    def _train_step(self, graphs, apply_optim: bool, compute_acc_h_dot: bool) -> Dict[str, Tensor]:
        env, hp = self._env, self.params
        bucket = self._ensure_bucket()
        dev = graphs.states.device
        red = self._reducer()
        world = red.world
        M = graphs.u_ref.shape[0]
        a_dim = self.action_dim

        # h and the actor's actions are independent: the actor's forward (and, through autograd's stream bookkeeping, its
        # backward) runs on a side stream so its kernels fill the CBF net's wave tails (GCBF_TWO_STREAMS=0 disables)
        side = self._side_stream(dev, int(graphs.edge_index.shape[1]))
        if side is not None:
            main = torch.cuda.current_stream(dev)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                actions = self.actor(graphs)                             # gcbf.py:162
            h = self.cbf(graphs)                                         # gcbf.py:161  (power iteration #1)
            main.wait_stream(side)
        else:
            h = self.cbf(graphs)                                         # gcbf.py:161  (power iteration #1)
            actions = self.actor(graphs)                                 # gcbf.py:162
        masks = env._masks(graphs)                                       # gcbf.py:168, 180 -- one launch
        graphs_next = env.forward_graph(graphs, actions)                 # gcbf.py:193
        if side is not None:
            inputs_ready = torch.cuda.Event()
            inputs_ready.record()                                        # actions / graphs_next exist from here on
        h_next = self.cbf(graphs_next)                                   # gcbf.py:194  (power iteration #2)
        # the re-linked graph's value-only pass (gcbf.py:195-201, batched) overlaps h_next's forward on the side stream; its
        # host sync (edge count) then waits for the side stream only, and ops.sn_power_iter_batched keeps power iteration #3
        # behind #2
        with torch.no_grad():
            if side is not None:
                side.wait_event(inputs_ready)
                with torch.cuda.stream(side):
                    st_relink = env.next_states_single(graphs, actions)
                    relinked = env.add_communication_links(env.make_graph(st_relink))
                    h_next_new = self.cbf(relinked)                      # power iteration #3, value only
                torch.cuda.current_stream(dev).wait_stream(side)
            else:
                st_relink = env.next_states_single(graphs, actions)
                relinked = env.add_communication_links(env.make_graph(st_relink))
                h_next_new = self.cbf(relinked)                          # power iteration #3, value only

        partial = torch.empty(16, device=dev, dtype=torch.float64)
        hdot = torch.empty(M, device=dev, dtype=torch.float32)
        hd, hnd, hnnd, actd = h.detach(), h_next.detach(), h_next_new, actions.detach()
        safe_u8, unsafe_u8 = masks[0].view(torch.uint8), masks[1].view(torch.uint8)
        dt = float(env.dt)
        _C.call('gcbf_loss_partials', _C.ptr(hd), _C.ptr(hnd), _C.ptr(hnnd), _C.ptr(actd), a_dim, _C.ptr(safe_u8),
                _C.ptr(unsafe_u8), M, float(hp['alpha']), float(hp['eps']), dt, _C.ptr(partial), _C.ptr(hdot))
        red.sum_(partial)                                                # global counts => global masked means
        d_h = torch.empty_like(hd)
        d_hn = torch.empty_like(hnd)
        d_act = torch.empty_like(actd)
        scalars = torch.empty(8, device=dev, dtype=torch.float32)
        _C.call('gcbf_loss_grads', _C.ptr(hd), _C.ptr(hnd), _C.ptr(hnnd), _C.ptr(actd), a_dim, _C.ptr(safe_u8),
                _C.ptr(unsafe_u8), M, float(hp['alpha']), float(hp['eps']), dt, float(hp['loss_unsafe_coef']),
                float(hp['loss_safe_coef']), float(hp['loss_h_dot_coef']), float(hp['loss_action_coef']),
                _C.ptr(partial), _C.ptr(d_h), _C.ptr(d_hn), _C.ptr(d_act), _C.ptr(scalars))

        bucket.zero_grad()                                               # gcbf.py:220-221
        ops.GRAD_INTO_PARAM = True     # weight-grad kernels accumulate straight into the bucket's .grad views
        try:
            torch.autograd.backward([h, h_next, actions], [d_h, d_hn, d_act])  # gcbf.py:222
        finally:
            ops.GRAD_INTO_PARAM = False
        if side is not None:
            # the actor's weight-grad kernels wrote into the bucket on the side stream and return no tensors to autograd, so
            # nothing else orders them before the all-reduce / clip+Adam below
            torch.cuda.current_stream(dev).wait_stream(side)

        # results leave the arena as private copies (tiny: O(num_agents))
        out = dict(scalars=scalars, h=hd.clone(), actions=actd.clone(), h_next=hnd.clone(), h_next_new=hnnd.clone(),
                   safe_mask=masks[0], unsafe_mask=masks[1], edge_index_new=relinked.edge_index, hdot=hdot)
        if compute_acc_h_dot:                                            # gcbf.py:209 (M x M broadcast mean)
            cnt = torch.empty(1, device=dev, dtype=torch.int64)
            sizes = red.sizes(M)                                         # ranks may own different numbers of agents
            hdot_all = red.gather_cat(hdot, sizes)
            _C.call('gcbf_pair_count', _C.ptr(hdot_all), hdot_all.numel(), _C.ptr(hd), M, float(hp['alpha']), _C.ptr(cnt))
            red.sum_(cnt)
            out['acc_h_dot'] = cnt.to(torch.float64) / float(sum(sizes)) / float(sum(sizes))

        red.sum_(bucket.grad)                                            # the ONE gradient collective (K9)
        if apply_optim:
            self.optim_step()
        return out

    # ---- the train step through the chain-level C ABI (csrc/step.cu): three calls, two collectives in between ----------------
    def _step_desc(self):
        """gcbf_step_desc of this algorithm: built once (parameter / gradient / companion pointers are stable: they are views
        into the flat bucket), the per-step fields are refreshed by the caller."""
        import ctypes
        from .. import native
        env, hp = self._env, self.params
        bucket = self._ensure_bucket()
        key = (id(env), id(env._goal), env._goal.data_ptr() if env._goal is not None else 0, bucket.flat.data_ptr(), self._matmul_mode())
        cached = getattr(self, '_native_desc', None)
        if cached is not None and cached[0] == key:
            return cached[1]
        cbf_layer, act_layer = self.cbf.feat_transformer.module_0, self.actor.feat_transformer.module_0
        cbf_spec, act_spec = cbf_layer.net_spec(self.cbf.feat_2_CBF), act_layer.net_spec(self.actor.feat_2_action)
        d = native.StepDesc()
        ctypes.memmove(ctypes.byref(d.cbf), ctypes.byref(native.make_net_desc(cbf_spec, 0, 'param')), ctypes.sizeof(native.NetDesc))
        ctypes.memmove(ctypes.byref(d.actor), ctypes.byref(native.make_net_desc(act_spec, self.action_dim, 'param')),
                       ctypes.sizeof(native.NetDesc))
        goal, ldg = ops._mat(env._goal)
        gain = env._gain()
        d.goal, d.lqr_gain, d.ld_goal = goal.data_ptr(), (gain.data_ptr() if gain is not None else None), ldg
        d.state_dim, d.pos_dim, d.action_dim = env.state_dim, env.POS_DIM, self.action_dim
        d.graph_metric, d.comm_radius = env.GRAPH_METRIC, float(env._params['comm_radius'])
        d.alpha, d.eps = float(hp['alpha']), float(hp['eps'])
        d.coef_unsafe, d.coef_safe = float(hp['loss_unsafe_coef']), float(hp['loss_safe_coef'])
        d.coef_hdot, d.coef_action = float(hp['loss_h_dot_coef']), float(hp['loss_action_coef'])
        d.grad_bucket, d.grad_bucket_floats = bucket.grad.data_ptr(), bucket.grad.numel()
        keep = (goal, gain, cbf_spec, act_spec)
        self._native_desc = (key, (d, keep, cbf_spec.all_layers(), act_spec.all_layers()))
        return self._native_desc[1]

    def _native_inputs(self, graphs):
        """(gcbf_step_desc, gcbf_step_batch, tensors the two point into, layer lists, M, E) for a batch of graphs: what every
        chain-level call of the library takes."""
        import ctypes
        from .. import native
        from ..nn.gnn import cached_rowptr
        env = self._env
        d, _keep, cbf_layers, act_layers = self._step_desc()
        ops.sync_gemm_impl()
        d.cbf.refresh_weights = 1 if native._weights_stale(cbf_layers) else 0
        d.actor.refresh_weights = 1 if native._weights_stale(act_layers) else 0
        B = env._num_graphs_of(graphs)
        cfg = env._cfg(B)
        ctypes.memmove(ctypes.byref(d.env), ctypes.byref(cfg), ctypes.sizeof(_C.EnvCfg))
        goal_pg = getattr(graphs, 'goal', None) if hasattr(graphs, 'goal') else None       # [B * n, goal_dim]: per-graph goal sets
        if goal_pg is not None:
            gpg, ldg = ops._mat(goal_pg.contiguous())
            d.goal, d.ld_goal, d.goal_per_graph = gpg.data_ptr(), ldg, 1
        else:
            gpg = None
            d.goal, d.ld_goal, d.goal_per_graph = _keep[0].data_ptr(), ops._mat(_keep[0])[1], 0
        st, ld = ops._mat(graphs.states.detach())
        x, ea, ei = graphs.x.contiguous(), graphs.edge_attr.detach().contiguous(), graphs.edge_index.contiguous()
        uref = graphs.u_ref.contiguous()
        rows = agent_row_index(graphs)
        rowptr = cached_rowptr(graphs.edge_index, x.shape[0])
        M, E = int(uref.shape[0]), int(ei.shape[1])
        b = native.StepBatch()
        b.states, b.ld_state, b.x = st.data_ptr(), ld, x.data_ptr()
        b.edge_attr, b.edge_index = (ea.data_ptr(), ei.data_ptr()) if E else (None, None)
        b.rowptr, b.u_ref, b.row_index = rowptr.data_ptr(), uref.data_ptr(), (rows.data_ptr() if rows is not None else None)
        b.num_edges, b.num_nodes, b.num_agents_total = E, int(x.shape[0]), M
        return d, b, (gpg, st, x, ea, ei, uref, rows, rowptr), cbf_layers, act_layers, M, E

    def _train_step_native(self, graphs, apply_optim: bool, compute_acc_h_dot: bool) -> Dict[str, Tensor]:
        import ctypes
        from .. import native
        bucket = self._ensure_bucket()
        red = self._reducer()
        dev = graphs.states.device
        d, b, _alive, cbf_layers, act_layers, M, E = self._native_inputs(graphs)
        bufs = getattr(self, '_native_ws', None)
        if bufs is None:
            bufs = self._native_ws = (native.GrowBuffer(), native.GrowBuffer())
        need = native.fn('gcbf_step_workspace_bytes')(ctypes.byref(d), ctypes.byref(b))
        if need == 0:
            native.check(-1, 'gcbf_step_workspace_bytes')
        ws = bufs[0].get(need, dev)
        ctx, out = native.StepCtx(), native.StepOut()
        main = _C.stream()
        side_t = self._side_stream(dev, E)
        side = side_t.cuda_stream if side_t is not None else None
        native.check(native.fn('gcbf_step_forward')(ctypes.byref(d), ctypes.byref(b), ws.data_ptr(), ws.numel(), ctypes.byref(ctx),
                                                   ctypes.byref(out), main, side), 'gcbf_step_forward')
        native._mark_fresh(cbf_layers)
        native._mark_fresh(act_layers)
        # the re-linked value pass: its workspace is sized for the previous step's edge count (+ head-room); the call reports the
        # exact need BEFORE launching anything, so a too small buffer costs one retry, not a wrong result
        needed = ctypes.c_size_t(0)
        ws2 = bufs[1].get(max(1, bufs[1].buf.numel() if bufs[1].buf is not None else need // 6), dev)
        rc = native.fn('gcbf_step_relink')(ctypes.byref(d), ctypes.byref(b), ctypes.byref(ctx), ws2.data_ptr(), ws2.numel(),
                                           ctypes.byref(needed), ctypes.byref(out), main, side)
        if rc == native.E_WORKSPACE:
            ws2 = bufs[1].get(needed.value, dev)
            rc = native.fn('gcbf_step_relink')(ctypes.byref(d), ctypes.byref(b), ctypes.byref(ctx), ws2.data_ptr(), ws2.numel(),
                                               ctypes.byref(needed), ctypes.byref(out), main, side)
        native.check(rc, 'gcbf_step_relink')
        partial = native.view(ws, out.partial, (16,), torch.float64)
        red.sum_(partial)                                                # global counts => global masked means
        a_dim = self.action_dim
        En = int(out.num_edges_new)
        res = dict(scalars=native.view(ws, out.scalars, (8,), torch.float32), h=native.view(ws, out.h, (M, 1), torch.float32),
                   actions=native.view(ws, out.actions, (M, a_dim), torch.float32), h_next=native.view(ws, out.h_next, (M, 1), torch.float32),
                   h_next_new=native.view(ws, out.h_next_new, (M,), torch.float32),
                   safe_mask=native.view(ws, out.safe, (M,), torch.uint8).view(torch.bool),
                   unsafe_mask=native.view(ws, out.unsafe, (M,), torch.uint8).view(torch.bool),
                   edge_index_new=(native.view(ws2, out.edge_index_new, (2, En), torch.int64) if En else
                                   torch.empty(2, 0, device=dev, dtype=torch.int64)),
                   hdot=native.view(ws, out.hdot, (M,), torch.float32))
        # data-parallel: everything that is not on the critical path of the backward goes to a communication stream -- the
        # h_dot gather + pair count of `acc/derivative` (needs only the forward's outputs) and the gradient all-reduces, each started
        # as soon as its range of the flat bucket is final (events recorded inside gcbf_step_backward)
        overlap = red.world > 1 and dev.type == 'cuda' and os.environ.get('GCBF_OVERLAP_COMM', '1') != '0'
        comm, events, ev_arr = None, None, None
        if overlap:
            comm, events = self._comm_resources(dev)
            ev_arr = (ctypes.c_void_p * 4)(*[e.cuda_event for e in events])
            comm.wait_stream(torch.cuda.current_stream(dev))             # partial sums reduced, h / h_dot final
            if compute_acc_h_dot:
                with torch.cuda.stream(comm):
                    res['acc_h_dot'] = self._acc_h_dot(red, res['hdot'], res['h'], M, dev)
        native.check(native.fn('gcbf_step_backward')(ctypes.byref(d), ctypes.byref(b), ctypes.byref(ctx), ctypes.byref(out), ev_arr, main, side),
                     'gcbf_step_backward')
        if overlap:
            (c_lo, c_hi), (a_lo, a_hi) = bucket.ranges
            c_tail, a_tail = bucket.tail_start
            with torch.cuda.stream(comm):
                for ev, lo, hi in ((events[0], c_tail, c_hi), (events[2], a_tail, a_hi), (events[1], c_lo, c_tail), (events[3], a_lo, a_tail)):
                    comm.wait_event(ev)
                    red.sum_(bucket.grad[lo:hi])
            torch.cuda.current_stream(dev).wait_stream(comm)
        else:
            if compute_acc_h_dot:                                        # gcbf.py:209 (M x M broadcast mean)
                res['acc_h_dot'] = self._acc_h_dot(red, res['hdot'], res['h'], M, dev)
            red.sum_(bucket.grad)                                        # the ONE gradient collective (K9)
        if apply_optim:
            self.optim_step()
        return res

    def _acc_h_dot(self, red, hdot, h, M: int, dev):
        """mean over all (i, j) of [h_dot_j + alpha h_i >= 0] (the M x M broadcast of gcbf.py:209) over the GLOBAL agent set: the
        per-rank h_dot vectors are gathered (unequal shards allowed), every rank counts its rows, the counts are summed."""
        cnt = torch.empty(1, device=dev, dtype=torch.int64)
        sizes = red.sizes(M)
        hdot_all = red.gather_cat(hdot, sizes)
        _C.call('gcbf_pair_count', _C.ptr(hdot_all), hdot_all.numel(), _C.ptr(h), M, float(self.params['alpha']), _C.ptr(cnt))
        red.sum_(cnt)
        return cnt.to(torch.float64) / float(sum(sizes)) / float(sum(sizes))

    def _comm_resources(self, dev):
        r = getattr(self, '_comm', None)
        if r is None or r[0].device != dev:
            comm = torch.cuda.Stream(device=dev)
            events = [torch.cuda.Event() for _ in range(4)]
            for e in events:
                e.record()                                               # materialise the cudaEvent_t handles
            r = self._comm = (comm, events)
        return r

    def optim_step(self):
        """clip_grad_norm_(1e-3) per net + Adam (gcbf.py:223-226), fused, on the flat bucket."""
        b = self._ensure_bucket()
        b.step += 1
        b.sumsq.zero_()
        ops.WEIGHT_EPOCH += 1                 # the kernel below rewrites the parameters: fp16 weight companions are stale
        from .. import native
        native.WEIGHT_EPOCH += 1
        for i, lr in enumerate((self.lr_cbf, self.lr_actor)):
            lo, hi = b.ranges[i]
            g = b.grad[lo:hi]
            _C.call('gcbf_grad_sumsq', _C.ptr(g), hi - lo, _C.ptr(b.sumsq[i:i + 1]))
            _C.call('gcbf_clip_adam', _C.ptr(b.flat[lo:hi]), _C.ptr(g), _C.ptr(b.exp_avg[lo:hi]),
                    _C.ptr(b.exp_avg_sq[lo:hi]), hi - lo, _C.ptr(b.sumsq[i:i + 1]), self.max_grad_norm, lr, 0.9, 0.999,
                    1e-8, b.step)

    def update(self, step: int, writer=None) -> dict:
        """Reference-shaped update loop (gcbf.py:144-247): sample segments, collate, `inner_iter` train steps."""
        seg_len = 3
        info = {}
        for i_inner in range(self.params['inner_iter']):
            if self.memory.size == 0:
                graph_list = self.buffer.sample(self.batch_size // 5, seg_len)
                parts = [(self.buffer, graph_list)]
            else:
                from_buffer = self.buffer.sample(self.batch_size // 10, seg_len, True)
                from_memory = self.memory.sample(self.batch_size // 5 - self.batch_size // 10, seg_len, True)
                graph_list = from_buffer + from_memory
                parts = [(self.buffer, from_buffer), (self.memory, from_memory)]
            if self.device_replay:
                from .device_buffer import collate
                batch = collate(self._env, parts)            # gathers on the device rings + ONE batched graph build
            else:
                batch = Batch.from_data_list(graph_list)
            res = self.train_step(batch)
            s = res['scalars'].tolist()                                  # the one host sync per inner iteration
            info = {'acc/safe': s[5], 'acc/unsafe': s[4], 'acc/derivative': float(res['acc_h_dot'])}
            if writer is not None:
                it = step * self.params['inner_iter'] + i_inner
                for tag, val in (('loss/unsafe', s[0]), ('loss/safe', s[1]), ('loss/derivative', s[2]),
                                 ('loss/action', s[3]), ('acc/unsafe', s[4]), ('acc/safe', s[5]),
                                 ('acc/derivative', info['acc/derivative'])):
                    writer.add_scalar(tag, val, it)
        self.memory.merge(self.buffer)
        self.buffer.clear()
        return info

    # ---- test-time controller (SURVEY section 8f-1) -------------------------------------------------------
    def apply(self, data, rand: Optional[float] = 30, max_iter: int = 30) -> Tensor:
        """Reference gcbf.py:260-309 for ONE graph: keep the actor's action only where the nominal (zero) action
        violates the h_dot condition, then up to max_iter+1 per-agent Adam(lr=0.1) steps on the violating agents'
        actions through forward_graph -> CBF (same kernels as training: K2, K3, K4, K5 forward and input-gradient),
        plus the reference's gradient noise `rand * lr * randn * grad`.  The per-agent optimisers are kept as one
        vectorised state (m, v, step count per agent); the O(num_agents) arithmetic around the kernels is host glue."""
        self._matmul_mode()
        if ops.NATIVE and data.states.is_cuda:
            return self._apply_native(data, rand, max_iter, None, batched=False)
        return self._apply_python(data, rand, max_iter, None)

    def apply_batch(self, batch, rand: Optional[float] = 30, max_iter: int = 30, noise: Optional[Tensor] = None) -> Tensor:
        """`apply` for every graph of a collated batch of B graphs (with `u_ref`; optional per-graph goal sets in `batch.goal`
        [B * n, goal_dim]) in one call: graph g gets exactly what `apply` on graph g alone gives -- its own termination, its own
        per-agent Adam state, the mean of its loss over its own agents.  Returns the actions [B * n, action_dim]; the Adam rounds each
        graph did go to `self.last_apply_batch_rounds` (host int tensor [B]).  noise: the standard normals of the gradient noise
        [(max_iter + 1), B * n, action_dim] (default: drawn here); round k of graph g reads its rows of slice k, so concatenated
        per-graph draws reproduce per-graph calls."""
        self._matmul_mode()
        if ops.NATIVE and batch.states.is_cuda:
            return self._apply_native(batch, rand, max_iter, noise, batched=True)
        return self._apply_python(batch, rand, max_iter, noise)

    def _apply_python(self, data, rand: Optional[float], max_iter: int, noise: Optional[Tensor]) -> Tensor:
        """The Python-sequenced controller (autograd over the per-kernel ops) for B >= 1 graphs: per-graph done flags and loss means,
        per-agent Adam state."""
        env, alpha, lr = self._env, float(self.params['alpha']), 0.1
        dt = float(env.dt)
        B, n = env._num_graphs_of(data), env.num_agents
        goal = getattr(data, 'goal', None) if hasattr(data, 'goal') else None
        with torch.no_grad():
            h = self.cbf(data)
            action = self.actor(data)
            nominal = torch.zeros_like(action)
            h_next = self.cbf(env.forward_graph(data, nominal, single=True, goal=goal))
            viol = torch.relu(-(h_next - h) / dt - alpha * h).reshape(-1)
            act = torch.where((viol <= 0).unsqueeze(1), nominal, action).clone()
        m, v = torch.zeros_like(act), torch.zeros_like(act)
        t = torch.zeros(act.shape[0], device=act.device)
        if rand and noise is None:
            noise = torch.randn(max_iter + 1, *act.shape, device=act.device)     # one draw, like the library path
        done = torch.zeros(B, dtype=torch.bool, device=act.device)
        rounds = torch.zeros(B, dtype=torch.int64)
        it = 0
        while True:
            a = act.clone().requires_grad_(True)
            h_next = self.cbf(env.forward_graph(data, a, single=True, goal=goal))
            max_val = torch.relu(-(h_next - h) / dt - alpha * h).reshape(B, n)
            max_val = torch.where(done.unsqueeze(1), torch.zeros_like(max_val), max_val)   # a done graph is not re-evaluated
            loss = max_val.mean(dim=1)                                                       # per graph: mean over its agents
            finished = ~done & ((loss.detach() <= 0) | (it > max_iter))
            rounds[finished.cpu()] = it
            done = done | finished
            if bool(done.all()):
                self.last_apply_batch_rounds = rounds
                self.last_apply_rounds = int(rounds.max())
                return a.detach()
            sel = (max_val.detach().reshape(-1) != 0)
            ops.SKIP_WGRAD = True           # only d loss / d action is needed: skip every weight-gradient GEMM
            try:
                (g,) = torch.autograd.grad(loss.sum(), a)                    # graphs are independent: d sum_g loss_g / d a_g = d loss_g / d a_g
            finally:
                ops.SKIP_WGRAD = False
            with torch.no_grad():
                s2 = sel.unsqueeze(1)
                t = torch.where(sel, t + 1, t)
                m = torch.where(s2, m + (g - m) * (1 - 0.9), m)
                v = torch.where(s2, v * 0.999 + (1 - 0.999) * g * g, v)
                bc1 = (1 - 0.9 ** t).clamp(min=1e-30).unsqueeze(1)
                bc2 = (1 - 0.999 ** t).clamp(min=1e-30).unsqueeze(1)
                act = torch.where(s2, act - (lr / bc1) * m / (v.sqrt() / bc2.sqrt() + 1e-8), act)
                if rand:
                    act = torch.where(s2, act - rand * lr * noise[it] * g, act)
            it += 1

    def _apply_native(self, data, rand: Optional[float], max_iter: int, noise: Optional[Tensor], batched: bool) -> Tensor:
        """The same controller as ONE library call (gcbf_apply / gcbf_apply_batch, csrc/apply.cu): the whole refinement loop, the
        per-agent Adam kernel and the termination test run inside the library; this method only draws the noise and hands over
        pointers."""
        import ctypes
        from .. import native
        dev = data.states.device
        d, b, _alive, cbf_layers, act_layers, M, E = self._native_inputs(data)
        a = self.action_dim
        name = 'gcbf_apply_batch' if batched else 'gcbf_apply'
        need = native.fn(name + '_workspace_bytes')(ctypes.byref(d), ctypes.byref(b))
        if need == 0:
            native.check(-1, name + '_workspace_bytes')
        buf = getattr(self, '_apply_ws', None)
        if buf is None:
            buf = self._apply_ws = native.GrowBuffer()
        ws = buf.get(need, dev)
        rand = float(rand) if rand else 0.0
        if rand and noise is None:
            noise = torch.randn(max_iter + 1, M, a, device=dev)      # gcbf.py:305 draws randn_like per agent and round
        if noise is not None:
            if tuple(noise.shape) != (max_iter + 1, M, a):
                raise ValueError(f'noise must be [{max_iter + 1}, {M}, {a}], got {tuple(noise.shape)}')
            noise = noise.to(dev, torch.float32).contiguous()
        action = torch.empty(M, a, device=dev)
        rounds = ctypes.c_int(0)
        graph_rounds = torch.empty(d.env.num_graphs, device=dev, dtype=torch.int32) if batched else None
        # the library captures a round into CUDA graphs and replays it; capture is impossible on the legacy default stream, so the call
        # runs on a stream of its own, ordered after and before the caller's stream
        cur = torch.cuda.current_stream(dev)
        st = getattr(self, '_apply_stream', None)
        if st is None or st.device != dev:
            st = self._apply_stream = torch.cuda.Stream(dev)
        st.wait_stream(cur)
        noise_ptr = noise.data_ptr() if (rand and noise is not None) else None
        with torch.cuda.stream(st):
            if batched:
                rc = native.fn(name)(ctypes.byref(d), ctypes.byref(b), 0.1, rand, noise_ptr, int(max_iter), action.data_ptr(), a,
                                     graph_rounds.data_ptr(), ctypes.byref(rounds), ws.data_ptr(), ws.numel(), st.cuda_stream)
            else:
                rc = native.fn(name)(ctypes.byref(d), ctypes.byref(b), 0.1, rand, noise_ptr, int(max_iter), action.data_ptr(), a,
                                     ctypes.byref(rounds), ws.data_ptr(), ws.numel(), st.cuda_stream)
        cur.wait_stream(st)
        native.check(rc, name)
        native._mark_fresh(cbf_layers)
        native._mark_fresh(act_layers)
        self.last_apply_rounds = rounds.value
        if batched:
            self.last_apply_batch_rounds = graph_rounds.cpu().to(torch.int64)
        return action

    # ---- analytic h_dot (SURVEY section 8f-3; the training loss uses it when params['h_dot'] = 'analytic') --------------------------
    def h_dot_analytic(self, data, action: Optional[Tensor] = None, freeze: Optional[bool] = None):
        """(h, h_dot) with h_dot_i = sum_k dh_i/ds_k . f(s_k, clamp(u_k + u_ref)) as one forward-mode pass (gcbf_b200/jvp.py): the
        derivative the finite difference (h(x + dt f) - h(x)) / dt of gcbf.py:193-207 approximates, edges held fixed.  action: the
        policy's correction (default: the actor's).  The CBF condition of the paper is h_dot + alpha h >= 0."""
        from .. import jvp
        self._refuse_fp16('h_dot_analytic')
        if action is None:
            action = self.act(data)
        return jvp.cbf_value_and_h_dot(self.cbf, self._env, data, action, freeze)

    # ---- CBF level-set field (the data of plot_cbf.py / plot_cbf_contour, gcbf/trainer/utils.py:226-298) ----------------------------
    FIELD_MAX_PROBES = 65536            # default probe bound of one chunk
    FIELD_MAX_EDGES = 262144            # default probe-edge bound of one chunk (7 GB of workspace at C3 with the 2048-wide phi)

    @staticmethod
    def field_grid(lims, x_dim: int, y_dim: int, n_mesh: int):
        """The grid axes of plot_cbf_contour (utils.py:259-262): np.linspace over the limits' own dtype (float32 box ->
        float32 axes), as the reference computes them."""
        lo, hi = lims
        val = lambda v: v.cpu() if isinstance(v, Tensor) else v
        xs = np.linspace(val(lo[x_dim]), val(hi[x_dim]), n_mesh)
        ys = np.linspace(val(lo[y_dim]), val(hi[y_dim]), n_mesh)
        return xs, ys

    def cbf_field(self, data, agents=0, x_dim: int = 0, y_dim: int = 1, n_mesh: int = 30, lims=None, relink: bool = False,
                  max_probes: Optional[int] = None, max_edges: Optional[int] = None):
        """h of the given agents over an n_mesh x n_mesh grid of state dimensions (x_dim, y_dim), everyone else fixed: what
        plot_cbf_contour draws (gcbf/trainer/utils.py:259-273), for every graph of `data` (one graph or a Batch of equally sized
        graphs, e.g. every step of an episode) and every agent in `agents` (an id or a list of ids) in ONE library call.

        Returns (xs [n_mesh], ys [n_mesh], h [B, A, n_mesh, n_mesh]) with h[b, k, i, j] = h of agent agents[k] of graph b at
        state[x_dim] = xs[j], state[y_dim] = ys[i] (np.meshgrid 'xy' order, as the reference's `H[i, j]`).  xs, ys are the numpy
        axes of np.linspace over `lims` ((low, high), default env.state_lim); the states get their fp32 roundings.
        relink=False keeps the given edge_index (the reference's plot); relink=True re-links the moved agent to every node inside
        the communication radius, as add_communication_links would (neighbours enter and leave as it moves).  Like the reference's
        single cbf(plot_data) call, a call advances the CBF's spectral-norm vectors by ONE power iteration, however many chunks of
        at most max_probes probes / max_edges probe edges it runs in (gcbf_cbf_field, csrc/field.cu); one host sync per call.
        The chunk count and the probe edges go to self.last_field_chunks / self.last_field_edges.  The workspace is sized for the
        call's largest chunk: at most max_probes probes with at most nodes_per_graph - 1 edges each, and at most max_edges edges."""
        import ctypes
        from .. import native
        self._matmul_mode()
        d, keep, xs, ys, B, A, T = self._field_desc(data, agents, x_dim, y_dim, n_mesh, lims, relink, max_probes, max_edges)
        layers = keep[-1]
        dev = data.states.device
        need = native.fn('gcbf_cbf_field_workspace_bytes')(ctypes.byref(d))
        if need == 0:
            native.check(-1, 'gcbf_cbf_field_workspace_bytes')
        ws = native.workspace(need, dev)
        h = torch.empty(T, device=dev, dtype=torch.float32)
        info = (ctypes.c_int64 * 2)()
        native.check(native.fn('gcbf_cbf_field')(ctypes.byref(d), h.data_ptr(), info, ws.data_ptr(), ws.numel(), _C.stream()), 'gcbf_cbf_field')
        native._mark_fresh(layers)
        self.last_field_chunks, self.last_field_edges = int(info[0]), int(info[1])
        return xs, ys, h.view(B, A, n_mesh, n_mesh)

    def cbf_field_probe_graph(self, data, agents=0, x_dim: int = 0, y_dim: int = 1, n_mesh: int = 30, lims=None, relink: bool = False):
        """The probe graphs cbf_field feeds the CBF (gcbf_cbf_field_probe_count / _fill), for inspection: (edge_index [2, E],
        edge_attr [E, edge_dim]) with target = the probe id t = ((b * A + k) * n_mesh + i) * n_mesh + j (agent agents[k] of graph b at
        (xs[j], ys[i])) and source = the node id in `data`, sorted (t asc, source asc); edge_attr = g(s_source) - g(s'_t).  Same
        arguments as cbf_field; the CBF is not evaluated (u, v unchanged).  One host sync (the edge count)."""
        from .. import native
        import ctypes
        d, keep, xs, ys, B, A, T = self._field_desc(data, agents, x_dim, y_dim, n_mesh, lims, relink, None, None)
        dev = data.states.device
        rowptr = torch.empty(T + 1, device=dev, dtype=torch.int32)
        native.check(native.fn('gcbf_cbf_field_probe_count')(ctypes.byref(d), rowptr.data_ptr(), _C.stream()), 'gcbf_cbf_field_probe_count')
        E = int(rowptr[-1].item())
        ei = torch.empty(2, E, device=dev, dtype=torch.int64)
        ea = torch.empty(E, self._env.edge_dim, device=dev, dtype=torch.float32)
        native.check(native.fn('gcbf_cbf_field_probe_fill')(ctypes.byref(d), rowptr.data_ptr(), ei.data_ptr() if E else None, E,
                                                            ea.data_ptr() if E else None, _C.stream()), 'gcbf_cbf_field_probe_fill')
        return ei, ea

    # ---- CBF-condition field: where the learned controller keeps h_dot + alpha h >= 0 ---------------------------------------------
    COND_MAX_PROBES = 65536             # default probe bound of one chunk
    COND_MAX_EDGES = 262144             # default two-hop edge bound of one chunk (actor and CBF passes over at most this many edges)

    def cbf_condition_field(self, data, agents=0, x_dim: int = 0, y_dim: int = 1, n_mesh: int = 30, lims=None, relink: bool = False,
                            max_probes: Optional[int] = None, max_edges: Optional[int] = None):
        """h and h_dot of the given agents over the grid of cbf_field, under the learned controller: for graph b, agent a = agents[k]
        and grid point (i, j), G' is graph b alone with s_a[x_dim] = xs[j], s_a[y_dim] = ys[i] (edges kept with edge_attr recomputed,
        or with relink=True the radius graph of the moved states), u = actor(G') with u_ref(G') as its head input, x_dot = f(s,
        clamp(u + u_ref)) with the single-graph reach-freeze, and (h, h_dot) = h_dot_analytic(G', u, freeze=True) at row a: h_dot with
        the edges of G' held fixed.  Goals: data.goal of graph b if present, else env._goal.  The CBF condition h_dot + alpha h >= 0
        certifies safety where it holds.

        Returns (xs, ys, h, h_dot), the fields [B, A, n_mesh, n_mesh] in cbf_field's index order.  Instead of n_mesh^2 copies per agent,
        each grid point is a two-hop probe graph (gcbf_cbf_condition_probe_count / _fill, csrc/condition.cu): the moved agent a' and
        one row j' per agent neighbour j, whose actions the derivative needs.  A call advances the spectral-norm vectors of the actor and
        of the CBF by ONE power iteration each and uses that 1/sigma in every chunk of at most max_probes probes / max_edges two-hop
        edges; one host sync per call (the per-probe counts).  The chunk count and the two-hop edges go to self.last_field_chunks /
        self.last_field_edges."""
        self._refuse_fp16('cbf_condition_field')
        d, keep, xs, ys, B, A, T, plan = self._condition_plan(data, agents, x_dim, y_dim, n_mesh, lims, relink, max_probes, max_edges)
        from .. import jvp
        env = self._env
        dev = data.states.device
        actor_spec = self.actor.feat_transformer.module_0.net_spec(self.actor.feat_2_action)
        cbf_spec = self.cbf.feat_transformer.module_0.net_spec(self.cbf.feat_2_CBF)
        h = torch.empty(T, device=dev, dtype=torch.float32)
        h_dot = torch.empty(T, device=dev, dtype=torch.float32)
        edges = 0
        with torch.no_grad():
            sig_actor = ops.sn_power_iter_batched(actor_spec.all_layers())     # ONE power iteration per net for the whole call
            sig_cbf = ops.sn_power_iter_batched(cbf_spec.all_layers())
            for t0, t1, Ea, Rc, Ec, off in plan['chunks']:
                ck = self._condition_fill(d, keep, plan, t0, t1, Rc, Ec, off, rows=False)
                xb, st, gl, ei, ea, NN = ck['x'], ck['states'], ck['goal'], ck['edge_index'], ck['edge_attr'], ck['num_rows']
                rowptr = ops.rowptr_from_edge_index(ei, NN, check_sorted=False)
                rows = torch.arange(Rc, device=dev, dtype=torch.int64)
                # per-row closed loop: every a' / j' row is a graph of one agent with its own goal (bit for bit the per-graph kernels)
                cfg1 = self._row_cfg(Rc, 1)
                uref = torch.empty(Rc, env.action_dim, device=dev, dtype=torch.float32)
                _C.call('gcbf_u_ref_multi', ctypes.byref(cfg1), _C.ptr(st), env.state_dim, _C.ptr(gl), plan['goal_dim'],
                        _C.ptr(env._gain()), _C.ptr(uref))
                u, _ = ops.net_forward(actor_spec, xb, ea, ei, rowptr, rows, uref, False, sigma=sig_actor)
                sdot = torch.empty(NN, env.state_dim, device=dev, dtype=torch.float32)
                _C.call('gcbf_state_dot', ctypes.byref(cfg1), _C.ptr(st), env.state_dim, _C.ptr(u), _C.ptr(uref), _C.ptr(gl),
                        plan['goal_dim'], 1, 1, _C.ptr(sdot), env.state_dim)
                # the original rows are read as obstacle sources of a' only: x_dot of a node without an action
                cfg0 = self._row_cfg(B, 0)
                _C.call('gcbf_state_dot', ctypes.byref(cfg0), _C.ptr(st[Rc:]), env.state_dim, None, None, None, 0, 0, 0,
                        _C.ptr(sdot[Rc:]), env.state_dim)
                # the CBF over the a' rows and their edges (the first Ea: edges are target-sorted, a' rows first)
                ei_a = ei[:, :Ea].contiguous()
                rowptr_a = ops.rowptr_from_edge_index(ei_a, NN, check_sorted=False)
                h_c, ctx = ops.net_forward(cbf_spec, xb, ea[:Ea], ei_a, rowptr_a, rows[:t1 - t0], None, True, sigma=sig_cbf)
                t_ea = jvp.edge_attr_tangent(env, st, sdot, ei_a)
                hd_c = jvp.net_tangent(cbf_spec, ctx, t_ea, rowptr_a, rows[:t1 - t0])
                h[t0:t1].copy_(h_c.view(-1))
                h_dot[t0:t1].copy_(hd_c.view(-1))
                edges += Ec
        self.last_field_chunks, self.last_field_edges = len(plan['chunks']), edges
        shape = (B, A, int(n_mesh), int(n_mesh))
        return xs, ys, h.view(shape), h_dot.view(shape)

    def cbf_condition_field_probe_graph(self, data, agents=0, x_dim: int = 0, y_dim: int = 1, n_mesh: int = 30, lims=None,
                                        relink: bool = False) -> dict:
        """The two-hop probe graphs cbf_condition_field feeds the nets, all probes as one chunk, for inspection: 'rows' [R, 3] int64 =
        (kind 0 a' / 1 j', node id in `data`, probe id) of the probe rows, 'edge_index' [2, E] over rows (a source >= R is the original
        node source - R), target-sorted with the a' rows first, 'edge_attr' [E, edge_dim] = g(s_src) - g(s_tgt) in G', 'states' [R,
        state_dim] and 'goal' [R, goal_dim] of the rows.  Same arguments as cbf_condition_field; no net is evaluated (u, v unchanged)."""
        d, keep, xs, ys, B, A, T, plan = self._condition_plan(data, agents, x_dim, y_dim, n_mesh, lims, relink, None, None,
                                                              one_chunk=True)
        t0, t1, Ea, Rc, Ec, off = plan['chunks'][0]
        ck = self._condition_fill(d, keep, plan, t0, t1, Rc, Ec, off, rows=True)
        return dict(rows=ck['rows'], edge_index=ck['edge_index'], edge_attr=ck['edge_attr'], states=ck['states'][:Rc],
                    goal=ck['goal'], num_moved_edges=Ea)

    def _row_cfg(self, num_graphs: int, num_agents: int):
        """gcbf_env_cfg of num_graphs graphs of max(num_agents, 1) nodes: the per-row closed loop of the condition field."""
        cfg = self._env._cfg(num_graphs)
        if num_agents == 1:
            cfg.nodes_per_graph, cfg.num_agents = 1, 1
        else:
            cfg.num_agents = 0
        return cfg

    def _condition_plan(self, data, agents, x_dim, y_dim, n_mesh, lims, relink, max_probes, max_edges, one_chunk: bool = False):
        """Argument checks (all before any launch), the per-probe counts (the call's one host sync) and the chunks: (desc, tensors it
        points into, xs, ys, B, A, T, plan)."""
        if max_probes is not None and int(max_probes) < 1:
            raise ValueError(f'max_probes must be >= 1, got {max_probes}')
        if max_edges is not None and not 1 <= int(max_edges) < 2 ** 31:
            raise ValueError(f'max_edges must be in [1, 2^31), got {max_edges}')
        d, keep, xs, ys, B, A, T = self._field_desc(data, agents, x_dim, y_dim, n_mesh, lims, relink, None, None)
        env = self._env
        dev = data.states.device
        goal_pg = getattr(data, 'goal', None) if hasattr(data, 'goal') else None
        goals = (goal_pg if goal_pg is not None else env._goal)
        if goals is None:
            raise RuntimeError('cbf_condition_field needs the goals (data.goal or env._goal: reset() or set_goal() first)')
        goals = goals.detach().to(dev, torch.float32).contiguous()
        gd = min(int(goals.shape[1]), 6)
        counts = torch.empty(3, T, device=dev, dtype=torch.int32)
        _C.call('gcbf_cbf_condition_probe_count', ctypes.byref(d), _C.ptr(counts))
        c = counts.cpu().numpy().astype(np.int64)                      # the call's one host sync
        ea, nj, ej = c[0], c[1], c[2]
        e_all = ea + ej
        BN = B * env.nodes_per_graph
        P = T if one_chunk else min(T, int(max_probes) if max_probes is not None else self.COND_MAX_PROBES)
        Emax = 2 ** 31 - 1 if one_chunk else (int(max_edges) if max_edges is not None else self.COND_MAX_EDGES)
        big = int(e_all.max()) if T else 0
        if big > Emax:
            raise ValueError(f'a probe has {big} two-hop edges > max_edges {Emax}')
        cum = np.concatenate([[0], np.cumsum(e_all)])
        chunks, offs = [], []
        t0, pos = 0, 0
        while t0 < T:
            t1 = min(t0 + P, int(np.searchsorted(cum, cum[t0] + Emax, side='right')) - 1)
            sl = slice(t0, t1)
            Ea, Rc = int(ea[sl].sum()), (t1 - t0) + int(nj[sl].sum())
            Ec = Ea + int(ej[sl].sum())
            if Ec >= 2 ** 31 or Rc + BN >= 2 ** 31:
                raise ValueError(f'probes [{t0}, {t1}): {Rc} rows / {Ec} edges overflow int32; lower max_probes / max_edges')
            excl = lambda v, start: start + np.concatenate([[0], np.cumsum(v)[:-1]])
            offs.append(np.concatenate([excl(ea[sl], 0), excl(nj[sl], t1 - t0), excl(ej[sl], Ea)]))
            chunks.append((t0, t1, Ea, Rc, Ec, (pos, 3 * (t1 - t0))))
            pos += 3 * (t1 - t0)
            t0 = t1
        host = torch.from_numpy(np.concatenate(offs).astype(np.int32))
        if torch.cuda.is_available():
            host = host.pin_memory()
        off_dev = host.to(dev, non_blocking=True)                       # every chunk's offsets in one copy, no second sync
        plan = dict(chunks=chunks, offsets=off_dev, goals=goals, goal_dim=gd, goal_per_graph=goal_pg is not None, BN=BN,
                    counts=counts)
        return d, keep, xs, ys, B, A, T, plan

    def _condition_fill(self, d, keep, plan, t0, t1, Rc, Ec, off, rows: bool) -> dict:
        """Rows [0, Rc) and the Ec edges of probes [t0, t1), followed by the original rows (gcbf_cbf_condition_probe_fill)."""
        env = self._env
        st0, x0 = keep[0], keep[1]
        dev = x0.device
        BN, gd, goals = plan['BN'], plan['goal_dim'], plan['goals']
        NN = Rc + BN
        nd, sd = int(x0.shape[1]), env.state_dim
        xb = torch.empty(NN, nd, device=dev, dtype=torch.float32)
        xb[Rc:].copy_(x0)
        st = torch.empty(NN, sd, device=dev, dtype=torch.float32)
        st[Rc:].copy_(st0[:, :sd])
        gl = torch.empty(Rc, gd, device=dev, dtype=torch.float32)
        rw = torch.empty(Rc, 3, device=dev, dtype=torch.int64) if rows else None
        ei = torch.empty(2, Ec, device=dev, dtype=torch.int64)
        ea = torch.empty(Ec, env.edge_dim, device=dev, dtype=torch.float32)
        o0, _ = off
        offp = plan['offsets'].data_ptr() + 4 * o0
        _C.call('gcbf_cbf_condition_probe_fill', ctypes.byref(d), _C.ptr(goals), int(goals.shape[1]), gd, 1 if plan['goal_per_graph'] else 0,
                t0, t1 - t0, offp, Rc, _C.ptr(xb), _C.ptr(st), _C.ptr(gl), _C.ptr(rw), _C.ptr(ei) if Ec else None, Ec,
                _C.ptr(ea) if Ec else None)
        return dict(x=xb, states=st, goal=gl, rows=rw, edge_index=ei, edge_attr=ea, num_rows=NN)

    def _field_desc(self, data, agents, x_dim, y_dim, n_mesh, lims, relink, max_probes, max_edges):
        """Argument checks (all before any launch) and the gcbf_field_desc of a field call: (desc, tensors it points into + the CBF's
        layer list, xs, ys, B, A, T)."""
        import ctypes
        from .. import native
        from ..nn.gnn import cached_rowptr
        if not isinstance(self.cbf, CBFGNN):
            raise NotImplementedError(f'cbf_field needs a per-agent CBF (CBFGNN); {type(self).__name__} has a per-edge CBF')
        env = self._env
        n, sd = env.num_agents, env.state_dim
        ids = [agents] if isinstance(agents, (int, np.integer)) else list(agents)
        if not ids or any(not isinstance(a, (int, np.integer)) or not 0 <= int(a) < n for a in ids):
            raise ValueError(f'agents must be ids in [0, {n}), got {agents!r}')
        ids = [int(a) for a in ids]
        for name, d in (('x_dim', x_dim), ('y_dim', y_dim)):
            if not isinstance(d, (int, np.integer)) or not 0 <= int(d) < sd:
                raise ValueError(f'{name} must be in [0, {sd}), got {d!r}')
        if x_dim == y_dim:
            raise ValueError(f'x_dim and y_dim must differ, got {x_dim} twice')
        if not isinstance(n_mesh, (int, np.integer)) or n_mesh < 2:
            raise ValueError(f'n_mesh must be an integer >= 2, got {n_mesh!r}')
        if max_probes is not None and int(max_probes) < 1:
            raise ValueError(f'max_probes must be >= 1, got {max_probes}')
        for t in (data.states, data.x) + (() if relink else (data.edge_index,)):
            if not (isinstance(t, Tensor) and t.is_cuda):
                raise RuntimeError('cbf_field needs CUDA tensors (states, x[, edge_index]): there is no CPU fallback')
        B = env._num_graphs_of(data)
        N = env.nodes_per_graph
        xs, ys = self.field_grid(env.state_lim if lims is None else lims, int(x_dim), int(y_dim), int(n_mesh))
        dev = data.states.device
        T = B * len(ids) * n_mesh * n_mesh
        probes = min(T, int(max_probes) if max_probes is not None else self.FIELD_MAX_PROBES)
        edge_cap = int(max_edges) if max_edges is not None else max(self.FIELD_MAX_EDGES, N - 1)
        if edge_cap < N - 1:
            raise ValueError(f'max_edges must be >= nodes_per_graph - 1 = {N - 1} (the edges one probe can have), got {edge_cap}')

        ops.sync_gemm_impl()
        spec = self.cbf.feat_transformer.module_0.net_spec(self.cbf.feat_2_CBF)
        layers = spec.all_layers()
        d = native.FieldDesc()
        ctypes.memmove(ctypes.byref(d.cbf), ctypes.byref(native.make_net_desc(spec, 0, None)), ctypes.sizeof(native.NetDesc))
        d.cbf.refresh_weights = 1 if native._weights_stale(layers) else 0
        ctypes.memmove(ctypes.byref(d.env), ctypes.byref(env._cfg(B)), ctypes.sizeof(_C.EnvCfg))
        st, ld = ops._mat(data.states.detach())
        x = data.x.detach().contiguous()
        if relink:                                       # the given edges are not read
            ei, rowptr, E = None, None, 0
        else:
            ei = data.edge_index.contiguous()
            E = int(ei.shape[1])
            rowptr = cached_rowptr(data.edge_index, int(x.shape[0]))
        agents_t = torch.tensor(ids, device=dev, dtype=torch.int32)
        xs_t = torch.from_numpy(np.asarray(xs, dtype=np.float32)).to(dev)
        ys_t = torch.from_numpy(np.asarray(ys, dtype=np.float32)).to(dev)
        d.states, d.x, d.num_edges = st.data_ptr(), x.data_ptr(), E
        d.edge_index, d.rowptr = (ei.data_ptr() if E else None), (rowptr.data_ptr() if rowptr is not None else None)
        d.agents, d.xs, d.ys = agents_t.data_ptr(), xs_t.data_ptr(), ys_t.data_ptr()
        d.max_edges, d.max_probes = edge_cap, probes
        d.ld_state, d.state_dim, d.pos_dim, d.graph_metric = ld, sd, env.POS_DIM, env.GRAPH_METRIC
        d.comm_radius, d.relink = float(env._params['comm_radius']), 1 if relink else 0
        d.num_probe_agents, d.x_dim, d.y_dim, d.nx, d.ny = len(ids), int(x_dim), int(y_dim), int(n_mesh), int(n_mesh)
        return d, (st, x, ei, rowptr, agents_t, xs_t, ys_t, layers), xs, ys, B, len(ids), T

    # ---- checkpoints (file names and keys of gcbf.py:249-258) ------------------------------------------
    def save(self, save_dir: str):
        os.makedirs(save_dir, exist_ok=True)
        # parameters are views into the flat bucket: clone them, or each file would serialise the whole bucket storage
        for mod, name in ((self.cbf, 'cbf.pkl'), (self.actor, 'actor.pkl')):
            torch.save({k: v.detach().clone() for k, v in mod.state_dict().items()}, os.path.join(save_dir, name))

    def load(self, load_dir: str):
        assert os.path.exists(load_dir)
        self.cbf.load_state_dict(torch.load(os.path.join(load_dir, 'cbf.pkl'), map_location=self.device))
        self.actor.load_state_dict(torch.load(os.path.join(load_dir, 'actor.pkl'), map_location=self.device))
