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
import os
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

    def _build_networks(self, num_agents: int, node_dim: int, edge_dim: int, action_dim: int, device):
        # models: same construction order as the reference (gcbf.py:87-100) => same seeded initialisation
        self.cbf = CBFGNN(num_agents=num_agents, node_dim=node_dim, edge_dim=edge_dim, phi_dim=256).to(device)
        self.actor = GNNController(num_agents=num_agents, node_dim=node_dim, edge_dim=edge_dim, phi_dim=256,
                                   action_dim=action_dim).to(device)

    # ---- rollout-time API ---------------------------------------------------------------------------
    @torch.no_grad()
    def act(self, data) -> Tensor:
        return self.actor(data)

    @torch.no_grad()
    def step(self, data, prob: float) -> Tensor:
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
        workspace: valid until the next train_step of this object)."""
        if ops.NATIVE:
            return self._train_step_native(graphs, apply_optim, compute_acc_h_dot)
        from ..arena import ARENA
        ARENA.begin(graphs.states.device)      # every activation / gradient below is a view into the step arena
        try:
            return self._train_step(graphs, apply_optim, compute_acc_h_dot)
        finally:
            ARENA.end()

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
        key = (id(env), id(env._goal), env._goal.data_ptr() if env._goal is not None else 0, bucket.flat.data_ptr())
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
        if ops.NATIVE and data.states.is_cuda:
            return self._apply_native(data, rand, max_iter)
        env, alpha, lr = self._env, float(self.params['alpha']), 0.1
        dt = float(env.dt)
        with torch.no_grad():
            h = self.cbf(data)
            action = self.actor(data)
            nominal = torch.zeros_like(action)
            h_next = self.cbf(env.forward_graph(data, nominal))
            viol = torch.relu(-(h_next - h) / dt - alpha * h).reshape(-1)
            act = torch.where((viol <= 0).unsqueeze(1), nominal, action).clone()
        m, v = torch.zeros_like(act), torch.zeros_like(act)
        t = torch.zeros(act.shape[0], device=act.device)
        noise = torch.randn(max_iter + 1, *act.shape, device=act.device) if rand else None     # one draw, like the library path
        it = 0
        while True:
            a = act.clone().requires_grad_(True)
            h_next = self.cbf(env.forward_graph(data, a))
            max_val = torch.relu(-(h_next - h) / dt - alpha * h)
            loss = torch.mean(max_val)
            if float(loss.detach()) <= 0 or it > max_iter:
                return a.detach()
            sel = (max_val.detach().reshape(-1) != 0)
            ops.SKIP_WGRAD = True           # only d loss / d action is needed: skip every weight-gradient GEMM
            try:
                (g,) = torch.autograd.grad(loss, a)
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

    def _apply_native(self, data, rand: Optional[float], max_iter: int) -> Tensor:
        """The same controller as ONE library call (gcbf_apply, csrc/apply.cu): the whole refinement loop, the per-agent Adam
        kernel and the termination test run inside the library; this method only draws the noise and hands over pointers."""
        import ctypes
        from .. import native
        dev = data.states.device
        d, b, _alive, cbf_layers, act_layers, M, E = self._native_inputs(data)
        a = self.action_dim
        need = native.fn('gcbf_apply_workspace_bytes')(ctypes.byref(d), ctypes.byref(b))
        if need == 0:
            native.check(-1, 'gcbf_apply_workspace_bytes')
        buf = getattr(self, '_apply_ws', None)
        if buf is None:
            buf = self._apply_ws = native.GrowBuffer()
        ws = buf.get(need, dev)
        rand = float(rand) if rand else 0.0
        noise = torch.randn(max_iter + 1, M, a, device=dev) if rand else None      # gcbf.py:305 draws randn_like per agent and round
        action = torch.empty(M, a, device=dev)
        rounds = ctypes.c_int(0)
        # the library captures a round into CUDA graphs and replays it; capture is impossible on the legacy default stream, so the call
        # runs on a stream of its own, ordered after and before the caller's stream
        cur = torch.cuda.current_stream(dev)
        st = getattr(self, '_apply_stream', None)
        if st is None or st.device != dev:
            st = self._apply_stream = torch.cuda.Stream(dev)
        st.wait_stream(cur)
        with torch.cuda.stream(st):
            rc = native.fn('gcbf_apply')(ctypes.byref(d), ctypes.byref(b), 0.1, rand, noise.data_ptr() if noise is not None else None,
                                         int(max_iter), action.data_ptr(), a, ctypes.byref(rounds), ws.data_ptr(), ws.numel(), st.cuda_stream)
        cur.wait_stream(st)
        native.check(rc, 'gcbf_apply')
        native._mark_fresh(cbf_layers)
        native._mark_fresh(act_layers)
        self.last_apply_rounds = rounds.value
        return action

    # ---- analytic h_dot (SURVEY section 8f-3; additive: the training loss keeps the reference's finite difference) ------------------
    def h_dot_analytic(self, data, action: Optional[Tensor] = None, freeze: Optional[bool] = None):
        """(h, h_dot) with h_dot_i = sum_k dh_i/ds_k . f(s_k, clamp(u_k + u_ref)) as one forward-mode pass (gcbf_b200/jvp.py): the
        derivative the finite difference (h(x + dt f) - h(x)) / dt of gcbf.py:193-207 approximates, edges held fixed.  action: the
        policy's correction (default: the actor's).  The CBF condition of the paper is h_dot + alpha h >= 0."""
        from .. import jvp
        if action is None:
            action = self.act(data)
        return jvp.cbf_value_and_h_dot(self.cbf, self._env, data, action, freeze)

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
