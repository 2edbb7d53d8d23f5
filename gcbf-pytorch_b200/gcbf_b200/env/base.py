"""MultiAgentEnv: the reference's environment interface (gcbf/env/base.py:11-398) with the hot-path methods
-- radius graph, edge features, nominal controller, finite-difference step, safe/unsafe masks -- running in
the sm_90a kernels, batched over all graphs of a `Batch` in ONE launch instead of the reference's per-graph
Python loops (`to_data_list()` at simple_car.py:313, 338 and the re-linking loop at gcbf/algo/gcbf.py:195-199).

Graph layout contract (what every reference env produces): per graph the `num_agents` agents come first, then the
obstacles; a batch is the concatenation of equally sized graphs.
"""
import ctypes
from abc import ABC, abstractmethod
from typing import Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from .. import _C, ops
from ..data import Batch, Data


def lqr(A: np.ndarray, B: np.ndarray, Q: np.ndarray, R: np.ndarray) -> np.ndarray:
    """Discrete-time LQR gain, u = -K x (what reference gcbf/env/utils.py:14-36 computes with the same scipy
    routines; evaluated once per env on the host)."""
    from scipy.linalg import inv, solve_discrete_are
    X = solve_discrete_are(A, B, Q, R)
    return inv(B.T @ X @ B + R) @ (B.T @ X @ A)


def plot_box(points: np.ndarray, agent_radius: float) -> Tuple[np.ndarray, np.ndarray]:
    """The square x-y plotting box the reference's SimpleCar / DubinsCar `reset()` stores for `state_lim` (simple_car.py:136-142,
    dubins_car.py:491-497): the bounding box of `points` (agent positions, goals[, obstacle positions], float32 [k, 2]) grown by
    5 agent radii, then widened along its shorter side to a square about the same centre.  Returns (xy_min, xy_max)."""
    xy_min = np.min(points, axis=0) - agent_radius * 5
    xy_max = np.max(points, axis=0) + agent_radius * 5
    max_interval = (xy_max - xy_min).max()
    return xy_min - 0.5 * (max_interval - (xy_max - xy_min)), xy_max + 0.5 * (max_interval - (xy_max - xy_min))


class _StepFunction(torch.autograd.Function):
    """x+ = x + dt f(x, clamp(u + u_ref(x))): forward_graph's state update with its VJP to the action."""

    @staticmethod
    def forward(ctx, states, action, env, num_graphs, freeze, goal_per_graph=None):
        _C.require_cuda(states, action)
        st, ld = ops._mat(states)
        act = action.detach().contiguous()
        cfg = env._cfg(num_graphs)
        nxt = torch.empty(st.shape[0], ld, device=st.device, dtype=torch.float32)
        pass_mask = torch.empty(act.shape, device=st.device, dtype=torch.uint8)
        goal, ldg = ops._mat(env._goal if goal_per_graph is None else goal_per_graph.contiguous())
        _C.call('gcbf_step_fwd' if goal_per_graph is None else 'gcbf_step_fwd_multi', ctypes.byref(cfg), _C.ptr(st), ld, _C.ptr(act),
                _C.ptr(goal), ldg, _C.ptr(env._gain()), 1 if freeze else 0, _C.ptr(nxt), _C.ptr(pass_mask))
        ctx.env, ctx.num_graphs, ctx.ld = env, num_graphs, ld
        ctx.save_for_backward(pass_mask)
        return nxt[:, :st.shape[1]] if ld != st.shape[1] else nxt

    @staticmethod
    def backward(ctx, d_next):
        (pass_mask,) = ctx.saved_tensors
        dn, ld = ops._mat(d_next)
        cfg = ctx.env._cfg(ctx.num_graphs)
        d_action = torch.empty(pass_mask.shape, device=dn.device, dtype=torch.float32)
        _C.call('gcbf_step_bwd', ctypes.byref(cfg), _C.ptr(dn), ld, _C.ptr(pass_mask), _C.ptr(d_action))
        return None, d_action, None, None, None, None


class MultiAgentEnv(ABC):
    ENV_NAME = ''
    POS_DIM = 2
    RADIUS_KEY = 'car_radius'
    GRAPH_METRIC = 1          # 0: squared distance (torch_cluster), 1: torch.norm then compare
    GOAL_DIM = 2              # goal columns the kernels read (SimpleCar 2, DubinsCar 2, SimpleDrone 6)
    # reset(): agents / goals pairwise farther than RESET_*_SPACING agent radii, and (envs with obstacles) farther than
    # RESET_CLEARANCE[0] * R + RESET_CLEARANCE[1] * obs_point_r from every obstacle; goal rows of RESET_GOAL_DIM columns.  The device
    # reset (env/device_reset.py) reads the same attributes.
    RESET_AGENT_SPACING = 4
    RESET_GOAL_SPACING = 4
    RESET_CLEARANCE = (2, 2)
    RESET_GOAL_DIM = 2
    _xy_min = _xy_max = None  # x-y plotting box of state_lim (SimpleCar / DubinsCar: set by reset(), see plot_box)

    def __init__(self, num_agents: int, device: torch.device, dt: float = 0.03, params: Optional[dict] = None,
                 max_neighbors: Optional[int] = None):
        self._num_agents = num_agents
        self._device = device
        self._dt = dt
        self._params = self.default_params if params is None else params
        if max_neighbors is not None and int(max_neighbors) < 1:
            raise ValueError(f'max_neighbors must be >= 1, got {max_neighbors}')
        # top-k neighbour filter of the MACBF baseline (train.py:30 builds the env with max_neighbors = 12): switches
        # add_communication_links to the filtered radius-graph kernel (csrc/macbf.cu)
        self._max_neighbors = None if max_neighbors is None else int(max_neighbors)
        self._data = None
        self._goal = None
        self._K = None
        self._t = 0
        self._mode = 'train'

    # ---- bookkeeping identical to the reference interface ---------------------------------------------
    def train(self):
        self._mode = 'train'

    def test(self):
        self._mode = 'test'

    num_agents = property(lambda self: self._num_agents)
    dt = property(lambda self: self._dt)
    device = property(lambda self: self._device)
    data = property(lambda self: self._data)
    state = property(lambda self: self._data.states)

    @property
    @abstractmethod
    def default_params(self) -> dict:
        ...

    @property
    @abstractmethod
    def state_dim(self) -> int:
        ...

    @property
    def node_dim(self) -> int:
        return 4

    @property
    @abstractmethod
    def edge_dim(self) -> int:
        ...

    @property
    @abstractmethod
    def action_dim(self) -> int:
        ...

    @property
    @abstractmethod
    def action_lim(self) -> Tuple[Tensor, Tensor]:
        ...

    @property
    def num_obstacles(self) -> int:
        return 0

    @property
    def nodes_per_graph(self) -> int:
        return self._num_agents + self.num_obstacles

    # ---- kernel plumbing -----------------------------------------------------------------------------
    def _num_graphs_of(self, data) -> int:
        total = int(data.states.shape[0])
        N = self.nodes_per_graph
        if total % N != 0:
            raise ValueError(f'{total} nodes is not a multiple of {N} nodes per graph')
        return total // N

    def _cfg(self, num_graphs: int) -> _C.EnvCfg:
        p = self._params
        return _C.EnvCfg(ops.ENV_IDS[self.ENV_NAME], num_graphs, self.nodes_per_graph, self._num_agents,
                         float(p[self.RADIUS_KEY]), float(p['speed_limit']), float(p['dist2goal']), float(self._dt))

    def _gain(self) -> Optional[Tensor]:
        return None

    def _plot_box(self):
        if self._xy_min is None:
            raise RuntimeError(f'{self.ENV_NAME}.state_lim: its x-y box is set by reset(); call reset() first or pass the limits explicitly')
        return self._xy_min, self._xy_max

    def set_goal(self, goal: Tensor):
        """Install the goal set [num_agents, goal_dim] (the reference keeps it in `env._goal`).  Rows narrower than the
        kernels read (SimpleDrone: 6 columns, position + zero velocity) are zero-padded; fewer than POS_DIM columns raise."""
        goal = goal.to(self._device, torch.float32)
        if goal.dim() != 2 or goal.shape[0] != self._num_agents or goal.shape[1] < self.POS_DIM:
            raise ValueError(f'goal must be [{self._num_agents}, >= {self.POS_DIM}], got {tuple(goal.shape)}')
        if goal.shape[1] < self.GOAL_DIM:
            goal = torch.cat([goal, goal.new_zeros(goal.shape[0], self.GOAL_DIM - goal.shape[1])], dim=1)
        self._goal = goal.contiguous()

    # ---- hot path ------------------------------------------------------------------------------------
    def edge_attr(self, state: Tensor, edge_index: Tensor) -> Tensor:
        return ops.EdgeAttrFunction.apply(state, edge_index, ops.ENV_IDS[self.ENV_NAME])

    def add_communication_links(self, data):
        """Radius graph + edge features (K1 + K2) for a single graph or a whole batch in one launch."""
        B = self._num_graphs_of(data)
        if self._max_neighbors is not None:
            ei, _ = ops.radius_graph_topk(data.states.detach(), self.POS_DIM, B, self.nodes_per_graph, self._num_agents,
                                          self._params['comm_radius'], self.GRAPH_METRIC, self._max_neighbors)
        else:
            ei, _ = ops.radius_graph(data.states.detach(), self.POS_DIM, B, self.nodes_per_graph, self._num_agents,
                                     self._params['comm_radius'], self.GRAPH_METRIC)
        data.update(Data(edge_index=ei, edge_attr=self.edge_attr(data.states, ei)))
        from ..nn.gnn import prime_rowptr
        prime_rowptr(ei, int(data.states.shape[0]))      # the CSR the GNN passes need: known sorted, no check / host sync later
        return data

    def u_ref(self, data) -> Tensor:
        B = self._num_graphs_of(data)
        st, ld = ops._mat(data.states.detach())
        out = torch.empty(B * self._num_agents, self.action_dim, device=st.device, dtype=torch.float32)
        goal, ldg = ops._mat(self._goal)
        cfg = self._cfg(B)
        _C.call('gcbf_u_ref', ctypes.byref(cfg), _C.ptr(st), ld, _C.ptr(goal), ldg, _C.ptr(self._gain()), _C.ptr(out))
        return out

    def forward(self, data, u: Tensor) -> Tensor:
        """Next state for an ALREADY clamped total action is not exposed by the kernels; the reference's
        `forward(data, action)` is only reached through forward_graph / step, which are implemented below."""
        raise NotImplementedError('use forward_graph(data, action) / step(action)')

    def next_states(self, data, action: Tensor) -> Tensor:
        B = self._num_graphs_of(data)
        # the reference's single-graph discriminator (dubins_car.py:126, simple_drone.py:113): a batch of ONE graph
        # takes the reach-freeze branch too
        return _StepFunction.apply(data.states, action, self, B, B == 1)

    def next_states_single(self, data, action: Tensor) -> Tensor:
        """Next states as the reference computes them graph by graph in the re-linking loop
        (gcbf/algo/gcbf.py:195-199): every graph is a *single* graph there, so the reach-freeze branch applies."""
        return _StepFunction.apply(data.states, action, self, self._num_graphs_of(data), True)

    def forward_graph(self, data, action: Tensor, single: bool = False, goal: Optional[Tensor] = None):
        """Graph after one step with RETAINED edges and recomputed edge features (differentiable w.r.t. action).  single: every graph
        of the batch is a single graph of the reference (reach-freeze branch per graph, as the test-time controller needs);
        goal [B * n, goal_dim]: one goal set per graph instead of env._goal."""
        B = self._num_graphs_of(data)
        state = _StepFunction.apply(data.states, action, self, B, single or B == 1, goal)     # = next_states by default
        fields = dict(x=data.x, edge_index=data.edge_index, edge_attr=self.edge_attr(state, data.edge_index),
                      pos=state[:, :self.POS_DIM], states=state)
        if hasattr(data, 'agent_mask'):
            fields['agent_mask'] = data.agent_mask
        return Data(**fields)

    def _masks(self, data):
        B = self._num_graphs_of(data)
        st, ld = ops._mat(data.states.detach())
        na = B * self._num_agents
        out = torch.empty(3, na, device=st.device, dtype=torch.uint8)
        cfg = self._cfg(B)
        _C.call('gcbf_masks', ctypes.byref(cfg), _C.ptr(st), ld, _C.ptr(out[0]), _C.ptr(out[1]), _C.ptr(out[2]))
        return out.view(torch.bool)

    def edge_masks(self, data) -> Tensor:
        """[2, E] bool: (safe, unsafe) per edge = the `return_edge=True` branches of safe_mask / unsafe_mask (simple_car.py:307-311,
        332-336 and siblings): dist = ||edge_attr[:, :pos_dim]||, safe = dist > 4R, unsafe = dist < 2R.  One launch for both."""
        return ops.edge_masks(data.edge_attr, self.POS_DIM, float(self._params[self.RADIUS_KEY]))

    def safe_mask(self, data, return_edge: bool = False) -> Tensor:
        if return_edge:
            return self.edge_masks(data)[0]
        return self._masks(data)[0]

    def unsafe_mask(self, data, return_edge: bool = False) -> Tensor:
        if return_edge:
            return self.edge_masks(data)[1]
        return self._masks(data)[1]

    def collision_mask(self, data) -> Tensor:
        return self._masks(data)[2]

    # ---- rollout scaffolding (host glue; SURVEY section 8f "next") --------------------------------------------
    @abstractmethod
    def make_graph(self, states: Tensor):
        """Data for `states` [B*N, state_dim] (x, pos, states[, agent_mask]) without edges."""

    def graph_from_states(self, states: Tensor, with_u_ref: bool = True):
        data = self.add_communication_links(self.make_graph(states.to(self._device, torch.float32)))
        if with_u_ref:
            data.update(Data(u_ref=self.u_ref(data)))
        return data

    @abstractmethod
    def reset(self):
        ...

    def step(self, action: Tensor):
        """One environment step of a single graph (reference simple_car.py:146-176 and siblings)."""
        self._t += 1
        prev = self._data
        n, pd = self._num_agents, self.POS_DIM
        prev_reach = torch.norm(prev.states[:n, :pd] - self._goal[:, :pd], dim=1) < self._params['dist2goal']
        with torch.no_grad():
            state = self.next_states(prev, action)
        self._data = self.add_communication_links(self.make_graph(state))
        reach = torch.norm(state[:n, :pd] - self._goal[:, :pd], dim=1) < self._params['dist2goal']
        done = self._t >= self.max_episode_steps or bool(reach.all())
        collision = self.collision_mask(self._data)
        reward = self._reward(action, reach, prev_reach, collision)
        info = {'safe': float(1.0 - collision.sum() / n), 'reach': reach, 'collision': torch.where(collision)[0]}
        return self._data, reward.detach().cpu().numpy(), done, info

    def _reward(self, action, reach, prev_reach, collision):
        return (reach.int() - prev_reach.int()) * 4 - collision.int() * 2 - 0.01 - torch.norm(action, dim=1) * 0.0001

    @property
    def max_episode_steps(self) -> int:
        return 500 if self._mode == 'train' else 2500
