"""SimpleCar: double integrator in the plane, state [x, y, vx, vy], no obstacles (reference
gcbf/env/simple_car.py).  Graph = torch_cluster-style radius graph (squared distance < r^2)."""
from typing import Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from ..data import Data
from ._sampling import sample_separated
from .base import MultiAgentEnv, lqr, plot_box


class SimpleCar(MultiAgentEnv):
    ENV_NAME = 'SimpleCar'
    POS_DIM = 2
    RADIUS_KEY = 'car_radius'
    GRAPH_METRIC = 0

    state_dim = property(lambda self: 4)
    edge_dim = property(lambda self: 4)
    action_dim = property(lambda self: 2)

    @property
    def default_params(self) -> dict:
        return {'m': 1.0, 'comm_radius': 1.0, 'car_radius': 0.05, 'dist2goal': 0.04, 'speed_limit': 0.8,
                'max_distance': 4.0, 'area_size': 4.0}

    @property
    def action_lim(self) -> Tuple[Tensor, Tensor]:
        hi = torch.ones(2, device=self.device) * 10.
        return -hi, hi

    def _gain(self) -> Optional[Tensor]:
        if self._K is None:   # LQR on the discretised double integrator (reference simple_car.py:274-290)
            A = np.eye(4)
            A[0, 2] = A[1, 3] = self.dt
            B = np.zeros((4, 2))
            B[2, 0] = B[3, 1] = self.dt
            self._K = torch.from_numpy(lqr(A, B, np.eye(4), np.eye(2))).to(self.device, torch.float32).contiguous()
        return self._K

    @property
    def state_lim(self) -> Tuple[Tensor, Tensor]:
        """(low, high) of [x, y, vx, vy] for plotting (reference simple_car.py:254-262): the x-y box of the last reset()."""
        xy_min, xy_max = self._plot_box()
        low_lim = torch.tensor([xy_min[0], xy_min[1], -self._params['speed_limit'], -self._params['speed_limit']],
                               device=self.device)
        high_lim = torch.tensor([xy_max[0], xy_max[1], self._params['speed_limit'], self._params['speed_limit']],
                                device=self.device)
        return low_lim, high_lim

    def make_graph(self, states: Tensor) -> Data:
        return Data(x=torch.zeros_like(states), pos=states[:, :2], states=states)

    def reset(self) -> Data:
        self._t = 0
        side, R = self._params['area_size'], self._params['car_radius']
        pos = sample_separated(self.num_agents, 2, side, self.RESET_AGENT_SPACING * R)
        goal = sample_separated(self.num_agents, 2, side, self.RESET_GOAL_SPACING * R)
        self.set_goal(goal)
        self._xy_min, self._xy_max = plot_box(torch.cat([pos, goal], dim=0).float().numpy(), R)
        states = torch.cat([pos, torch.zeros(self.num_agents, 2)], dim=1).to(self.device)
        self._data = self.add_communication_links(self.make_graph(states))
        return self._data
