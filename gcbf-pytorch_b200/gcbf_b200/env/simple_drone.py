"""SimpleDrone: 3-D linear drone model [x, y, z, vx, vy, vz] with `num_agents` static point obstacles
(reference gcbf/env/simple_drone.py: reset() always creates num_agents obstacles, :130-135)."""
from typing import Optional, Tuple

import numpy as np
import torch
from torch import Tensor

from ..data import Data
from ._sampling import sample_separated
from .base import MultiAgentEnv, lqr


class SimpleDrone(MultiAgentEnv):
    ENV_NAME = 'SimpleDrone'
    POS_DIM = 3
    GOAL_DIM = 6
    RADIUS_KEY = 'drone_radius'
    GRAPH_METRIC = 1

    state_dim = property(lambda self: 6)
    edge_dim = property(lambda self: 6)
    action_dim = property(lambda self: 3)

    @property
    def default_params(self) -> dict:
        return {'area_size': 2., 'speed_limit': 0.6, 'drone_radius': 0.05, 'comm_radius': 0.5, 'dist2goal': 0.02,
                'obs_point_r': 0.05, 'obs_len_max': 0.5, 'max_distance': 4.0, 'num_obs': 4}

    @property
    def num_obstacles(self) -> int:
        return self.num_agents

    @property
    def action_lim(self) -> Tuple[Tensor, Tensor]:
        hi = torch.ones(3, device=self.device) * 10.
        return -hi, hi

    def _gain(self) -> Optional[Tensor]:
        if self._K is None:   # reference simple_drone.py:85-101, 354-361
            A0 = np.zeros((6, 6), dtype=np.float32)
            A0[0, 3] = A0[1, 4] = A0[2, 5] = 1.
            A0[3, 3] = A0[4, 4] = -1.1
            A0[5, 5] = -6.
            B0 = np.zeros((6, 3), dtype=np.float32)
            B0[3, 0] = B0[4, 1] = 1.1
            B0[5, 2] = 6.
            K = lqr(A0 * self.dt + np.eye(6), B0 * self.dt, np.eye(6), np.eye(3))
            self._K = torch.from_numpy(K).to(self.device, torch.float32).contiguous()
        return self._K

    @property
    def state_lim(self) -> Tuple[Tensor, Tensor]:
        """(low, high) of [x, y, z, vx, vy, vz] for plotting (reference simple_drone.py:44-45, 335-341): the cube [0, area_size]^3."""
        xyz_min, xyz_max = np.array([0, 0, 0]), np.ones(3) * self._params['area_size']
        low_lim = torch.tensor([xyz_min[0], xyz_min[1], xyz_min[2], -10, -10, -10], device=self.device)
        high_lim = torch.tensor([xyz_max[0], xyz_max[1], xyz_max[2], 10, 10, 10], device=self.device)
        return low_lim, high_lim

    def make_graph(self, states: Tensor) -> Data:
        n = self.num_agents
        B = states.shape[0] // (2 * n)
        x = torch.cat([torch.zeros(n, 4), torch.ones(n, 4)], dim=0).repeat(B, 1).to(states)
        mask = torch.cat([torch.ones(n, dtype=torch.bool), torch.zeros(n, dtype=torch.bool)]).repeat(B).to(states.device)
        return Data(x=x, pos=states[:, :3], states=states, agent_mask=mask)

    def reset(self) -> Data:
        self._t = 0
        p = self._params
        side, R = p['area_size'], p['drone_radius']
        clear = 2 * R + 2 * p['obs_point_r']
        n = self.num_agents
        obs_pos = torch.rand(n, 3) * side
        pos = sample_separated(n, 3, side, 4 * R, obs_pos, clear)
        goal = sample_separated(n, 3, side, 4 * R, obs_pos, clear)
        self.set_goal(torch.cat([goal, torch.zeros(n, 3)], dim=1))
        agents = torch.cat([pos, torch.zeros(n, 3)], dim=1)
        obstacles = torch.cat([obs_pos, torch.zeros(n, 3)], dim=1)
        self._data = self.add_communication_links(self.make_graph(torch.cat([agents, obstacles], dim=0).to(self.device)))
        return self._data

    @property
    def max_episode_steps(self) -> int:
        return 500 if self._mode == 'train' else 2000
