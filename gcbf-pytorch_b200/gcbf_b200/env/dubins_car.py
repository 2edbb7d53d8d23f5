"""DubinsCar: unicycle agents [x, y, theta, v] plus `num_obs` moving point obstacles with the same state
(reference gcbf/env/dubins_car.py, modes train/test only -- the pybullet / LiDAR demo modes are simulation
scaffolding outside the hot path).  Graph = dense torch.norm(pos_i - pos_j) < r on agent rows."""
from typing import Optional, Tuple

import math
import torch
from torch import Tensor

from ..data import Data
from ._sampling import sample_separated
from .base import MultiAgentEnv, plot_box


class DubinsCar(MultiAgentEnv):
    ENV_NAME = 'DubinsCar'
    POS_DIM = 2
    RADIUS_KEY = 'car_radius'
    GRAPH_METRIC = 1

    state_dim = property(lambda self: 4)
    edge_dim = property(lambda self: 5)
    action_dim = property(lambda self: 2)

    def __init__(self, num_agents, device, dt=0.03, params=None, max_neighbors=None):
        super().__init__(num_agents, device, dt, params, max_neighbors)
        self._num_obs = int(self._params['num_obs'])
        self._obs = None

    @property
    def default_params(self) -> dict:
        return {'max_distance': 4.0, 'area_size': 4.0, 'car_radius': 0.05, 'dist2goal': 0.05, 'comm_radius': 1.0,
                'obs_point_r': 0.05, 'obs_len_max': 0.5, 'speed_limit': 0.8, 'obs_speed_limit': 0.2, 'num_obs': 0}

    @property
    def num_obstacles(self) -> int:
        return self._num_obs

    @property
    def action_lim(self) -> Tuple[Tensor, Tensor]:
        hi = torch.ones(2, device=self.device) * 2.
        return -hi, hi

    @property
    def state_lim(self) -> Tuple[Tensor, Tensor]:
        """(low, high) of [x, y, theta, v] for plotting (reference dubins_car.py:748-756): the x-y box of the last reset()."""
        xy_min, xy_max = self._plot_box()
        low_lim = torch.tensor([xy_min[0], xy_min[1], -10, -10], device=self.device)
        high_lim = torch.tensor([xy_max[0], xy_max[1], 10, 10], device=self.device)
        return low_lim, high_lim

    def make_graph(self, states: Tensor) -> Data:
        n, o = self.num_agents, self._num_obs
        B = states.shape[0] // (n + o)
        x = torch.cat([torch.zeros(n, 4), torch.ones(o, 4)], dim=0).repeat(B, 1).to(states)
        mask = torch.cat([torch.ones(n, dtype=torch.bool), torch.zeros(o, dtype=torch.bool)]).repeat(B).to(states.device)
        return Data(x=x, pos=states[:, :2], states=states, agent_mask=mask)

    def reset(self) -> Data:
        self._t = 0
        p = self._params
        side, R = p['area_size'], p['car_radius']
        clear = 2 * R + 2 * p['obs_point_r']
        obs = torch.rand(self._num_obs, 4)
        obs[:, :2] *= side
        obs[:, 2] *= 2 * math.pi
        obs[:, 3] *= p['obs_speed_limit']
        self._obs = obs.to(self.device)
        pos = sample_separated(self.num_agents, 2, side, 4 * R, obs[:, :2], clear)
        goal_xy = sample_separated(self.num_agents, 2, side, 5 * R, obs[:, :2], clear)
        heading = torch.rand(self.num_agents, 1) * 2 * math.pi - math.pi
        agents = torch.cat([pos, heading, torch.zeros(self.num_agents, 1)], dim=1)
        goal_heading = torch.rand(self.num_agents, 1) * 2 * math.pi - math.pi
        self.set_goal(torch.cat([goal_xy, goal_heading, torch.zeros(self.num_agents, 1)], dim=1))
        states = torch.cat([agents, obs], dim=0).to(self.device)
        self._xy_min, self._xy_max = plot_box(torch.cat([pos, goal_xy, obs[:, :2]], dim=0).float().numpy(), R)
        self._data = self.add_communication_links(self.make_graph(states))
        return self._data

    def _reward(self, action, reach, prev_reach, collision):
        return (reach.int() - prev_reach.int()) * 10 - collision.int() * 0.1 - 0.0001 - torch.norm(action, dim=1).sum() * 0.01   # dubins_car.py:535 (summed over agents)
