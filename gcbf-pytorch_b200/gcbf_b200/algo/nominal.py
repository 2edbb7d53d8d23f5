"""The nominal baseline (reference gcbf/algo/nominal.py:14-59): nothing is learned, the policy's correction is zero and the env adds
u_ref.  Only `act` / `apply` do anything; the training-side methods of the Algorithm interface refuse, as in the reference."""
from typing import Optional

import torch
from torch import Tensor

from ..controller import NominalController
from .base import Algorithm


def _refuse(name: str):
    def method(self, *args, **kwargs):
        raise NotImplementedError(f'Nominal.{name}: the nominal baseline has nothing to train, store or restore')
    method.__name__ = name
    return method


class Nominal(Algorithm):
    step, is_update, update, save, load = (_refuse(n) for n in ('step', 'is_update', 'update', 'save', 'load'))

    def __init__(self, env, num_agents: int, node_dim: int, edge_dim: int, action_dim: int, device: torch.device):
        super().__init__(env=env, num_agents=num_agents, node_dim=node_dim, edge_dim=edge_dim, action_dim=action_dim, device=device)
        self.actor = NominalController(num_agents, node_dim, edge_dim, action_dim).to(device)

    @torch.no_grad()
    def act(self, data) -> Tensor:
        return self.actor(data)

    def apply(self, data, rand: Optional[float] = 30) -> Tensor:
        return self.act(data)

    def apply_batch(self, batch, rand: Optional[float] = 30, max_iter: int = 30, noise: Optional[Tensor] = None) -> Tensor:
        """The nominal action for every graph of a collated batch (nothing to refine: zero rounds per graph)."""
        self.last_apply_batch_rounds = torch.zeros(self._env._num_graphs_of(batch), dtype=torch.int64)
        return self.act(batch)
