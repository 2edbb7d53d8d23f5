"""The GCBF policy network: one attention message-passing layer producing a 1024-wide feature per node, restricted to the agent
rows, concatenated with the nominal control u_ref and reduced by a 4-layer head to the action correction.  Same constructor,
sub-module names (= checkpoint keys `feat_transformer.module_0.*`, `feat_2_action.net.*`) and `forward(data)` contract as the
reference's gcbf/controller/gnn_controller.py:13-48; here the whole chain -- edge MLP, aggregation, node MLP, row selection,
concat, head -- is ONE autograd node over the sm_90a kernels (`ops.GNNNetFunction`, reached through the layer's `run`)."""
from torch import Tensor

from ..data import agent_row_index
from ..nn.gnn import ControllerGNNLayer, GraphSequential
from ..nn.mlp import MLP
from .base import MultiAgentController


class GNNController(MultiAgentController):
    FEATURE_WIDTH = 1024
    HEAD_WIDTHS = (512, 128, 32)

    def __init__(self, num_agents: int, node_dim: int, edge_dim: int, phi_dim: int, action_dim: int):
        super().__init__(num_agents, node_dim, edge_dim, action_dim)
        gnn = ControllerGNNLayer(node_dim, edge_dim, self.FEATURE_WIDTH, phi_dim)
        # construction order (message-passing layer, then head) fixes the seeded initialisation; the attribute names are the
        # state-dict contract with the reference's actor.pkl
        self.feat_transformer = GraphSequential(gnn)
        self.feat_2_action = MLP(self.FEATURE_WIDTH + action_dim, action_dim, self.HEAD_WIDTHS)

    def forward(self, data) -> Tensor:
        """data: x, edge_attr, edge_index, u_ref [, agent_mask]  ->  actions [num_graphs * num_agents, action_dim]."""
        gnn = self.feat_transformer.module_0
        return gnn.run(data.x, data.edge_attr, data.edge_index, row_index=agent_row_index(data), head=self.feat_2_action,
                       head_extra=data.u_ref)
