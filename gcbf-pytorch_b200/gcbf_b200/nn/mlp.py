"""gcbf.nn.MLP on the sm_90a kernels.

Same constructor, same `.net` nn.Sequential (so the state-dict keys `net.{0,2,4}.{weight|weight_orig,weight_u,
weight_v,bias}` and the RNG stream of the initialisation are identical to reference gcbf/nn/mlp.py:9-47), but
`forward` never calls the nn.Linear modules: it hands their parameters to MLPFunction (ops.py), i.e. to the
CUDA GEMM + fused bias/activation kernels, including the per-forward spectral-norm power iteration that
torch.nn.utils.spectral_norm would run as a forward-pre-hook.
"""
from typing import List, Sequence

import torch
import torch.nn as nn
from torch.nn.utils import spectral_norm

from .. import ops
from .utils import init_param


def _make_linear(n_in: int, n_out: int, init: bool, gain: float, limit_lip: bool) -> nn.Module:
    layer = nn.Linear(n_in, n_out)
    if limit_lip:
        layer = spectral_norm(layer)       # registers weight_orig / weight_u / weight_v (old-style SN)
    if init:
        layer = init_param(layer, gain=gain)
    return layer


class MLP(nn.Module):

    def __init__(self, in_channels: int, out_channels: int, hidden_layers: tuple,
                 hidden_activation: nn.Module = nn.ReLU(), output_activation: nn.Module = None,
                 init: bool = True, gain: float = 1., limit_lip: bool = False):
        super().__init__()
        widths = [in_channels, *hidden_layers, out_channels]
        mods: List[nn.Module] = []
        for i in range(len(widths) - 1):
            mods.append(_make_linear(widths[i], widths[i + 1], init, gain, limit_lip))
            if i < len(widths) - 2:
                mods.append(hidden_activation)
        if output_activation is not None:
            mods.append(output_activation)
        self.net = nn.Sequential(*mods)
        self.limit_lip = limit_lip

    # ---- kernel-facing description -----------------------------------------------------------------
    def specs(self) -> List[ops.LinearSpec]:
        out: List[ops.LinearSpec] = []
        mods = list(self.net)
        for i, m in enumerate(mods):
            if not isinstance(m, nn.Linear):
                continue
            nxt = mods[i + 1] if i + 1 < len(mods) else None
            if nxt is None or isinstance(nxt, nn.Linear):
                act = ops.ACT_NONE
            elif isinstance(nxt, nn.ReLU):
                act = ops.ACT_RELU
            elif isinstance(nxt, nn.Tanh):
                act = ops.ACT_TANH
            else:
                raise NotImplementedError(f'activation {type(nxt).__name__} has no fused epilogue '
                                          '(the reference only uses ReLU / Tanh)')
            if hasattr(m, 'weight_orig'):
                out.append(ops.LinearSpec(m.weight_orig, m.bias, m.weight_u, m.weight_v, act))
            else:
                out.append(ops.LinearSpec(m.weight, m.bias, None, None, act))
        return out

    @staticmethod
    def flat_params(specs: Sequence[ops.LinearSpec]) -> List[torch.Tensor]:
        flat = []
        for s in specs:
            flat += [s.W, s.b]
        return flat

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        specs = self.specs()
        lead = x.shape[:-1]
        if x.numel() == 0:        # no rows (e.g. the edge MLP of a graph without edges): nothing to launch, no gradient to anybody
            return x.new_zeros(*lead, int(specs[-1].W.shape[0]))
        if not torch.is_grad_enabled() and ops.NATIVE and len(specs) <= ops.native.MAX_LAYERS and x.is_cuda:
            y = ops.native_mlp_forward(x.reshape(-1, x.shape[-1]), specs, False)[0]      # inference: nothing saved (see gnn.py run())
        else:
            y = ops.MLPFunction.apply(x.reshape(-1, x.shape[-1]), specs, *self.flat_params(specs))
        return y.reshape(*lead, y.shape[-1])
