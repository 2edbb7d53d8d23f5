"""Shared builders for the parity tests: the same (synthetic states, seeded weights) on the oracle side
(CPU tensors / state dicts) and on the product side (gcbf_b200 modules)."""
import copy

import torch

import gcbf_oracle as O
from gcbf_b200 import ops, synth


def case_inputs(meta):
    sb = synth.make_states(meta['env'], meta['n'], meta['obs'], meta['graphs'], meta['area'], meta['seed'])
    return sb


from gcbf_b200.synth import seeded_algo, product_batch  # noqa: E402,F401


def oracle_batch(sb):
    """edge_index / u_ref / x / agent_mask / K on the CPU oracle for a SynthBatch."""
    env, n, o, B = sb.env, sb.num_agents, sb.num_obs, sb.num_graphs
    N = n + o
    ei = O.batch_radius_graph(env, sb.states, B, N, n)
    K = O.lqr_gain(env) if env != 'DubinsCar' else None
    x, am = O.make_graph_inputs(env, sb.states, B, n, o)
    ag = sb.states if am is None else sb.states[am]
    ur = O.u_ref(env, ag, sb.goals, K)
    return dict(edge_index=ei, K=K, x=x, agent_mask=am, u_ref=ur, N=N)


def sd_clone(module):
    return {k: v.detach().cpu().clone() for k, v in module.state_dict().items()}


def per_tensor(t):
    """(gcbf_h16 descriptor, the ops.H16 that owns its buffers) of an fp32 device matrix: amax + split kernels, one scale word."""
    h = ops.split_h(t)
    return h.desc(), h


def tiled_buffers(rows, cols, device='cuda:0'):
    """(gcbf_h16 descriptor, planes, tile maxima) of a zero-filled tile-scaled companion for an epilogue to write."""
    ld = (cols + 7) // 8 * 8
    buf = torch.zeros(2, rows, ld, device=device, dtype=torch.float16)
    tr, tc = (rows + 127) // 128, (cols + 255) // 256
    amax = torch.zeros(tr, tc, device=device, dtype=torch.int32)
    return ops.H16(buf, amax, rows, cols, ld, tc, 1).desc(), buf, amax
