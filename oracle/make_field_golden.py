"""TEST INFRASTRUCTURE ONLY (needs a checkout of the reference).  Generates tests/golden/cbf_field/*.pt: the CBF level-set field of
the reference's plot_cbf_contour (gcbf/trainer/utils.py:259-273), computed by the UNMODIFIED reference on oracle/shim.

Per case: the reference env's own reset() under a seed gives the states, goals, graph and state_lim; the CBF is the reference's seeded
initialisation (torch.manual_seed(init_seed) before make_algo, as oracle/ref_harness.py) with the last head layer scaled by HEAD_GAIN
(the seeded-init field alone is nearly flat).  The field is built the way plot_cbf_contour builds it: the
np.linspace axes over state_lim, np.meshgrid, one copy of the graph per grid point with state[agent, x_dim], state[agent, y_dim]
overwritten, the given edge_index, edge_attr recomputed by env.edge_attr, ONE cbf call on the Batch of all copies, agent's row kept.
Stored: inputs (states, goals, obstacles, edge_index, state_lim, xs, ys), the field [n_mesh, n_mesh], the CBF's spectral-norm vectors
before and after the call (one power iteration), and how the weights were made.

    python oracle/make_field_golden.py
Files go to tests/golden/cbf_field/ (NOT tests/golden/*.pt: those are the per-case train-step fixtures other tests enumerate).
"""
import copy
import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
OUT_DIR = os.path.join(ROOT, 'tests', 'golden', 'cbf_field')
N_MESH = 30
INIT_SEED = 0
HEAD_GAIN = 200.0      # the seeded init's last head layer alone gives fields with a spread of ~1e-4, too flat to test at 1e-5
HEAD_KEYS = ('feat_2_CBF.net.6.weight', 'feat_2_CBF.net.6.bias')

# name, env, agents, obstacles, area, reset seed, agent ('busiest': most in-edges, lowest id first; 'isolated': first without), dims
CASES = [
    ('simplecar_n16', 'SimpleCar', 16, 0, 4.0, 11, 'busiest', (0, 1)),
    ('dubins_n16_o4_xy', 'DubinsCar', 16, 4, 4.0, 12, 'busiest', (0, 1)),
    ('dubins_n16_o4_theta_v', 'DubinsCar', 16, 4, 4.0, 12, 'busiest', (2, 3)),
    ('drone_n8_o8', 'SimpleDrone', 8, 8, 2.0, 13, 'busiest', (0, 1)),
    ('simplecar_n6_isolated', 'SimpleCar', 6, 0, 8.0, 14, 'isolated', (0, 1)),
]


def field_weights(sd):
    """The CBF weights of every fixture: the seeded initialisation with the last head layer times HEAD_GAIN (h = tanh(HEAD_GAIN z): the
    fields then span a good part of (-1, 1) and cross zero, i.e. have a level set, while staying well conditioned)."""
    out = {k: v.clone() for k, v in sd.items()}
    for k in HEAD_KEYS:
        out[k] = out[k] * HEAD_GAIN
    return out


def sn_vectors(cbf):
    return {k: v.detach().clone() for k, v in cbf.state_dict().items() if k.endswith(('weight_u', 'weight_v'))}


def make_case(name, env_name, n, obs, area, seed, agent, dims):
    from gcbf.algo import make_algo
    from gcbf.env import make_env
    from gcbf.trainer.utils import read_params
    from torch_geometric.data import Batch, Data

    dev = torch.device('cpu')
    params = make_env(env_name, n, dev).default_params
    params['area_size'] = area
    params['num_obs'] = obs
    env = make_env(env_name, n, dev, params=params)
    env.train()
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    data = env.reset()
    ei = data.edge_index
    indeg = torch.bincount(ei[1], minlength=n)[:n]
    if agent == 'isolated':
        free = torch.nonzero(indeg == 0).reshape(-1)
        assert free.numel() > 0, f'{name}: every agent has in-edges'
        agent = int(free[0])
    else:
        agent = int(torch.argmax(indeg))
    torch.manual_seed(INIT_SEED)
    algo = make_algo('gcbf', env, n, env.node_dim, env.edge_dim, env.action_dim, dev, 512, read_params(env_name, 'gcbf'))
    algo.cbf.load_state_dict(field_weights(algo.cbf.state_dict()))
    uv_before = sn_vectors(algo.cbf)

    x_dim, y_dim = dims
    lo, hi = env.state_lim
    xs = np.linspace(lo[x_dim].cpu(), hi[x_dim].cpu(), N_MESH)
    ys = np.linspace(lo[y_dim].cpu(), hi[y_dim].cpu(), N_MESH)
    gx, gy = np.meshgrid(xs, ys)
    graphs = []
    for i in range(N_MESH):
        for j in range(N_MESH):
            st = copy.deepcopy(data.states)
            # plot_cbf_contour writes the numpy scalar itself; torch 2.11 refuses a numpy.float32 there, so it goes through a
            # python float (exact for float32 and float64 grid values: the fp32 state rounds it the same way)
            st[agent, x_dim] = float(gx[i, j])
            st[agent, y_dim] = float(gy[i, j])
            fields = dict(x=data.x, edge_index=ei, pos=st[:, :2], edge_attr=env.edge_attr(st, ei))
            if hasattr(data, 'agent_mask') and data.agent_mask is not None:
                fields['agent_mask'] = data.agent_mask
            graphs.append(Data(**fields))
    with torch.no_grad():
        h = algo.cbf(Batch.from_data_list(graphs)).view(N_MESH, N_MESH, n)[:, :, agent].clone()
    N = data.states.shape[0]
    obs_states = data.states[n:].clone() if N > n else torch.zeros(0, data.states.shape[1])
    return dict(meta=dict(name=name, env=env_name, n=n, obs=N - n, area=area, seed=seed, agent=agent, x_dim=x_dim, y_dim=y_dim,
                          n_mesh=N_MESH, init_seed=INIT_SEED, head_gain=HEAD_GAIN),
                states=data.states.clone(), goals=env._goal.clone(), obstacles=obs_states, x=data.x.clone(), edge_index=ei.clone(),
                state_lim=(lo.clone(), hi.clone()), xs=xs, ys=ys, field=h, uv_before=uv_before, uv_after=sn_vectors(algo.cbf))


def main():
    sys.path.insert(0, HERE)
    from ref_loader import load_reference
    load_reference()
    os.makedirs(OUT_DIR, exist_ok=True)
    for case in CASES:
        fix = make_case(*case)
        path = os.path.join(OUT_DIR, case[0] + '.pt')
        torch.save(fix, path)
        f = fix['field']
        print(path, os.path.getsize(path), 'agent', fix['meta']['agent'], 'field range', float(f.min()), float(f.max()), 'in-edges', int((fix['edge_index'][1] == fix['meta']['agent']).sum()))


if __name__ == '__main__':
    main()
