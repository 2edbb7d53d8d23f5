"""CPU oracle of the CBF level-set field (GCBF.cbf_field), composed from oracle/gcbf_oracle.py: brute-force probe graphs, one probe
(= one grid point of one agent of one graph) at a time, and the CBF over all probes in one oracle forward (one power iteration).

Probe t = ((b * A + k) * ny + iy) * nx + ix: agent agents[k] of graph b with state[x_dim] = xs[ix], state[y_dim] = ys[iy].
  fixed:  its in-edges of the given edge_index, in order;
  relink: the radius graph of the moved graph b (oracle radius_graph) restricted to target a.
The virtual graph has the B * N original nodes followed by one node per probe; edges point from original nodes to probe nodes.
"""
import numpy as np
import torch

import gcbf_oracle as O


def probe_states(states, N, B, agents, x_dim, y_dim, xs, ys):
    """[T, state_dim] moved states and [T] node ids of the probed agents."""
    xs32, ys32 = torch.as_tensor(np.asarray(xs, np.float32)), torch.as_tensor(np.asarray(ys, np.float32))
    rows, nodes = [], []
    for b in range(B):
        for a in agents:
            for iy in range(len(ys32)):
                for ix in range(len(xs32)):
                    s = states[b * N + a].clone()
                    s[x_dim], s[y_dim] = xs32[ix], ys32[iy]
                    rows.append(s)
                    nodes.append(b * N + a)
    return torch.stack(rows), torch.tensor(nodes, dtype=torch.int64)


def probe_graph(env, states, x, edge_index, n, N, B, agents, x_dim, y_dim, xs, ys, relink):
    """(x_all [B*N + T, nd], edge_index [2, E'], edge_attr [E', ed], counts [T]) of the virtual graph, per probe in order."""
    sp, nodes = probe_states(states, N, B, agents, x_dim, y_dim, xs, ys)
    Nt, T = B * N, sp.shape[0]
    pd = O.ENV_PARAMS[env]['pos_dim']
    src, dst, counts = [], [], []
    for t in range(T):
        node = int(nodes[t])
        b, a = node // N, node % N
        if relink:
            g = states[b * N:(b + 1) * N].clone()
            g[a] = sp[t]
            pos = g[:n, :pd] if env == 'SimpleCar' else g[:, :pd]
            ei = O.radius_graph(env, pos, n)
            s = ei[0][ei[1] == a] + b * N
        else:
            s = edge_index[0][edge_index[1] == node]
        src.append(s)
        dst.append(torch.full_like(s, Nt + t))
        counts.append(int(s.numel()))
    src = torch.cat(src) if src else torch.zeros(0, dtype=torch.int64)
    dst = torch.cat(dst) if dst else torch.zeros(0, dtype=torch.int64)
    g_src = O.edge_feature_state(env, states)[src]
    g_dst = O.edge_feature_state(env, sp)[dst - Nt]
    x_all = torch.cat([x, x[nodes]], dim=0)
    return x_all, torch.stack([src, dst]), g_src - g_dst, counts


def field(sd, env, states, x, edge_index, n, N, B, agents, x_dim, y_dim, xs, ys, relink):
    """h [T] of every probe through the oracle CBF (mutates the spectral-norm vectors of `sd` by one power iteration)."""
    x_all, ei, ea, _ = probe_graph(env, states, x, edge_index, n, N, B, agents, x_dim, y_dim, xs, ys, relink)
    mask = torch.zeros(x_all.shape[0], dtype=torch.bool)
    mask[B * N:] = True
    with torch.no_grad():
        return O.cbf_forward(sd, x_all, ea, ei, mask).reshape(-1)
