"""CPU oracle of the CBF-condition field's two-hop probe graphs (GCBF.cbf_condition_field_probe_graph), built from explicit copies:
for probe t (agent a of graph b moved to s'_t, as in field_oracle.py) the copy G' is graph b with a moved, and keeps the given edges
(fixed) or gets the oracle radius graph of its states (relink).  Its rows are
  a'  (kind 0, node of a, t): the in-edges of a in G', in G''s order;
  j'  (kind 1, node of j, t): one per agent source j of a, in that order, with the in-edges of j in G', in G''s order;
with all a' rows first (probe order), then all j' rows (probe order, then a'-edge order).  Edges are target-sorted; an a' edge from an
agent j reads the j' row, a j' edge from a reads the a' row, every other source is row R + original node id.  edge_attr = g(s_src) -
g(s_tgt) with the states of G'.
"""
import torch

import field_oracle as FO
import gcbf_oracle as O


def _copy_edges(env, states, edge_index, n, N, b, a, s_moved, relink):
    """(states of G' [N, sd], local edge list [(src, dst)] of G' in order)"""
    g = states[b * N:(b + 1) * N].clone()
    g[a] = s_moved
    if relink:
        pd = O.ENV_PARAMS[env]['pos_dim']
        pos = g[:n, :pd] if env == 'SimpleCar' else g[:, :pd]
        ei = O.radius_graph(env, pos, n)
    else:
        sel = (edge_index[1] >= b * N) & (edge_index[1] < (b + 1) * N)
        ei = edge_index[:, sel] - b * N
    return g, list(zip(ei[0].tolist(), ei[1].tolist()))


def two_hop_graph(env, states, x, edge_index, n, N, B, agents, x_dim, y_dim, xs, ys, relink):
    """dict(rows [R, 3], edge_index [2, E] over rows, edge_attr [E, ed], states [R, sd], x [R, nd], num_moved_edges,
    counts [3, T] (a' edges, j' rows, j' edges per probe))."""
    sp, nodes = FO.probe_states(states, N, B, agents, x_dim, y_dim, xs, ys)
    T = sp.shape[0]
    a_rows, j_rows = [], []            # (node, t, G' states, local id, edge list of the row's in-edges [(src local, ...)])
    counts = []
    for t in range(T):
        node = int(nodes[t])
        b, a = node // N, node % N
        g, edges = _copy_edges(env, states, edge_index, n, N, b, a, sp[t], relink)
        a_in = [s for s, d in edges if d == a]
        js = [s for s in a_in if s < n]
        a_rows.append((b, a, t, g, a_in, js))
        ej = 0
        for j in js:
            j_in = [s for s, d in edges if d == j]
            j_rows.append((b, j, t, g, j_in, a))
            ej += len(j_in)
        counts.append((len(a_in), len(js), ej))
    R = T + len(j_rows)
    # where the j' rows of each probe start
    j_start, r = [], T
    for (_, _, _, _, _, js) in a_rows:
        j_start.append(r)
        r += len(js)
    rows, st, xr, src, dst, g_src, g_dst = [], [], [], [], [], [], []

    def feat(s):
        return O.edge_feature_state(env, s.unsqueeze(0))[0]
    for i, (b, a, t, g, a_in, js) in enumerate(a_rows):
        rows.append((0, b * N + a, t))
        st.append(g[a])
        xr.append(x[b * N + a])
        k = 0
        for s in a_in:
            if s < n:
                src.append(j_start[i] + k)
                k += 1
            else:
                src.append(R + b * N + s)
            dst.append(i)
            g_src.append(feat(g[s]))
            g_dst.append(feat(g[a]))
    for r, (b, j, t, g, j_in, a) in enumerate(j_rows):
        row = T + r
        rows.append((1, b * N + j, t))
        st.append(g[j])
        xr.append(x[b * N + j])
        for s in j_in:
            src.append(t if s == a else R + b * N + s)
            dst.append(row)
            g_src.append(feat(g[s]))
            g_dst.append(feat(g[j]))
    Ea = sum(c[0] for c in counts)
    ed = O.edge_feature_state(env, states[:1]).shape[1]
    ea = torch.stack(g_src) - torch.stack(g_dst) if src else torch.zeros(0, ed)
    return dict(rows=torch.tensor(rows, dtype=torch.int64), edge_index=torch.tensor([src, dst], dtype=torch.int64).view(2, -1),
                edge_attr=ea, states=torch.stack(st), x=torch.stack(xr), num_moved_edges=Ea,
                counts=torch.tensor(counts, dtype=torch.int32).t().contiguous())
