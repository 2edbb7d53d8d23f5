"""CPU tests of the CBF-condition field (GCBF.cbf_condition_field, csrc/condition.cu):
  1. the two-hop count / fill kernel bodies (csrc/condition_kernels.cuh) on an emulated grid, in several launch geometries and split
     into chunks, against a construction from explicit copies of the graph (tests/condition_oracle.py), three envs, fixed and relink:
     row sets, edge lists in the copy's order, a' as a source of j', obstacle sources, a probe without in-edges, goal rows;
  2. argument checks of GCBF.cbf_condition_field and of the C entry points, none of which needs a GPU.
"""
import ctypes

import numpy as np
import pytest
import torch

import condition_oracle as CO
import gcbf_oracle as O
from test_cbf_field_cpu import ENV_ID, _build, _ea_equal, _grid_case, _p


@pytest.fixture(scope='module')
def cgrid():
    return _build('condition_grid')


def _excl(v, start=0):
    return start + np.concatenate([[0], np.cumsum(v)[:-1]]) if len(v) else np.zeros(0, np.int64)


def _run(cgrid, env_name, sb, n, N, B, x, ei, agents, x_dim, y_dim, xs, ys, relink, grid, block, goal, goal_gstride, chunks):
    p = O.ENV_PARAMS[env_name]
    states = sb.states.contiguous()
    sd = states.shape[1]
    nodes = B * N
    rowptr = torch.zeros(nodes + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(torch.bincount(ei[1], minlength=nodes), 0).to(torch.int32)
    ag = torch.tensor(agents, dtype=torch.int32)
    xs_t, ys_t = torch.tensor(xs, dtype=torch.float32), torch.tensor(ys, dtype=torch.float32)
    T = B * len(agents) * len(xs) * len(ys)
    metric = 0 if env_name == 'SimpleCar' else 1
    common = (_p(states), sd, sd, B, N, n, _p(ag), len(agents), x_dim, y_dim, _p(xs_t), _p(ys_t), len(xs), len(ys), p['pos_dim'],
              ctypes.c_float(p['comm_radius']), metric, 1 if relink else 0, _p(rowptr), _p(ei.contiguous()))
    counts = torch.full((3, T), -7, dtype=torch.int32)
    cgrid.grid_cond_count(grid, block, *common, ctypes.c_int64(T), _p(counts))
    c = counts.numpy().astype(np.int64)
    nd, ed, gd = x.shape[1], {'SimpleCar': 4, 'DubinsCar': 5, 'SimpleDrone': 6}[env_name], goal.shape[1]
    out = []
    for t0, t1 in chunks:
        sl = slice(t0, t1)
        Tc = t1 - t0
        Ea, Rc = int(c[0, sl].sum()), Tc + int(c[1, sl].sum())
        E = Ea + int(c[2, sl].sum())
        off = torch.from_numpy(np.concatenate([_excl(c[0, sl]), _excl(c[1, sl], Tc), _excl(c[2, sl], Ea)]).astype(np.int32))
        pad = 5
        x_out = torch.full((Rc + pad, nd), -9.0)
        st_out = torch.full((Rc + pad, sd), -9.0)
        g_out = torch.full((Rc + pad, gd), -9.0)
        rows = torch.full((Rc + pad, 3), -9, dtype=torch.int64)
        ei_out = torch.full((2 * E + pad,), -9, dtype=torch.int64)
        ea_out = torch.full((E * ed + pad,), -9.0)
        cgrid.grid_cond_fill(grid, block, ENV_ID[env_name], *common, ctypes.c_int64(t0), Tc, _p(off), ctypes.c_int64(Rc), _p(x.contiguous()),
                             nd, _p(goal), gd, gd, goal_gstride, _p(x_out), _p(st_out), _p(g_out), _p(rows), _p(ei_out), ctypes.c_int64(E),
                             _p(ea_out))
        for t in (x_out, st_out, g_out, rows):
            assert bool((t[Rc:] == -9).all())                                           # padding never written
        assert bool((ei_out[2 * E:] == -9).all()) and bool((ea_out[E * ed:] == -9.0).all())
        out.append(dict(rows=rows[:Rc], x=x_out[:Rc], states=st_out[:Rc], goal=g_out[:Rc], edge_index=ei_out[:2 * E].view(2, E),
                        edge_attr=ea_out[:E * ed].view(E, ed), Ea=Ea, Rc=Rc, t0=t0, t1=t1))
    return counts, out


def _restrict(want, T, R, t0, t1):
    """the oracle's single-chunk graph restricted to probes [t0, t1), renumbered as one chunk of its own"""
    rows, ei = want['rows'], want['edge_index']
    keep = (rows[:, 2] >= t0) & (rows[:, 2] < t1)
    old = torch.nonzero(keep).view(-1)
    Rc = int(old.numel())
    new = torch.full((R,), -1, dtype=torch.int64)
    a_keep = old[old < T]
    new[a_keep] = torch.arange(a_keep.numel())
    j_keep = old[old >= T]
    new[j_keep] = a_keep.numel() + torch.arange(j_keep.numel())
    esel = keep[ei[1]]
    src, dst = ei[0][esel], ei[1][esel]
    src = torch.where(src < R, new[src.clamp(max=R - 1)], src - R + Rc)
    order = torch.argsort(new[dst], stable=True)
    return dict(rows=rows[old][torch.argsort(new[old])], edge_index=torch.stack([src, new[dst]])[:, order],
                edge_attr=want['edge_attr'][esel][order], x=want['x'][old][torch.argsort(new[old])],
                states=want['states'][old][torch.argsort(new[old])])


@pytest.mark.parametrize('relink', [False, True])
@pytest.mark.parametrize('env_name', ['SimpleCar', 'DubinsCar', 'SimpleDrone'])
def test_emulated_kernels_equal_explicit_copies(cgrid, env_name, relink):
    sb, n, N, B, x, ei = _grid_case(env_name, 21)
    agents = [0, 1, n - 1]
    x_dim, y_dim = (2, 3) if (env_name == 'DubinsCar' and not relink) else (0, 1)
    xs, ys = np.linspace(0.1, 1.4, 4).astype(np.float32), np.linspace(-0.2, 1.3, 3).astype(np.float32)
    want = CO.two_hop_graph(env_name, sb.states, x, ei, n, N, B, agents, x_dim, y_dim, xs, ys, relink)
    T = B * len(agents) * len(xs) * len(ys)
    R = int(want['rows'].shape[0])
    a_counts = want['counts'][0].tolist()
    assert 0 in a_counts and max(a_counts) > 0                     # graph 1's agent 0 has no neighbours, others have
    assert int(want['counts'][1].sum()) > 0                         # agent sources: j' rows exist
    wei = want['edge_index']
    assert bool(((wei[0] < T) & (wei[1] >= T)).any())               # a' is a source of j'
    if env_name != 'SimpleCar':
        assert bool(((wei[0] >= R + 0) & ((wei[0] - R) % N >= n) & (wei[1] < T)).any())   # obstacle sources of a'
    gd = 4 if env_name == 'DubinsCar' else (6 if env_name == 'SimpleDrone' else 2)
    goal = torch.arange(B * n * gd, dtype=torch.float32).view(B * n, gd) + 0.5
    for grid, block in ((1, 1), (1, 7), (3, 5), (T + 3, 2)):        # one thread .. more threads than probes
        counts, out = _run(cgrid, env_name, sb, n, N, B, x, ei, agents, x_dim, y_dim, xs, ys, relink, grid, block, goal, n, [(0, T)])
        assert torch.equal(counts, want['counts'])
        o = out[0]
        assert torch.equal(o['rows'], want['rows'])
        assert torch.equal(o['edge_index'], wei) and o['Ea'] == want['num_moved_edges']
        assert _ea_equal(env_name, o['edge_attr'], want['edge_attr'], sb.states)
        assert torch.equal(o['x'], want['x']) and torch.equal(o['states'], want['states'])
        r = want['rows']
        local = r[:, 1] % N + (r[:, 1] // N) * n
        assert torch.equal(o['goal'], goal[local])                  # per-graph goal rows
    # shared goals, and chunks that split agents' grids
    splits = [(0, 5), (5, 17), (17, T)]
    _, out = _run(cgrid, env_name, sb, n, N, B, x, ei, agents, x_dim, y_dim, xs, ys, relink, 2, 3, goal[:n].contiguous(), 0, splits)
    for o in out:
        w = _restrict(want, T, R, o['t0'], o['t1'])
        assert torch.equal(o['rows'], w['rows']) and torch.equal(o['edge_index'], w['edge_index'])
        assert _ea_equal(env_name, o['edge_attr'], w['edge_attr'], sb.states)
        assert torch.equal(o['goal'], goal[o['rows'][:, 1] % N])


# ---- 2. argument checks -----------------------------------------------------------------------------------------------------------
def _cpu_algo(env_name='DubinsCar', n=4, obs=2):
    from gcbf_b200.synth import seeded_algo
    return seeded_algo(env_name, n, torch.device('cpu'), 0, {'num_obs': obs, 'area_size': 1.0})


def test_condition_field_rejects_bad_arguments_before_any_launch():
    from gcbf_b200.data import Data
    env, algo = _cpu_algo()
    N = env.nodes_per_graph
    data = Data(x=torch.zeros(N, 4), states=torch.rand(N, 4), edge_index=torch.zeros(2, 0, dtype=torch.int64))
    lims = (torch.zeros(4), torch.ones(4))
    for kw, exc in ((dict(agents=4), ValueError), (dict(agents=-1), ValueError), (dict(agents=[]), ValueError), (dict(x_dim=4), ValueError),
                    (dict(x_dim=1, y_dim=1), ValueError), (dict(y_dim=-1), ValueError), (dict(n_mesh=1), ValueError),
                    (dict(max_probes=0), ValueError), (dict(max_edges=0), ValueError), (dict(max_edges=1 << 31), ValueError),
                    (dict(), RuntimeError), (dict(relink=True), RuntimeError)):
        with pytest.raises(exc):
            algo.cbf_condition_field(data, lims=lims, **kw)
        if 'max_probes' not in kw and 'max_edges' not in kw:        # the probe-graph export has no chunk bounds
            with pytest.raises(exc):
                algo.cbf_condition_field_probe_graph(data, lims=lims, **kw)
    with pytest.raises(RuntimeError, match='CUDA'):
        algo.cbf_condition_field(data, lims=lims)


def test_condition_field_refuses_macbf_and_nominal():
    from gcbf_b200.algo import make_algo
    from gcbf_b200.data import Data
    from gcbf_b200.env import make_env
    env = make_env('SimpleCar', 4, torch.device('cpu'))
    data = Data(x=torch.zeros(4, 4), states=torch.rand(4, 4), edge_index=torch.zeros(2, 0, dtype=torch.int64))
    algo = make_algo('macbf', env, 4, env.node_dim, env.edge_dim, env.action_dim, torch.device('cpu'), 64, None)
    with pytest.raises(NotImplementedError):
        algo.cbf_condition_field(data, lims=(torch.zeros(4), torch.ones(4)))
    nominal = make_algo('nominal', env, 4, env.node_dim, env.edge_dim, env.action_dim, torch.device('cpu'), 64, None)
    assert not hasattr(nominal, 'cbf_condition_field')             # no CBF, no condition


def test_entry_points_reject_bad_descriptors_without_a_gpu():
    from gcbf_b200 import _C, native
    env, algo = _cpu_algo()
    spec = algo.cbf.feat_transformer.module_0.net_spec(algo.cbf.feat_2_CBF)
    fake = 1 << 20

    def desc(**kw):
        d = native.FieldDesc()
        ctypes.memmove(ctypes.byref(d.cbf), ctypes.byref(native.make_net_desc(spec, 0, None)), ctypes.sizeof(native.NetDesc))
        ctypes.memmove(ctypes.byref(d.env), ctypes.byref(env._cfg(2)), ctypes.sizeof(_C.EnvCfg))
        d.states = d.x = d.edge_index = d.rowptr = d.agents = d.xs = d.ys = fake
        d.num_edges, d.max_edges, d.max_probes = 10, 4096, 512
        d.ld_state, d.state_dim, d.pos_dim, d.graph_metric, d.comm_radius = 4, 4, 2, 1, 1.0
        d.num_probe_agents, d.x_dim, d.y_dim, d.nx, d.ny = 2, 0, 1, 30, 30
        for k, v in kw.items():
            setattr(d, k, v)
        return d
    count, fill = native.fn('gcbf_cbf_condition_probe_count'), native.fn('gcbf_cbf_condition_probe_fill')

    def fill_call(d, **kw):
        a = dict(goal=fake, ld_goal=4, goal_dim=4, gpg=0, t0=0, num=100, off=fake, src_off=4000, x_out=fake, st=fake, g_out=fake,
                 rows=None, ei=fake, E=10, ea=fake)
        a.update(kw)
        return fill(ctypes.byref(d), a['goal'], a['ld_goal'], a['goal_dim'], a['gpg'], a['t0'], a['num'], a['off'], a['src_off'], a['x_out'],
                    a['st'], a['g_out'], a['rows'], a['ei'], a['E'], a['ea'], None)
    for bad in (dict(x_dim=-1), dict(y_dim=0), dict(nx=0), dict(agents=None), dict(rowptr=None), dict(graph_metric=2), dict(state_dim=6),
                dict(num_probe_agents=0), dict(pos_dim=4)):
        assert count(ctypes.byref(desc(**bad)), fake, None) == -1, bad
        assert fill_call(desc(**bad)) == -1, bad
    assert count(ctypes.byref(desc()), None, None) == -1
    T = 2 * 2 * 30 * 30
    for bad in (dict(t0=-1), dict(t0=T - 10, num=11), dict(num=-1), dict(E=-1), dict(E=1 << 31), dict(src_off=-1), dict(goal_dim=7),
                dict(ld_goal=2), dict(goal=None), dict(off=None), dict(x_out=None), dict(st=None), dict(g_out=None), dict(ei=None),
                dict(ea=None)):
        assert fill_call(desc(), **bad) == -1, bad
    d = desc()
    d.cbf.node_dim = 0
    assert fill_call(d) == -1
