"""CPU tests of the CBF level-set field (GCBF.cbf_field, gcbf_cbf_field):
  1. the probe-graph oracle (tests/field_oracle.py) reproduces the reference's plot_cbf_contour fields (tests/golden/cbf_field, made by
     oracle/make_field_golden.py) and their grids;
  2. state_lim and the plotting-box formula against the fixtures;
  3. the per-element functions (csrc/field_core.h, csrc/graph_core.h via tests/host_driver/field_host.cpp) against the oracle, bit for
     bit, including grid points within 3 ulps of the communication radius;
  4. the count / fill kernel bodies (csrc/field_kernels.cuh) on an emulated grid against a brute-force construction, both modes;
  5. argument checks of GCBF.cbf_field and of the C entry points, none of which needs a GPU.
"""
import ctypes
import glob
import os
import subprocess

import numpy as np
import pytest
import torch

import field_oracle as FO
import gcbf_oracle as O
from conftest import GOLDEN_DIR, ROOT
from helpers import sd_clone
import make_field_golden as MFG

ENV_ID = {'SimpleCar': 0, 'DubinsCar': 1, 'SimpleDrone': 2}
FIELD_DIR = os.path.join(GOLDEN_DIR, 'cbf_field')
FIXTURES = sorted(os.path.basename(p)[:-3] for p in glob.glob(os.path.join(FIELD_DIR, '*.pt')))
TOL = 1e-5


def _build(name):
    out = os.path.join(ROOT, 'tests', 'host_driver', '_build')
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, name + '.so')
    subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-I', os.path.join(ROOT, 'gcbf-pytorch_b200', 'csrc'),
                           '-I', os.path.join(ROOT, 'include'), '-I', os.path.join(ROOT, 'tests', 'host_driver'), '-o', so,
                           os.path.join(ROOT, 'tests', 'host_driver', name + '.cpp')])
    return ctypes.CDLL(so)


@pytest.fixture(scope='module')
def fhost():
    return _build('field_host')


@pytest.fixture(scope='module')
def fgrid():
    return _build('field_grid')


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None and t.numel() else None


def load_fixture(name):
    return torch.load(os.path.join(FIELD_DIR, name + '.pt'), weights_only=False)


def fixture_cbf(fix, device='cpu'):
    """The product's GCBF on `device` with the fixture's CBF weights (seeded init, head gain) and u, v."""
    from gcbf_b200.synth import seeded_algo
    m = fix['meta']
    env, algo = seeded_algo(m['env'], m['n'], torch.device(device), m['init_seed'], {'num_obs': m['obs'], 'area_size': m['area']})
    assert m['head_gain'] == MFG.HEAD_GAIN
    sd = MFG.field_weights(sd_clone(algo.cbf))
    sd.update({k: v.clone() for k, v in fix['uv_before'].items()})
    algo.cbf.load_state_dict({k: v.to(device) for k, v in sd.items()})
    return env, algo


# ---- 1. the oracle's probe graphs against the reference's copies ------------------------------------------------------------------
def test_fixtures_exist():
    assert len(FIXTURES) == 5, FIXTURES


@pytest.mark.parametrize('name', FIXTURES)
def test_probe_oracle_equals_reference_fixture(name):
    from gcbf_b200.algo.gcbf import GCBF
    fix = load_fixture(name)
    m = fix['meta']
    xs, ys = GCBF.field_grid(fix['state_lim'], m['x_dim'], m['y_dim'], m['n_mesh'])
    assert np.array_equal(xs, fix['xs']) and xs.dtype == fix['xs'].dtype       # the grid is the reference's np.linspace, bit for bit
    assert np.array_equal(ys, fix['ys']) and ys.dtype == fix['ys'].dtype
    _, algo = fixture_cbf(fix)
    sd = sd_clone(algo.cbf)
    N = fix['states'].shape[0]
    h = FO.field(sd, m['env'], fix['states'], fix['x'], fix['edge_index'], m['n'], N, 1, [m['agent']], m['x_dim'], m['y_dim'], xs, ys,
                 relink=False).reshape(m['n_mesh'], m['n_mesh'])
    ref = fix['field']
    assert float((h - ref).abs().max()) <= TOL, float((h - ref).abs().max())
    if m['name'].endswith('isolated'):
        assert int((fix['edge_index'][1] == m['agent']).sum()) == 0 and float(ref.max() - ref.min()) == 0.0
    else:
        assert float(ref.max() - ref.min()) >= 100 * TOL                           # the field discriminates at the tolerance
    for k, v in fix['uv_after'].items():                                          # one power iteration, as the reference's one call
        assert torch.allclose(sd[k], v, rtol=0, atol=1e-6), k


# ---- 2. state_lim ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', FIXTURES)
def test_state_lim_and_box_formula_equal_the_fixture(name):
    from gcbf_b200.env import make_env
    from gcbf_b200.env.base import plot_box
    fix = load_fixture(name)
    m = fix['meta']
    env = make_env(m['env'], m['n'], torch.device('cpu'), params={**make_env(m['env'], m['n'], torch.device('cpu')).default_params,
                                                                  'num_obs': m['obs'], 'area_size': m['area']})
    if m['env'] != 'SimpleDrone':
        with pytest.raises(RuntimeError, match='reset'):
            env.state_lim
        n = m['n']
        pts = [fix['states'][:n, :2], fix['goals'][:, :2]] + ([fix['obstacles'][:, :2]] if m['env'] == 'DubinsCar' else [])
        env._xy_min, env._xy_max = plot_box(torch.cat(pts).numpy(), env._params[env.RADIUS_KEY])
    lo, hi = env.state_lim
    for got, want in ((lo, fix['state_lim'][0]), (hi, fix['state_lim'][1])):
        assert got.dtype == want.dtype and torch.equal(got, want), (got, want)


def test_reset_sets_a_square_box_around_agents_and_goals():
    from gcbf_b200.env import make_env
    for name in ('SimpleCar', 'DubinsCar'):
        env = make_env(name, 6, torch.device('cpu'), params={**make_env(name, 6, torch.device('cpu')).default_params, 'num_obs': 2})
        torch.manual_seed(3)
        try:
            env.reset()
        except RuntimeError:          # the radius graph needs CUDA; the box is set before it
            pass
        lo, hi = env.state_lim
        assert torch.isclose(hi[0] - lo[0], hi[1] - lo[1]) and lo.dtype == torch.float32


# ---- 3. per-element functions ----------------------------------------------------------------------------------------------------
def test_probe_state_and_index(fhost):
    s = torch.tensor([0.5, -1.25, 2.0, 0.3, 7.0, -2.0])
    out = torch.empty(6)
    fhost.host_probe_state(_p(s), 6, 4, ctypes.c_float(1.5), 1, ctypes.c_float(-0.75), _p(out))
    want = s.clone()
    want[4], want[1] = 1.5, -0.75
    assert torch.equal(out, want)
    idx = (ctypes.c_int64 * 4)()
    for t in (0, 1, 29, 30, 899, 900, 3 * 900 * 5 + 17):
        fhost.host_probe_index(t, 5, 30, 30, idx)
        b, ai, iy, ix = idx
        assert ((b * 5 + ai) * 30 + iy) * 30 + ix == t and 0 <= ai < 5 and 0 <= iy < 30 and 0 <= ix < 30


def _trig_close(got, want, vmax):
    """v cos(theta) - v' cos(theta') (and sin) from two faithful but different cosf / sinf: within 2 ulps of max |v| per term."""
    return got.numel() == 0 or float((got - want).abs().max()) <= 4 * float(torch.finfo(torch.float32).eps) * float(vmax)


def _ea_equal(env_name, got, want, states):
    """edge features bit for bit; DubinsCar's trig columns to _trig_close"""
    if env_name != 'DubinsCar':
        return torch.equal(got, want)
    return torch.equal(got[:, :3], want[:, :3]) and _trig_close(got[:, 3:], want[:, 3:], states[:, 3].abs().max())


@pytest.mark.parametrize('env_name', ['SimpleCar', 'DubinsCar', 'SimpleDrone'])
def test_probe_edge_attr_matches_the_oracle(fhost, env_name):
    sd = 6 if env_name == 'SimpleDrone' else 4
    g = torch.Generator().manual_seed(4)
    states = (torch.rand(64, sd, generator=g) * 6 - 3).float()
    ed = {'SimpleCar': 4, 'DubinsCar': 5, 'SimpleDrone': 6}[env_name]
    ei = torch.stack([torch.arange(0, 32), torch.arange(32, 64)])
    want = O.edge_attr(env_name, states, ei)
    out = torch.empty(ed)
    # bit for bit, except DubinsCar's v cos(theta), v sin(theta): the host's libm cosf / sinf and torch's vectorised ones are both faithful
    # but not the same function (the GPU build uses CUDA's cosf / sinf), so those two columns agree to 2 ulps of their operands
    exact = 3 if env_name == 'DubinsCar' else ed
    for e in range(32):
        fhost.host_probe_edge_attr(ENV_ID[env_name], _p(states[e].contiguous()), _p(states[32 + e].contiguous()), _p(out))
        assert torch.equal(out[:exact], want[e, :exact]), (e, out, want[e])
        assert _trig_close(out[exact:], want[e, exact:], states[[e, 32 + e], 3].abs().max()), (e, out, want[e])


@pytest.mark.parametrize('env_name', ['SimpleCar', 'DubinsCar', 'SimpleDrone'])
def test_pair_rule_at_the_radius_boundary(fhost, env_name):
    """Grid points placed within 3 ulps of the communication radius on both sides: the host build of the pair rule decides every one as
    the oracle's radius graph does."""
    p = O.ENV_PARAMS[env_name]
    r, pd = float(p['comm_radius']), p['pos_dim']
    metric = 0 if env_name == 'SimpleCar' else 1
    g = torch.Generator().manual_seed(7)
    base = (torch.rand(pd, generator=g) * 2).float()
    hits = {True: 0, False: 0}
    for trial in range(60):
        d = torch.nn.functional.normalize(torch.randn(pd, generator=g), dim=0)
        x = np.float32(r)
        for k in range(-3, 4):
            rr = x
            for _ in range(abs(k)):
                rr = np.nextafter(rr, np.float32(np.inf if k > 0 else -np.inf), dtype=np.float32)
            q = (base + d * float(rr)).float()
            pos = torch.stack([q, base])
            ei = O.radius_graph(env_name, pos, 2 if env_name == 'SimpleCar' else 1)
            want = bool(((ei[0] == 1) & (ei[1] == 0)).any())
            got = bool(fhost.host_pair_hit(_p(q.contiguous()), _p(base.contiguous()), pd, ctypes.c_float(r), metric))
            assert got == want, (trial, k)
            hits[want] += 1
    assert hits[True] > 0 and hits[False] > 0


# ---- 4. kernel bodies on the emulated grid ---------------------------------------------------------------------------------------
def _grid_case(env_name, seed):
    from gcbf_b200 import synth
    n, obs, B, area = {'SimpleCar': (6, 0, 2, 1.5), 'DubinsCar': (5, 3, 2, 1.5), 'SimpleDrone': (4, 4, 2, 0.8)}[env_name]
    sb = synth.make_states(env_name, n, obs, B, area, seed)
    N = sb.nodes_per_graph
    ei = O.batch_radius_graph(env_name, sb.states, B, N, n)
    x, _ = O.make_graph_inputs(env_name, sb.states, B, n, sb.num_obs)
    # an agent without neighbours: graph 1's agent 0 moved far away
    sb.states[N, :O.ENV_PARAMS[env_name]['pos_dim']] += 50.0
    ei = O.batch_radius_graph(env_name, sb.states, B, N, n)
    return sb, n, N, B, x, ei


def _run_grid(fgrid, env_name, sb, n, N, B, x, ei, agents, x_dim, y_dim, xs, ys, relink, grid, block, src_off=0):
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
    common = (_p(states), sd, sd, B, N, _p(ag), len(agents), x_dim, y_dim, _p(xs_t), _p(ys_t), len(xs), len(ys), p['pos_dim'],
              ctypes.c_float(p['comm_radius']), metric, 1 if relink else 0, _p(rowptr), _p(ei.contiguous()))
    counts = torch.full((T,), -7, dtype=torch.int32)
    fgrid.grid_probe_count(grid, block, *common, ctypes.c_int64(T), _p(counts))
    E = int(counts.sum())
    rp = torch.zeros(T + 1, dtype=torch.int32)
    rp[1:] = torch.cumsum(counts, 0)
    nd = x.shape[1]
    ed = {'SimpleCar': 4, 'DubinsCar': 5, 'SimpleDrone': 6}[env_name]
    pad = 5
    x_out = torch.full((T + pad, nd), -9.0)
    ei_out = torch.full((2 * E + pad,), -9, dtype=torch.int64)
    ea_out = torch.full((E * ed + pad,), -9.0)
    # targets numbered after the original nodes, as the brute-force construction does
    fgrid.grid_probe_fill(grid, block, ENV_ID[env_name], *common, ctypes.c_int64(0), T, _p(rp), ctypes.c_int64(src_off), ctypes.c_int64(nodes),
                          _p(x.contiguous()), nd, _p(x_out), _p(ei_out), ctypes.c_int64(E), _p(ea_out))
    return counts, x_out, ei_out, ea_out, E, nodes, T, pad


@pytest.mark.parametrize('relink', [False, True])
@pytest.mark.parametrize('env_name', ['SimpleCar', 'DubinsCar', 'SimpleDrone'])
def test_emulated_kernels_equal_brute_force_probe_graphs(fgrid, env_name, relink):
    sb, n, N, B, x, ei = _grid_case(env_name, 21)
    agents = [0, n - 1]
    x_dim, y_dim = (2, 3) if (env_name == 'DubinsCar' and not relink) else (0, 1)
    xs, ys = np.linspace(0.1, 1.4, 4).astype(np.float32), np.linspace(-0.2, 1.3, 3).astype(np.float32)
    x_want, ei_want, ea_want, c_want = FO.probe_graph(env_name, sb.states, x, ei, n, N, B, agents, x_dim, y_dim, xs, ys, relink)
    assert 0 in c_want and max(c_want) > 0          # graph 1's agent 0 has no neighbours, others have
    T = len(c_want)
    for grid, block in ((1, 1), (1, 7), (3, 5), (T + 3, 2)):         # one thread .. more threads than probes
        counts, x_out, ei_out, ea_out, E, nodes, T, pad = _run_grid(fgrid, env_name, sb, n, N, B, x, ei, agents, x_dim, y_dim, xs, ys,
                                                                    relink, grid, block)
        assert counts.tolist() == c_want
        assert torch.equal(ei_out[:2 * E].view(2, E), ei_want)
        assert _ea_equal(env_name, ea_out[:E * ea_want.shape[1]].view(E, -1), ea_want, sb.states)
        assert torch.equal(x_out[:T], x_want[nodes:])
        assert bool((x_out[T:] == -9.0).all())                                                          # padding never written
        assert bool((ei_out[2 * E:] == -9).all()) and bool((ea_out[E * ea_want.shape[1]:] == -9.0).all())
    _, _, ei_off, _, E, _, _, _ = _run_grid(fgrid, env_name, sb, n, N, B, x, ei, agents, x_dim, y_dim, xs, ys, relink, 2, 3, src_off=7)
    assert torch.equal(ei_off[:E], ei_want[0] + 7) and torch.equal(ei_off[E:2 * E], ei_want[1])      # the chunk layout's source offset


# ---- 5. argument checks -----------------------------------------------------------------------------------------------------------
def _cpu_algo(env_name='DubinsCar', n=4, obs=2):
    from gcbf_b200.synth import seeded_algo
    return seeded_algo(env_name, n, torch.device('cpu'), 0, {'num_obs': obs, 'area_size': 1.0})


def test_cbf_field_rejects_bad_arguments_before_any_launch():
    from gcbf_b200.data import Data
    env, algo = _cpu_algo()
    N = env.nodes_per_graph
    data = Data(x=torch.zeros(N, 4), states=torch.rand(N, 4), edge_index=torch.zeros(2, 0, dtype=torch.int64))
    lims = (torch.zeros(4), torch.ones(4))
    for kw, exc in ((dict(agents=4), ValueError), (dict(agents=-1), ValueError), (dict(agents=[]), ValueError), (dict(x_dim=4), ValueError),
                    (dict(x_dim=1, y_dim=1), ValueError), (dict(y_dim=-1), ValueError), (dict(n_mesh=1), ValueError),
                    (dict(max_probes=0), ValueError), (dict(), RuntimeError)):
        with pytest.raises(exc):
            algo.cbf_field(data, lims=lims, **kw)
    with pytest.raises(RuntimeError, match='CUDA'):
        algo.cbf_field(data, lims=lims)


def test_cbf_field_refuses_macbf():
    from gcbf_b200.algo import make_algo
    from gcbf_b200.data import Data
    from gcbf_b200.env import make_env
    env = make_env('SimpleCar', 4, torch.device('cpu'))
    algo = make_algo('macbf', env, 4, env.node_dim, env.edge_dim, env.action_dim, torch.device('cpu'), 64, None)
    data = Data(x=torch.zeros(4, 4), states=torch.rand(4, 4), edge_index=torch.zeros(2, 0, dtype=torch.int64))
    with pytest.raises(NotImplementedError):
        algo.cbf_field(data, lims=(torch.zeros(4), torch.ones(4)))


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
    q, call = native.fn('gcbf_cbf_field_workspace_bytes'), native.fn('gcbf_cbf_field')
    good = q(ctypes.byref(desc()))
    assert good > 0, _C.lib().gcbf_last_error()
    assert q(ctypes.byref(desc(max_edges=1024))) < good                       # the edge bound sizes the workspace ...
    assert q(ctypes.byref(desc(max_edges=8192))) == good                      # ... up to what 512 probes x 5 sources can have
    for bad in (dict(x_dim=1), dict(y_dim=4), dict(x_dim=-1), dict(state_dim=6), dict(num_probe_agents=0), dict(agents=None),
                dict(nx=0), dict(max_probes=0), dict(max_edges=0), dict(max_edges=1 << 31), dict(pos_dim=4), dict(graph_metric=2),
                dict(rowptr=None)):
        d = desc(**bad)
        assert q(ctypes.byref(d)) == 0, bad
        assert call(ctypes.byref(d), fake, None, fake, 1 << 40, None) == -1, bad
    d = desc()
    d.cbf.head[d.cbf.n_head - 1].N = 2                                        # not a CBF head
    assert q(ctypes.byref(d)) == 0
    assert call(ctypes.byref(desc()), None, None, fake, 1 << 40, None) == -1                  # no output
    assert call(ctypes.byref(desc()), fake, None, fake + 8, 1 << 40, None) == -1              # misaligned workspace
    assert call(ctypes.byref(desc()), fake, None, fake, 1024, None) == native.E_WORKSPACE     # too small: refused before any launch
    assert ctypes.sizeof(native.FieldDesc) == _C.lib().gcbf_abi_struct_size(13)
    count, fill = native.fn('gcbf_cbf_field_probe_count'), native.fn('gcbf_cbf_field_probe_fill')
    for bad in (dict(x_dim=-1), dict(nx=0), dict(agents=None), dict(rowptr=None), dict(graph_metric=2)):
        assert count(ctypes.byref(desc(**bad)), fake, None) == -1, bad
        assert fill(ctypes.byref(desc(**bad)), fake, fake, 10, fake, None) == -1, bad
    assert count(ctypes.byref(desc()), None, None) == -1
    assert fill(ctypes.byref(desc()), fake, None, 10, fake, None) == -1
    assert fill(ctypes.byref(desc()), fake, fake, -1, fake, None) == -1


def _default_desc(cfg, agents):
    """gcbf_field_desc of GCBF.cbf_field's defaults (30 x 30, default chunk bounds) for one graph of a BASELINE config, on fake
    device pointers: only the workspace query reads it."""
    from gcbf_b200 import _C, native, synth
    from gcbf_b200.algo.gcbf import GCBF
    from gcbf_b200.synth import seeded_algo
    c = synth.CONFIGS[cfg]
    env, algo = seeded_algo(c['env'], c['num_agents'], torch.device('cpu'), 0, {'num_obs': c['num_obs'], 'area_size': c['area_size']})
    spec = algo.cbf.feat_transformer.module_0.net_spec(algo.cbf.feat_2_CBF)
    d = native.FieldDesc()
    ctypes.memmove(ctypes.byref(d.cbf), ctypes.byref(native.make_net_desc(spec, 0, None)), ctypes.sizeof(native.NetDesc))
    ctypes.memmove(ctypes.byref(d.env), ctypes.byref(env._cfg(1)), ctypes.sizeof(_C.EnvCfg))
    fake = 1 << 20
    d.states = d.x = d.edge_index = d.rowptr = d.agents = d.xs = d.ys = fake
    d.num_edges = 10
    N = env.nodes_per_graph
    d.max_probes, d.max_edges = min(agents * 900, GCBF.FIELD_MAX_PROBES), max(GCBF.FIELD_MAX_EDGES, N - 1)
    d.ld_state = d.state_dim = env.state_dim
    d.pos_dim, d.graph_metric, d.comm_radius = env.POS_DIM, env.GRAPH_METRIC, 1.0
    d.num_probe_agents, d.x_dim, d.y_dim, d.nx, d.ny = agents, 0, 1, 30, 30
    return native.fn('gcbf_cbf_field_workspace_bytes')(ctypes.byref(d))


def test_workspace_scales_with_the_call():
    """A chunk is sized for what its probes can have (at most nodes_per_graph - 1 sources each), not for the default edge bound: one
    C1 agent on a 30 x 30 grid (900 probes, <= 13,500 edges) needs a fraction of what all 1024 agents of a C3-sized graph need."""
    c1, c3 = _default_desc('C1', 1), _default_desc('C3', 1024)
    assert 0 < c1 < 0.5e9 and c3 > 10 * c1, (c1, c3)
