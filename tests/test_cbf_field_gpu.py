"""GPU tests of the CBF level-set field (GCBF.cbf_field -> gcbf_cbf_field, csrc/field.cu):
  1. fixed mode against the reference's plot_cbf_contour fields (tests/golden/cbf_field), grids bit-equal, u, v after the call equal to
     those after one CBF pass from the same start;
  2. on the fp32 paths (ops.GEMM_IMPL = 1, every row computed independently) bit-equal to this library's CBFGNN over the reference's
     construction (one copy of the graph per grid point); on the default path within 1e-5;
  3. the device-built probe edge lists and edge features, both modes, bit-identical to the in-edges of the agent in the reference's
     copies (relink: ops.radius_graph on the moved state); relink fields within 1e-5 of the per-point oracle on all three envs;
  4. B graphs x A agents in one call equal the per-(graph, agent) calls bit for bit;
  5. chunking (a chunk boundary inside one agent's grid) changes nothing and advances u, v once;
  6. a C3-sized DubinsCar graph, all 1024 agents on an 8 x 8 grid (phi / gamma on the wgmma kernel), against the oracle on sampled agents;
  7. two calls are bit-identical.
"""
import numpy as np
import pytest
import torch

import field_oracle as FO
from helpers import sd_clone
from test_cbf_field_cpu import FIXTURES, TOL, fixture_cbf, load_fixture

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')


def _uv(algo):
    return {k: v.detach().clone() for k, v in algo.cbf.state_dict().items() if k.endswith(('weight_u', 'weight_v'))}


def _set_uv(algo, uv):
    sd = algo.cbf.state_dict()
    with torch.no_grad():
        for k, v in uv.items():
            sd[k].copy_(v)


class gemm_impl:
    def __init__(self, impl):
        self.impl = impl

    def __enter__(self):
        from gcbf_b200 import ops
        self.prev, ops.GEMM_IMPL = ops.GEMM_IMPL, self.impl

    def __exit__(self, *a):
        from gcbf_b200 import ops
        ops.GEMM_IMPL = self.prev


def _graph(env, states, edge_index):
    """Data of B graphs (states [B * N, sd], target-sorted edge_index) with x / agent_mask of the env and the kernels' edge features."""
    from gcbf_b200.data import Data
    g = env.make_graph(states.to(DEV))
    ei = edge_index.to(DEV)
    fields = dict(x=g.x, states=g.states, pos=g.pos, edge_index=ei, edge_attr=env.edge_attr(g.states, ei))
    if hasattr(g, 'agent_mask'):
        fields['agent_mask'] = g.agent_mask
    return Data(**fields)


def _fixture_setup(name):
    fix = load_fixture(name)
    env, algo = fixture_cbf(fix, 'cuda')
    return fix, fix['meta'], env, algo, _graph(env, fix['states'], fix['edge_index'])


def _copies(env, data, agent, x_dim, y_dim, xs, ys, relink):
    """The reference's construction as one Batch: a copy of the graph per grid point (row-major over (iy, ix)), agent moved; edges
    kept (fixed) or rebuilt by the radius-graph kernels (relink)."""
    from gcbf_b200 import ops
    from gcbf_b200.data import Data
    N = data.states.shape[0]
    M = len(xs) * len(ys)
    st = data.states.repeat(M, 1)
    gx, gy = np.meshgrid(np.asarray(xs, np.float32), np.asarray(ys, np.float32))
    rows = torch.arange(M, device=DEV) * N + agent
    st[rows, x_dim] = torch.from_numpy(gx.reshape(-1)).to(DEV)
    st[rows, y_dim] = torch.from_numpy(gy.reshape(-1)).to(DEV)
    if relink:
        ei, _ = ops.radius_graph(st, env.POS_DIM, M, N, env.num_agents, env._params['comm_radius'], env.GRAPH_METRIC)
    else:
        E = data.edge_index.shape[1]
        ei = (data.edge_index.repeat(1, M) + (torch.arange(M, device=DEV) * N).repeat_interleave(E).unsqueeze(0))
    fields = dict(x=data.x.repeat(M, 1), states=st, edge_index=ei, edge_attr=env.edge_attr(st, ei))
    if hasattr(data, 'agent_mask'):
        fields['agent_mask'] = data.agent_mask.repeat(M)
    return Data(**fields), M


def _copies_field(algo, env, data, agent, x_dim, y_dim, xs, ys, relink):
    batch, M = _copies(env, data, agent, x_dim, y_dim, xs, ys, relink)
    with torch.no_grad():
        h = algo.cbf(batch).view(M, env.num_agents)[:, agent]
    return h.reshape(len(ys), len(xs))


# ---- 1. the reference fixtures ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', FIXTURES)
def test_fixed_field_equals_reference_fixture(name):
    fix, m, env, algo, data = _fixture_setup(name)
    uv0 = _uv(algo)
    xs, ys, h = algo.cbf_field(data, agents=m['agent'], x_dim=m['x_dim'], y_dim=m['y_dim'], n_mesh=m['n_mesh'], lims=fix['state_lim'])
    assert np.array_equal(xs, fix['xs']) and np.array_equal(ys, fix['ys']) and xs.dtype == fix['xs'].dtype
    assert tuple(h.shape) == (1, 1, m['n_mesh'], m['n_mesh'])
    err = float((h[0, 0].cpu() - fix['field']).abs().max())
    assert err <= TOL, err
    uv_field = _uv(algo)
    _set_uv(algo, uv0)
    with torch.no_grad():
        algo.cbf(data)                                   # one power iteration from the same start
    for k, v in _uv(algo).items():
        assert torch.equal(uv_field[k], v), k
        # the reference's CPU power iteration, on weights whose seeded init may differ in the last bits between host CPUs
        assert float((v.cpu() - fix['uv_after'][k]).abs().max()) <= TOL, k


# ---- 2. against this library's CBFGNN on the reference's copies -----------------------------------------------------------------------
@pytest.mark.parametrize('name', ['simplecar_n16', 'dubins_n16_o4_theta_v', 'drone_n8_o8'])
@pytest.mark.parametrize('relink', [False, True])
def test_field_equals_cbfgnn_over_copies(name, relink):
    fix, m, env, algo, data = _fixture_setup(name)
    x_dim, y_dim = (m['x_dim'], m['y_dim']) if not relink else (0, 1)
    uv0 = _uv(algo)
    for impl, exact in ((1, True), (0, False)):
        with gemm_impl(impl):
            _set_uv(algo, uv0)
            xs, ys, h = algo.cbf_field(data, agents=m['agent'], x_dim=x_dim, y_dim=y_dim, n_mesh=m['n_mesh'], lims=fix['state_lim'],
                                       relink=relink)
            uv_field = _uv(algo)
            _set_uv(algo, uv0)
            want = _copies_field(algo, env, data, m['agent'], x_dim, y_dim, xs, ys, relink)
        for k, v in _uv(algo).items():
            assert torch.equal(uv_field[k], v), k
        if exact:
            assert torch.equal(h[0, 0], want), float((h[0, 0] - want).abs().max())
        else:
            assert float((h[0, 0] - want).abs().max()) <= TOL


# ---- 3. relink against the per-point oracle ----------------------------------------------------------------------------------------
@pytest.mark.parametrize('name', ['simplecar_n16', 'dubins_n16_o4_xy', 'drone_n8_o8'])
def test_relink_field_equals_oracle(name):
    fix, m, env, algo, data = _fixture_setup(name)
    sd = sd_clone(algo.cbf)
    xs, ys, h = algo.cbf_field(data, agents=m['agent'], x_dim=0, y_dim=1, n_mesh=10, lims=fix['state_lim'], relink=True)
    N = fix['states'].shape[0]
    want = FO.field(sd, m['env'], fix['states'], fix['x'], fix['edge_index'], m['n'], N, 1, [m['agent']], 0, 1, xs, ys, relink=True)
    _, _, _, counts = FO.probe_graph(m['env'], fix['states'], fix['x'], fix['edge_index'], m['n'], N, 1, [m['agent']], 0, 1, xs, ys, True)
    assert len(set(counts)) > 1                           # neighbours enter and leave as the agent moves
    err = float((h.reshape(-1).cpu() - want).abs().max())
    assert err <= TOL, err


# ---- 4. batching ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('env_name,n,obs,area', [('SimpleCar', 8, 0, 2.0), ('DubinsCar', 6, 3, 2.0)])
@pytest.mark.parametrize('relink', [False, True])
def test_batch_equals_per_graph_per_agent_calls(env_name, n, obs, area, relink):
    from gcbf_b200 import synth
    from gcbf_b200.synth import product_batch, seeded_algo
    B = 3
    sb = synth.make_states(env_name, n, obs, B, area, 41)
    env, algo = seeded_algo(env_name, n, DEV, 0, {'num_obs': sb.num_obs, 'area_size': area})
    data = product_batch(env, sb, DEV)
    N = sb.nodes_per_graph
    agents = [0, 2, n - 1]
    lims = (torch.zeros(4), torch.full((4,), area))
    uv0 = _uv(algo)
    with gemm_impl(1):
        _, _, h = algo.cbf_field(data, agents=agents, n_mesh=6, lims=lims, relink=relink)
        for b in range(B):
            one = env.graph_from_states(sb.states[b * N:(b + 1) * N].to(DEV), with_u_ref=False)
            for k, a in enumerate(agents):
                _set_uv(algo, uv0)
                _, _, h1 = algo.cbf_field(one, agents=a, n_mesh=6, lims=lims, relink=relink)
                assert torch.equal(h[b, k], h1[0, 0]), (b, a)


# ---- 5. chunking, 7. reproducibility ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('relink', [False, True])
def test_chunking_and_repeat_calls_change_nothing(relink):
    fix, m, env, algo, data = _fixture_setup('dubins_n16_o4_xy')
    agents = [m['agent'], 0, 3]
    uv0 = _uv(algo)
    with gemm_impl(1):
        _, _, whole = algo.cbf_field(data, agents=agents, n_mesh=8, lims=fix['state_lim'], relink=relink)
        assert algo.last_field_chunks == 1
        _set_uv(algo, uv0)
        _, _, parts = algo.cbf_field(data, agents=agents, n_mesh=8, lims=fix['state_lim'], relink=relink, max_probes=37)
        assert algo.last_field_chunks == -(-3 * 64 // 37)           # boundaries at probe 37, 74, ...: inside agents' grids
        assert torch.equal(whole, parts)
        uv_field = _uv(algo)
        _set_uv(algo, uv0)
        with torch.no_grad():
            algo.cbf(data)
        for k, v in _uv(algo).items():                               # ONE power iteration for all the chunks
            assert torch.equal(uv_field[k], v), k
    _set_uv(algo, uv0)
    _, _, a = algo.cbf_field(data, agents=agents, n_mesh=8, lims=fix['state_lim'], relink=relink)
    _set_uv(algo, uv0)
    _, _, b = algo.cbf_field(data, agents=agents, n_mesh=8, lims=fix['state_lim'], relink=relink)
    assert torch.equal(a, b)                                         # no float atomics: two calls, same bits


def test_edge_bounded_chunks_equal_one_chunk():
    fix, m, env, algo, data = _fixture_setup('simplecar_n16')
    uv0 = _uv(algo)
    with gemm_impl(1):
        _, _, whole = algo.cbf_field(data, agents=list(range(16)), n_mesh=5, lims=fix['state_lim'], relink=True)
        _set_uv(algo, uv0)
        _, _, parts = algo.cbf_field(data, agents=list(range(16)), n_mesh=5, lims=fix['state_lim'], relink=True, max_edges=15)
        assert algo.last_field_chunks > 1
        assert torch.equal(whole, parts)


# ---- 6. a C3-sized graph on the tensor cores ---------------------------------------------------------------------------------------------
def test_c3_sized_all_agents_against_oracle():
    from gcbf_b200 import native, synth
    from gcbf_b200.synth import product_batch, seeded_algo
    c = synth.CONFIGS['C3']
    sb = synth.make_states(c['env'], c['num_agents'], c['num_obs'], 1, c['area_size'], c['seed'])
    env, algo = seeded_algo(sb.env, sb.num_agents, DEV, 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    data = product_batch(env, sb, DEV)
    E = int(data.edge_index.shape[1])
    n = sb.num_agents
    assert native.fn('gcbf_linear_h_supported')(E * 64, 2048, 2048) == 1      # phi's probe edges run on the wgmma kernel
    sd = sd_clone(algo.cbf)
    lims = (torch.zeros(4), torch.tensor([c['area_size'], c['area_size'], 10.0, 10.0]))
    xs, ys, h = algo.cbf_field(data, agents=list(range(n)), n_mesh=8, lims=lims)
    assert tuple(h.shape) == (1, n, 8, 8) and bool(torch.isfinite(h).all())
    ei = data.edge_index.cpu()
    indeg = torch.bincount(ei[1], minlength=n)[:n]
    sample = sorted({int(torch.argmax(indeg)), 0, 511, n - 1})
    want = FO.field(sd, sb.env, sb.states, data.x.cpu(), ei, n, sb.nodes_per_graph, 1, sample, 0, 1, xs, ys, relink=False)
    got = h[0, sample].reshape(-1).cpu()
    err = float((got - want).abs().max())
    assert err <= TOL, err


def test_cbf_contour_data_is_what_plot_cbf_contour_plots():
    from gcbf_b200.trainer.utils import cbf_contour_data
    fix, m, env, algo, data = _fixture_setup('drone_n8_o8')
    uv0 = _uv(algo)
    out = cbf_contour_data(algo, data, env, m['agent'], m['x_dim'], m['y_dim'])
    gx, gy = np.meshgrid(fix['xs'], fix['ys'])
    assert np.array_equal(out['x'], gx) and np.array_equal(out['y'], gy)     # drone: state_lim is [0, area]^3, no reset needed
    assert float((out['cbf'] - fix['field']).abs().max()) <= TOL
    _set_uv(algo, uv0)
    _, _, h = algo.cbf_field(data, agents=m['agent'], x_dim=m['x_dim'], y_dim=m['y_dim'])
    assert torch.equal(out['cbf'], h[0, 0].cpu())
    assert tuple(out['attention'].shape) == (data.edge_index.shape[1], 1)


@pytest.mark.parametrize('name', ['simplecar_n16', 'dubins_n16_o4_xy', 'drone_n8_o8'])
@pytest.mark.parametrize('relink', [False, True])
def test_probe_edge_lists_equal_radius_graph_of_moved_state(name, relink):
    """The device-built probe graphs (gcbf_cbf_field_probe_count / _fill: the ballot + popc ranks of the real kernels) against the
    reference's construction edge by edge: probe t's (source, edge_attr) list is bit-identical to the in-edges of the agent in copy t --
    ops.radius_graph on the moved state (relink) or the given edge_index (fixed) -- with the kernels' edge features."""
    fix, m, env, algo, data = _fixture_setup(name)
    a, N = m['agent'], data.states.shape[0]
    kw = dict(agents=a, x_dim=0, y_dim=1, n_mesh=10, lims=fix['state_lim'], relink=relink)
    uv0 = _uv(algo)
    ei, ea = algo.cbf_field_probe_graph(data, **kw)
    for k, v in _uv(algo).items():
        assert torch.equal(uv0[k], v), k                                      # no CBF pass
    xs, ys = algo.field_grid(fix['state_lim'], 0, 1, 10)
    batch, M = _copies(env, data, a, 0, 1, xs, ys, relink)
    sel = (batch.edge_index[1] % N) == a
    want_t = batch.edge_index[1][sel] // N
    want_src = batch.edge_index[0][sel] - want_t * N
    assert torch.equal(ei[1], want_t) and torch.equal(ei[0], want_src)
    assert torch.equal(ea, batch.edge_attr[sel])
    counts = torch.bincount(ei[1], minlength=M)
    if relink:
        assert int(counts.min()) != int(counts.max())                       # neighbours enter and leave as the agent moves
    algo.cbf_field(data, **kw)
    assert algo.last_field_edges == ei.shape[1]
