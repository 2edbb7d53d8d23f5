"""GPU tests of the CBF-condition field (GCBF.cbf_condition_field: two-hop probe graphs of csrc/condition.cu, the per-row closed loop
on the env kernels, the actor and CBF passes and the tangent pass of jvp.py):
  1. on the fp32 paths (ops.GEMM_IMPL = 1) h and h_dot equal, bit for bit, the copies oracle -- a Batch of one copy of the graph per
     grid point, u = algo.actor(batch), algo.h_dot_analytic(batch, u, freeze=True), row of the agent -- on three envs, fixed and
     relink, including a neighbour frozen on its goal; u, v of both nets afterwards equal the oracle's;
  2. the device-built two-hop graphs (ballot ranks of the real kernels) equal the construction from explicit copies edge by edge;
  3. h equals cbf_field's h from the same u, v;
  4. batching, chunking and repeated calls change no bit;
  5. against the float64-checked CPU oracle (oracle/jvp_oracle.py on the copies), and a C3-sized graph on the default dispatch
     against the copies of single agents.
"""
import numpy as np
import pytest
import torch

import condition_oracle as CO
import gcbf_oracle as O
import jvp_oracle as JO
from helpers import sd_clone
from test_cbf_field_gpu import _copies, gemm_impl

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda')

CASES = {'SimpleCar': (8, 0, 1.2), 'DubinsCar': (6, 3, 1.2), 'SimpleDrone': (6, 3, 0.7)}


def _uv(algo):
    return {f'{m}.{k}': v.detach().clone() for m, net in (('cbf', algo.cbf), ('actor', algo.actor))
            for k, v in net.state_dict().items() if k.endswith(('weight_u', 'weight_v'))}


def _set_uv(algo, uv):
    with torch.no_grad():
        for m, net in (('cbf', algo.cbf), ('actor', algo.actor)):
            sd = net.state_dict()
            for k, v in uv.items():
                if k.startswith(m + '.'):
                    sd[k[len(m) + 1:]].copy_(v)


def _setup(env_name, B=1, seed=7, freeze_neighbour=False):
    from gcbf_b200 import synth
    from gcbf_b200.synth import product_batch, seeded_algo
    n, obs, area = CASES[env_name]
    sb = synth.make_states(env_name, n, obs, B, area, seed)
    if freeze_neighbour and env_name != 'SimpleCar':
        pd = O.ENV_PARAMS[env_name]['pos_dim']
        sb.states[1, :pd] = sb.goals[1, :pd]              # agent 1 sits on its goal: the reach-freeze stops it
    env, algo = seeded_algo(env_name, n, DEV, 0, {'num_obs': sb.num_obs, 'area_size': area})
    data = product_batch(env, sb, DEV)
    lims = (torch.zeros(env.state_dim), torch.full((env.state_dim,), area))
    return sb, env, algo, data, lims


def _agent_with_agent_neighbours(env, data):
    n = env.num_agents
    ei = data.edge_index.cpu()
    deg = torch.bincount(ei[1][ei[0] % env.nodes_per_graph < n], minlength=n)[:n]
    return int(torch.argmax(deg))


def _oracle(algo, env, data, agent, x_dim, y_dim, xs, ys, relink):
    """(h, h_dot) [ny, nx] of the copies oracle"""
    from gcbf_b200.data import Data
    batch, M = _copies(env, data, agent, x_dim, y_dim, xs, ys, relink)
    batch.update(Data(u_ref=env.u_ref(batch)))
    with torch.no_grad():
        u = algo.actor(batch)
        h, hd = algo.h_dot_analytic(batch, u, freeze=True)
    n = env.num_agents
    return h.view(M, n)[:, agent].reshape(len(ys), len(xs)), hd.view(M, n)[:, agent].reshape(len(ys), len(xs)), batch, u


# ---- 1. bit for bit against the copies oracle ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('env_name', ['SimpleCar', 'DubinsCar', 'SimpleDrone'])
@pytest.mark.parametrize('relink', [False, True])
def test_field_equals_copies_oracle_bit_for_bit(env_name, relink):
    sb, env, algo, data, lims = _setup(env_name, freeze_neighbour=True)
    a = _agent_with_agent_neighbours(env, data)
    uv0 = _uv(algo)
    with gemm_impl(1):
        xs, ys, h, hd = algo.cbf_condition_field(data, agents=a, n_mesh=7, lims=lims, relink=relink)
        uv_call = _uv(algo)
        _set_uv(algo, uv0)
        want_h, want_hd, _, _ = _oracle(algo, env, data, a, 0, 1, xs, ys, relink)
    assert tuple(h.shape) == (1, 1, 7, 7) and tuple(hd.shape) == (1, 1, 7, 7)
    assert torch.equal(h[0, 0], want_h), float((h[0, 0] - want_h).abs().max())
    assert torch.equal(hd[0, 0], want_hd), float((hd[0, 0] - want_hd).abs().max())
    assert float(hd.abs().max()) > 0
    for k, v in _uv(algo).items():
        assert torch.equal(uv_call[k], v), k                          # ONE power iteration per net, as the oracle sequence


# ---- 2. the device-built two-hop graphs ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('env_name', ['SimpleCar', 'DubinsCar', 'SimpleDrone'])
@pytest.mark.parametrize('relink', [False, True])
def test_probe_graphs_equal_explicit_copies(env_name, relink):
    sb, env, algo, data, lims = _setup(env_name, B=2)
    n, N = env.num_agents, env.nodes_per_graph
    agents = [0, _agent_with_agent_neighbours(env, data), n - 1]
    uv0 = _uv(algo)
    g = algo.cbf_condition_field_probe_graph(data, agents=agents, n_mesh=5, lims=lims, relink=relink)
    for k, v in _uv(algo).items():
        assert torch.equal(uv0[k], v), k                              # no net evaluated
    xs, ys = algo.field_grid(lims, 0, 1, 5)
    want = CO.two_hop_graph(env_name, sb.states, data.x.cpu(), data.edge_index.cpu(), n, N, 2, agents, 0, 1, xs, ys, relink)
    assert torch.equal(g['rows'].cpu(), want['rows'])
    assert torch.equal(g['edge_index'].cpu(), want['edge_index']) and g['num_moved_edges'] == want['num_moved_edges']
    ea, wea = g['edge_attr'].cpu(), want['edge_attr']
    if env_name == 'DubinsCar':                                       # cos / sin: device vs host libm
        assert torch.equal(ea[:, :3], wea[:, :3]) and torch.allclose(ea[:, 3:], wea[:, 3:], rtol=0, atol=1e-6)
    else:
        assert torch.equal(ea, wea)
    assert torch.equal(g['states'].cpu(), want['states'])


# ---- 3. h is cbf_field's h --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('relink', [False, True])
def test_h_equals_cbf_field(relink):
    sb, env, algo, data, lims = _setup('DubinsCar')
    uv0 = _uv(algo)
    with gemm_impl(1):
        _, _, h, _ = algo.cbf_condition_field(data, agents=[0, 2], n_mesh=6, lims=lims, relink=relink)
        _set_uv(algo, uv0)
        _, _, h_field = algo.cbf_field(data, agents=[0, 2], n_mesh=6, lims=lims, relink=relink)
    assert torch.equal(h, h_field)


# ---- 4. batching, chunking, repeated calls ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize('relink', [False, True])
def test_batching_chunking_and_repeat_calls_change_nothing(relink):
    sb, env, algo, data, lims = _setup('DubinsCar', B=2)
    n, N = env.num_agents, env.nodes_per_graph
    agents = [0, 2, n - 1]
    uv0 = _uv(algo)
    with gemm_impl(1):
        _, _, h, hd = algo.cbf_condition_field(data, agents=agents, n_mesh=5, lims=lims, relink=relink)
        assert algo.last_field_chunks == 1
        uv_one = _uv(algo)
        _set_uv(algo, uv0)
        _, _, h2, hd2 = algo.cbf_condition_field(data, agents=agents, n_mesh=5, lims=lims, relink=relink, max_probes=7)
        assert algo.last_field_chunks == -(-2 * 3 * 25 // 7)
        assert torch.equal(h, h2) and torch.equal(hd, hd2)
        for k, v in _uv(algo).items():
            assert torch.equal(uv_one[k], v), k                       # one power iteration for all the chunks
        _set_uv(algo, uv0)
        _, _, h3, hd3 = algo.cbf_condition_field(data, agents=agents, n_mesh=5, lims=lims, relink=relink, max_edges=60)
        assert algo.last_field_chunks > 1
        assert torch.equal(h, h3) and torch.equal(hd, hd3)
        _set_uv(algo, uv0)
        _, _, h4, hd4 = algo.cbf_condition_field(data, agents=agents, n_mesh=5, lims=lims, relink=relink)
        assert torch.equal(h, h4) and torch.equal(hd, hd4)           # no float atomics: same bits
        for b in range(2):
            one = env.graph_from_states(sb.states[b * N:(b + 1) * N].to(DEV), with_u_ref=False)
            for k, a in enumerate(agents):
                _set_uv(algo, uv0)
                _, _, h1, hd1 = algo.cbf_condition_field(one, agents=a, n_mesh=5, lims=lims, relink=relink)
                assert torch.equal(h[b, k], h1[0, 0]) and torch.equal(hd[b, k], hd1[0, 0]), (b, a)


# ---- 5. tolerances: the float64-checked oracle, an isolated probe, a C3-sized graph ---------------------------------------------------
@pytest.mark.parametrize('env_name', ['DubinsCar', 'SimpleDrone'])
def test_against_cpu_jvp_oracle(env_name):
    sb, env, algo, data, lims = _setup(env_name, freeze_neighbour=True)
    a = _agent_with_agent_neighbours(env, data)
    sd = sd_clone(algo.cbf)
    uv0 = _uv(algo)
    xs, ys, h, hd = algo.cbf_condition_field(data, agents=a, n_mesh=5, lims=lims)
    _set_uv(algo, uv0)
    _, _, batch, u = _oracle(algo, env, data, a, 0, 1, xs, ys, False)
    M, n = 25, env.num_agents
    K = env._gain()
    want_h, want_hd, _ = JO.h_and_h_dot(env_name, sd, batch.states.cpu(), sb.goals.repeat(M, 1), batch.edge_index.cpu(), u.cpu(), M, n, sb.num_obs,
                                        K=K.cpu() if K is not None else None, freeze=True)
    want_h, want_hd = want_h.view(M, n)[:, a], want_hd.view(M, n)[:, a]
    assert float((h.reshape(-1).cpu() - want_h).abs().max()) <= 1e-5
    assert float((hd.reshape(-1).cpu() - want_hd).abs().max()) <= 1e-4 * float(want_hd.abs().max()) + 1e-6


def test_isolated_probe_in_relink_mode_has_zero_h_dot():
    sb, env, algo, data, lims = _setup('SimpleCar')
    far = (torch.full((4,), 40.0), torch.full((4,), 41.0))            # every grid point is out of everyone's radius
    _, _, h, hd = algo.cbf_condition_field(data, agents=0, n_mesh=3, lims=far, relink=True)
    assert algo.last_field_edges == 0 and bool((hd == 0).all()) and bool(torch.isfinite(h).all())


def test_c3_sized_graph_against_copies_of_single_agents():
    from gcbf_b200 import synth
    from gcbf_b200.synth import product_batch, seeded_algo
    c = synth.CONFIGS['C3']
    sb = synth.make_states(c['env'], c['num_agents'], c['num_obs'], 1, c['area_size'], c['seed'])
    env, algo = seeded_algo(sb.env, sb.num_agents, DEV, 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    data = product_batch(env, sb, DEV)
    n = sb.num_agents
    lims = (torch.zeros(4), torch.tensor([c['area_size'], c['area_size'], 10.0, 10.0]))
    sample = [0, _agent_with_agent_neighbours(env, data), n - 1]
    uv0 = _uv(algo)
    xs, ys, h, hd = algo.cbf_condition_field(data, agents=sample, n_mesh=4, lims=lims)
    assert bool(torch.isfinite(h).all()) and bool(torch.isfinite(hd).all())
    for k, a in enumerate(sample):
        _set_uv(algo, uv0)
        want_h, want_hd, _, _ = _oracle(algo, env, data, a, 0, 1, xs, ys, False)
        assert float((h[0, k] - want_h).abs().max()) <= 1e-5
        assert float((hd[0, k] - want_hd).abs().max()) <= 1e-4 * float(want_hd.abs().max()) + 1e-6


def test_cbf_contour_data_condition():
    from gcbf_b200.trainer.utils import cbf_contour_data
    sb, env, algo, data, lims = _setup('SimpleDrone')
    env.state_lim                                                       # drone: [0, area]^3 box without reset
    uv0 = _uv(algo)
    out = cbf_contour_data(algo, data, env, 0, 0, 1, attention=False, condition=True)
    _set_uv(algo, uv0)
    _, _, h, hd = algo.cbf_condition_field(data, agents=0, lims=env.state_lim)
    assert torch.equal(out['cbf'], h[0, 0].cpu()) and torch.equal(out['h_dot'], hd[0, 0].cpu())
    assert torch.equal(out['condition'], out['h_dot'] + float(algo.params['alpha']) * out['cbf'])
    plain = cbf_contour_data(algo, data, env, 0, 0, 1, attention=False)
    assert set(plain) == {'x', 'y', 'cbf'}
