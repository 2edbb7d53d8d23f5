"""CPU tests of the analytic h_dot (SURVEY 8f-3; gcbf_b200/jvp.py, csrc/jvp.cu):
  1. the oracle (oracle/jvp_oracle.py: autograd JVP through the GCBF port) against the defining limit -- a central finite difference
     of the same port in float64;
  2. the host build of the kernels' per-element functions (csrc/jvp_core.h via tests/host_driver/jvp_host.cpp) against autograd;
  3. the product's tangent pass (jvp.py over ops.net_forward) on the host emulation of the C ABI (tests/fake_device.py) against the
     oracle, three environments incl. the single-graph reach-freeze branch and a graph without edges.
"""
import copy
import ctypes
import os
import subprocess

import pytest
import torch

import gcbf_oracle as O
import jvp_oracle as JO
from conftest import ROOT
from helpers import oracle_batch, sd_clone, seeded_algo

ENV_ID = {'SimpleCar': 0, 'DubinsCar': 1, 'SimpleDrone': 2}


def _build(name):
    out = os.path.join(ROOT, 'tests', 'host_driver', '_build')
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, name + '.so')
    subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-I', os.path.join(ROOT, 'gcbf-pytorch_b200', 'csrc'), '-o', so,
                           os.path.join(ROOT, 'tests', 'host_driver', name + '.cpp')])
    return ctypes.CDLL(so)


@pytest.fixture(scope='module')
def jhost():
    return _build('jvp_host')


@pytest.fixture(scope='module')
def mhost():
    lib = _build('macbf_host')
    lib.host_radius_graph_topk.restype = ctypes.c_int64
    return lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def _case(env_name, n, obs, B, area, seed, on_goal=False):
    from gcbf_b200 import synth
    sb = synth.make_states(env_name, n, obs, B, area, seed)
    if on_goal:
        pd = O.ENV_PARAMS[env_name]['pos_dim']
        sb.states[1, :pd] = sb.goals[1, :pd]                    # agent 1 sits on its goal: frozen in a single graph
    return sb


CASES = [('DubinsCar', 12, 3, 2, 2.0, 31, False), ('SimpleCar', 10, 0, 3, 1.5, 32, False), ('SimpleDrone', 6, 6, 2, 0.9, 33, False),
         ('DubinsCar', 12, 3, 1, 2.0, 34, True), ('SimpleDrone', 6, 6, 1, 0.9, 35, True)]


@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal', CASES[:3])
def test_oracle_is_the_limit_of_the_finite_difference(env_name, n, obs, B, area, seed, on_goal):
    """h_dot of the oracle (fp32 autograd JVP) against (h(s + tau f) - h(s - tau f)) / 2 tau of the same port in float64."""
    sb = _case(env_name, n, obs, B, area, seed, on_goal)
    _, algo = seeded_algo(env_name, n, torch.device('cpu'), 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    cbf = sd_clone(algo.cbf)
    ob = oracle_batch(sb)
    g = torch.Generator().manual_seed(seed)
    action = torch.randn(B * n, O.ENV_PARAMS[env_name]['action_dim'], generator=g) * 0.3
    h, h_dot, sdot = JO.h_and_h_dot(env_name, copy.deepcopy(cbf), sb.states, sb.goals, ob['edge_index'], action, B, n, sb.num_obs, K=ob['K'])
    cbf64 = {k: v.double() for k, v in cbf.items()}
    s64, d64 = sb.states.double(), sdot.double()
    tau = 1e-6
    with torch.no_grad():
        hp = JO.cbf_of_states(env_name, cbf64, s64 + tau * d64, ob['edge_index'], B, n, sb.num_obs)
        hm = JO.cbf_of_states(env_name, cbf64, s64 - tau * d64, ob['edge_index'], B, n, sb.num_obs)
    fd = ((hp - hm) / (2 * tau)).float()
    scale = float(fd.abs().max()) + 1e-6
    assert float((h_dot - fd).abs().max()) <= 2e-3 * scale + 1e-6, (float((h_dot - fd).abs().max()), scale)
    assert scale > 1e-4                                   # the test is not vacuous


@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal', CASES)
def test_kernel_arithmetic_state_dot_and_edge_tangent(jhost, env_name, n, obs, B, area, seed, on_goal):
    sb = _case(env_name, n, obs, B, area, seed, on_goal)
    p = O.ENV_PARAMS[env_name]
    ob = oracle_batch(sb)
    N = sb.nodes_per_graph
    g = torch.Generator().manual_seed(seed)
    action = (torch.randn(B * n, p['action_dim'], generator=g) * 3.0).contiguous()        # large enough to hit the clamp sometimes
    want = JO.closed_loop_state_dot(env_name, sb.states, sb.goals, action, B, n, sb.num_obs, K=ob['K'])
    st = sb.states.contiguous()
    got = torch.full((B * N, p['state_dim']), 7.0)
    goal = sb.goals.contiguous()
    f = ctypes.c_float
    jhost.host_state_dot(ENV_ID[env_name], B, N, n, _p(st), st.shape[1], _p(action), _p(ob['u_ref'].contiguous()), _p(goal), goal.shape[1], 0,
                         f(p['action_lim']), f(p['speed_limit']), f(p['dist2goal']), 1 if B == 1 else 0, _p(got), p['state_dim'])
    assert torch.allclose(got, want, rtol=1e-6, atol=1e-6)
    if on_goal:
        assert float(got[1].abs().max()) == 0.0 and float(want[1].abs().max()) == 0.0      # the frozen agent
    # edge-feature tangent against autograd
    ei = ob['edge_index'].contiguous()
    E = ei.shape[1]
    _, t_want = torch.autograd.functional.jvp(lambda s: O.edge_attr(env_name, s, ei), sb.states, want)
    t_got = torch.full((E, p['edge_dim']), 7.0)
    jhost.host_edge_attr_tangent(ENV_ID[env_name], _p(st), st.shape[1], _p(got), got.shape[1], _p(ei), ctypes.c_int64(E), _p(t_got))
    assert torch.allclose(t_got, t_want, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize('C,deg_hi', [(256, 9), (7, 30)])
def test_kernel_arithmetic_attention_tangent(jhost, C, deg_hi):
    g = torch.Generator().manual_seed(C)
    Nn = 41
    deg = torch.randint(0, deg_hi + 1, (Nn,), generator=g)
    deg[2] = 0
    dst = torch.repeat_interleave(torch.arange(Nn), deg)
    E = int(deg.sum())
    rowptr = torch.zeros(Nn + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).int()
    msg, gate = torch.randn(E, C, generator=g), torch.randn(E, 1, generator=g)
    t_msg, t_gate = torch.randn(E, C, generator=g), torch.randn(E, 1, generator=g)

    def aggr(m, gt):
        a = O.segment_softmax(gt, dst, Nn)
        return torch.zeros(Nn, C).index_add(0, dst, a * m)
    _, want = torch.autograd.functional.jvp(aggr, (msg, gate), (t_msg, t_gate))
    att = O.segment_softmax(gate, dst, Nn).reshape(-1).contiguous()
    got = torch.full((Nn, C + 4), 7.0)
    jhost.host_attn_aggr_tangent(_p(msg), C, _p(t_msg), C, _p(att), _p(t_gate.reshape(-1).contiguous()), _p(rowptr), Nn, C, _p(got), C + 4)
    assert torch.allclose(got[:, :C], want, rtol=1e-4, atol=1e-5)
    assert float(got[2, :C].abs().max()) == 0.0 and float(got[:, C:].min()) == 7.0           # empty neighbourhood; padding untouched


def _product(env_name, sb, monkeypatch, mhost, jhost):
    import fake_device
    from gcbf_b200.data import Data
    fake_device.install(monkeypatch, mhost, jhost)
    env, algo = seeded_algo(env_name, sb.num_agents, torch.device('cpu'), 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    env.set_goal(sb.goals)
    ob = oracle_batch(sb)
    data = env.make_graph(sb.states.clone())
    data.update(Data(edge_index=ob['edge_index'], edge_attr=O.edge_attr(env_name, sb.states, ob['edge_index'])))
    return env, algo, data, ob


@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal', CASES)
def test_product_tangent_pass_on_the_fake_device(mhost, jhost, monkeypatch, env_name, n, obs, B, area, seed, on_goal):
    sb = _case(env_name, n, obs, B, area, seed, on_goal)
    env, algo, data, ob = _product(env_name, sb, monkeypatch, mhost, jhost)
    cbf = sd_clone(algo.cbf)
    g = torch.Generator().manual_seed(seed)
    action = torch.randn(B * n, O.ENV_PARAMS[env_name]['action_dim'], generator=g) * 0.3
    want_h, want_hd, _ = JO.h_and_h_dot(env_name, cbf, sb.states, sb.goals, ob['edge_index'], action, B, n, sb.num_obs, K=ob['K'])
    h, h_dot = algo.h_dot_analytic(data, action)
    assert h.shape == want_h.shape and h_dot.shape == want_hd.shape
    assert float((h - want_h).abs().max()) <= 1e-6
    scale = float(want_hd.abs().max())
    assert float((h_dot - want_hd).abs().max()) <= 1e-4 * scale + 1e-6, (float((h_dot - want_hd).abs().max()), scale)
    assert scale > 1e-4


def test_product_tangent_pass_on_a_graph_without_edges(mhost, jhost, monkeypatch):
    sb = _case('SimpleCar', 4, 0, 2, 50.0, 36)
    env, algo, data, ob = _product('SimpleCar', sb, monkeypatch, mhost, jhost)
    assert ob['edge_index'].shape[1] == 0
    h, h_dot = algo.h_dot_analytic(data, torch.zeros(8, 2))
    assert h.shape == (8, 1) and float(h_dot.abs().max()) == 0.0      # h depends on the states only through the edge features


# ---- the kernel bodies themselves on an emulated grid (tests/host_driver/cuda_emu.h) ---------------------------------------------
@pytest.fixture(scope='module')
def jgrid():
    out = os.path.join(ROOT, 'tests', 'host_driver', '_build')
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, 'jvp_grid.so')
    subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-I', os.path.join(ROOT, 'gcbf-pytorch_b200', 'csrc'),
                           '-I', os.path.join(ROOT, 'include'), '-I', os.path.join(ROOT, 'tests', 'host_driver'), '-o', so,
                           os.path.join(ROOT, 'tests', 'host_driver', 'jvp_grid.cpp')])
    return ctypes.CDLL(so)


GEOMETRIES = [(1, 1), (3, 7), (2, 256), (1056, 256)]       # one thread striding over everything ... more threads than work


@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal', CASES)
def test_kernel_bodies_on_an_emulated_grid(jhost, jgrid, env_name, n, obs, B, area, seed, on_goal):
    """csrc/jvp_kernels.cuh compiled as C++ and run thread by thread: every launch geometry must reproduce the serial per-element
    driver bit for bit (indexing, pitches, grid-stride loops, untouched padding)."""
    sb = _case(env_name, n, obs, B, area, seed, on_goal)
    p = O.ENV_PARAMS[env_name]
    ob = oracle_batch(sb)
    N, sd, ed = sb.nodes_per_graph, p['state_dim'], p['edge_dim']
    g = torch.Generator().manual_seed(seed)
    action = (torch.randn(B * n, p['action_dim'], generator=g) * 3.0).contiguous()
    st = torch.cat([sb.states, torch.full((B * N, 2), 9.0)], dim=1).contiguous()          # states with a pitch larger than state_dim
    goal, uref, f = sb.goals.contiguous(), ob['u_ref'].contiguous(), ctypes.c_float
    freeze = 1 if B == 1 else 0
    ref = torch.full((B * N, sd + 1), 7.0)
    jhost.host_state_dot(ENV_ID[env_name], B, N, n, _p(st), st.shape[1], _p(action), _p(uref), _p(goal), goal.shape[1], 0, f(p['action_lim']),
                         f(p['speed_limit']), f(p['dist2goal']), freeze, _p(ref), sd + 1)
    ei = ob['edge_index'].contiguous()
    E = ei.shape[1]
    t_ref = torch.full((E, ed), 7.0)
    jhost.host_edge_attr_tangent(ENV_ID[env_name], _p(st), st.shape[1], _p(ref), sd + 1, _p(ei), ctypes.c_int64(E), _p(t_ref))
    for grid, block in GEOMETRIES:
        got = torch.full((B * N, sd + 1), 7.0)
        jgrid.grid_state_dot(grid, block, ENV_ID[env_name], B, N, n, _p(st), st.shape[1], _p(action), _p(uref), _p(goal), goal.shape[1], 0,
                             f(p['action_lim']), f(p['speed_limit']), f(p['dist2goal']), freeze, _p(got), sd + 1)
        assert torch.equal(got, ref), (grid, block)
        assert float(got[:, sd].min()) == 7.0                                         # the pitch padding is never written
        if E:
            t_got = torch.full((E, ed), 7.0)
            jgrid.grid_edge_attr_tangent(grid, block, ENV_ID[env_name], _p(st), st.shape[1], _p(got), sd + 1, _p(ei), ctypes.c_int64(E), _p(t_got))
            assert torch.equal(t_got, t_ref), (grid, block)


@pytest.mark.parametrize('C,deg_hi', [(256, 9), (7, 30)])
def test_attention_tangent_kernel_on_an_emulated_grid(jhost, jgrid, C, deg_hi):
    g = torch.Generator().manual_seed(C + 1)
    Nn = 29
    deg = torch.randint(0, deg_hi + 1, (Nn,), generator=g)
    deg[0] = 0
    E = int(deg.sum())
    rowptr = torch.zeros(Nn + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).int()
    msg, t_msg = torch.randn(E, C + 4, generator=g), torch.randn(E, C, generator=g)        # msg with a padded pitch
    att, t_gate = torch.rand(E, generator=g), torch.randn(E, generator=g)
    ref = torch.full((Nn, C + 4), 7.0)
    jhost.host_attn_aggr_tangent(_p(msg), C + 4, _p(t_msg), C, _p(att), _p(t_gate), _p(rowptr), Nn, C, _p(ref), C + 4)
    for grid, block in GEOMETRIES:
        got = torch.full((Nn, C + 4), 7.0)
        jgrid.grid_attn_tangent(grid, block, _p(msg), C + 4, _p(t_msg), C, _p(att), _p(t_gate), _p(rowptr), Nn, C, _p(got), C + 4)
        assert torch.equal(got, ref), (grid, block)
