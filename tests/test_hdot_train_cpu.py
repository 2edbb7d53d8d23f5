"""CPU tests of the analytic-h_dot training loss (GCBF.params['h_dot'] = 'analytic'):
  1. the oracle (tests/hdot_train_oracle.py) against a float64 central finite difference of its own total loss along random parameter
     directions of both nets (three envs, the single-graph freeze, a batch without edges);
  2. the host build of the backward kernels' per-element functions (csrc/jvp_core.h via tests/host_driver/hdot_host.cpp) against
     torch autograd (double backward);
  3. the element-wise kernel bodies (csrc/jvp_kernels.cuh) on an emulated grid against the per-element driver, bit for bit;
  4. argument checks of the new entry points and of the mode switch.
"""
import copy
import ctypes
import os
import subprocess

import pytest
import torch

import gcbf_oracle as O
import hdot_train_oracle as HO
import jvp_oracle as JO
from conftest import ROOT
from helpers import oracle_batch, sd_clone, seeded_algo

ENV_ID = {'SimpleCar': 0, 'DubinsCar': 1, 'SimpleDrone': 2}


def _build(name):
    out = os.path.join(ROOT, 'tests', 'host_driver', '_build')
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, name + '.so')
    subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-I', os.path.join(ROOT, 'gcbf-pytorch_b200', 'csrc'),
                           '-I', os.path.join(ROOT, 'include'), '-I', os.path.join(ROOT, 'tests', 'host_driver'), '-o', so,
                           os.path.join(ROOT, 'tests', 'host_driver', name + '.cpp')])
    return ctypes.CDLL(so)


@pytest.fixture(scope='module')
def hhost():
    return _build('hdot_host')


@pytest.fixture(scope='module')
def hgrid():
    return _build('hdot_grid')


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def _case(env_name, n, obs, B, area, seed, on_goal=False):
    from gcbf_b200 import synth
    sb = synth.make_states(env_name, n, obs, B, area, seed)
    if on_goal:
        pd = O.ENV_PARAMS[env_name]['pos_dim']
        sb.states[1, :pd] = sb.goals[1, :pd]
    return sb


CASES = [('DubinsCar', 6, 2, 2, 1.0, 31, False), ('SimpleCar', 5, 0, 2, 0.8, 32, False), ('SimpleDrone', 4, 3, 2, 0.6, 33, False),
         ('DubinsCar', 6, 2, 1, 1.0, 34, True), ('SimpleCar', 4, 0, 2, 50.0, 36, False)]      # B = 1 freeze; a batch without edges


# ---- 1. the oracle against the finite difference ---------------------------------------------------------------------------------------
@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal', CASES)
def test_oracle_gradient_is_the_limit_of_the_finite_difference(env_name, n, obs, B, area, seed, on_goal, monkeypatch):
    """<grad L, d> of the oracle against (L(theta + tau d) - L(theta - tau d)) / 2 tau in float64 along three random directions per net.
    The spectral-norm vectors u, v of the one power iteration are held at their values for theta (as autograd does: they come from a
    no_grad iteration), so both sides differentiate the same function."""
    sb = _case(env_name, n, obs, B, area, seed, on_goal)
    _, algo = seeded_algo(env_name, n, torch.device('cpu'), 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    hp = dict(algo.params)
    hp['eps'] = 0.5                                                     # keep every loss term active
    ob = oracle_batch(sb)
    if area == 50.0:
        assert ob['edge_index'].shape[1] == 0
    d64 = lambda sd: {k: v.double() for k, v in sd.items()}
    cbf, act = d64(sd_clone(algo.cbf)), d64(sd_clone(algo.actor))
    # Move to a generic point.  The biases start at zero, and a row whose layer input is zero (an agent without in-edges: gamma's input is
    # [aggr = 0, x = 0]) then has every hidden pre-activation exactly at a ReLU kink, where autograd takes the slope 0 and a central
    # difference the mean of both one-sided slopes.  Noise of 1e-2 times the tensor's spread (absolute 1e-2 for the zero biases).
    gen = torch.Generator().manual_seed(seed + 1)
    for sd in (cbf, act):
        for k in O.trainable_keys(sd):
            spread = float(sd[k].std()) if sd[k].numel() > 1 else 0.0
            sd[k] = sd[k] + 1e-2 * (spread if spread > 0 else 1.0) * torch.randn(sd[k].shape, generator=gen, dtype=torch.float64)
    frozen = {}
    for k in list(cbf):
        if k.endswith('.weight_orig'):
            key = k[:-len('.weight_orig')]
            W, u = cbf[k], cbf[key + '.weight_u']
            v_new = torch.nn.functional.normalize(W.t() @ u, dim=0, eps=1e-12)
            frozen[key] = (torch.nn.functional.normalize(W @ v_new, dim=0, eps=1e-12), v_new)

    def sn_frozen(sd, key, update_uv=True):
        W = sd[key + '.weight_orig']
        u, v = frozen[key]
        return W / torch.dot(u, W @ v)
    monkeypatch.setattr(O, '_sn_weight', sn_frozen)
    prev = torch.get_default_dtype()
    torch.set_default_dtype(torch.float64)                              # the port's constant matrices (drone dynamics) follow it
    try:
        _fd_check(env_name, n, B, sb, ob, hp, cbf, act, seed)
    finally:
        torch.set_default_dtype(prev)


def _fd_check(env_name, n, B, sb, ob, hp, cbf, act, seed):
    states, goal, uref = sb.states.double(), sb.goals.double(), ob['u_ref'].double()
    K = ob['K'].double() if ob['K'] is not None else None

    def loss(c, a):
        return HO.analytic_losses(env_name, c, a, states, goal, ob['edge_index'], uref, B, n, sb.num_obs, hp, K)['loss']
    c0, a0 = copy.deepcopy(cbf), copy.deepcopy(act)
    ck, ak = O.trainable_keys(c0), O.trainable_keys(a0)
    for k in ck:
        c0[k].requires_grad_(True)
    for k in ak:
        a0[k].requires_grad_(True)
    L = loss(c0, a0)
    grads = torch.autograd.grad(L, [c0[k] for k in ck] + [a0[k] for k in ak], allow_unused=True)
    gc = {k: (g if g is not None else torch.zeros_like(c0[k])) for k, g in zip(ck, grads[:len(ck)])}
    ga = {k: (g if g is not None else torch.zeros_like(a0[k])) for k, g in zip(ak, grads[len(ck):])}
    gen = torch.Generator().manual_seed(seed)
    # two steps, 1e-6 and 1e-7: the difference must agree with <grad, d> at both (converged, and neither straddles a ReLU kink -- at 1e-5
    # the SimpleCar case already does).  float64 rounding of the difference at 1e-7 is ~1e-10 absolute, below 1e-5 of |<grad, d>| >= 1e-4
    steps = (1e-6, 1e-7)
    for which in ('cbf', 'actor'):
        for _ in range(3):
            base = cbf if which == 'cbf' else act
            keys, g = (ck, gc) if which == 'cbf' else (ak, ga)
            d = {k: torch.randn(base[k].shape, generator=gen, dtype=torch.float64) for k in keys}
            norm = torch.sqrt(sum((v ** 2).sum() for v in d.values()))
            gn = torch.sqrt(sum((g[k] ** 2).sum() for k in keys))
            # a random unit direction plus the gradient's: <grad, d> is then of the order of |grad|, well above the difference's rounding
            d = {k: v / norm + (g[k] / gn if gn > 0 else 0.0) for k, v in d.items()}
            an = float(sum((g[k] * d[k]).sum() for k in keys))
            assert abs(an) > 1e-4                                         # not vacuous
            for tau in steps:
                shifted = []
                for sgn in (1.0, -1.0):
                    sd = copy.deepcopy(base)
                    for k in keys:
                        sd[k] = sd[k] + sgn * tau * d[k]
                    shifted.append((loss(sd, act) if which == 'cbf' else loss(cbf, sd)).detach())   # (h_dot needs autograd)
                fd = float((shifted[0] - shifted[1]) / (2 * tau))
                assert abs(an - fd) <= 1e-5 * abs(an), (which, tau, an, fd)


# ---- 2. per-element functions against autograd -----------------------------------------------------------------------------------------
@pytest.mark.parametrize('C,deg_hi,pad', [(256, 9, 4), (7, 30, 3), (1, 3, 0)])
def test_attention_tangent_vjp_against_double_backward(hhost, C, deg_hi, pad):
    g = torch.Generator().manual_seed(C + 5)
    Nn = 23
    deg = torch.randint(0, deg_hi + 1, (Nn,), generator=g)
    deg[2], deg[5] = 0, 1                                        # an empty and a single-edge neighbourhood
    dst = torch.repeat_interleave(torch.arange(Nn), deg)
    rowptr = torch.zeros(Nn + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).int()
    E = int(deg.sum())
    r = lambda *s: torch.randn(*s, generator=g, dtype=torch.float64)
    msg, gate, t_msg, t_gate, tau = r(E, C), r(E, 1), r(E, C), r(E, 1), r(Nn, C)
    leaves = [t.clone().requires_grad_(True) for t in (msg, gate, t_msg, t_gate)]
    m, gt, tm, tg = leaves
    a = O.segment_softmax(gt, dst, Nn)
    (_, tang) = torch.autograd.functional.jvp(
        lambda mm, gg: torch.zeros(Nn, C, dtype=torch.float64).index_add(0, dst, O.segment_softmax(gg, dst, Nn) * mm), (m, gt), (tm, tg),
        create_graph=True)
    (tang * tau).sum().backward()
    want = [t.grad for t in leaves]
    f = lambda t: t.float()
    padc = lambda t: torch.cat([f(t), torch.full((t.shape[0], pad), 7.0)], 1).contiguous()
    ld = C + pad
    att = f(a.detach()).reshape(-1).contiguous()
    d_tmsg, d_msg = torch.full((E, ld), 7.0), torch.full((E, ld), 7.0)
    d_tgate, d_gate = torch.full((E,), 7.0), torch.full((E,), 7.0)
    keep = [padc(msg), padc(t_msg), f(t_gate).reshape(-1).contiguous(), padc(tau)]          # alive across the call
    hhost.host_attn_aggr_tangent_bwd(_p(keep[0]), ld, _p(keep[1]), ld, _p(att), _p(keep[2]), _p(rowptr), Nn, C, _p(keep[3]), ld, _p(d_tmsg), ld,
                                     _p(d_tgate), _p(d_msg), ld, _p(d_gate), 0)
    close = lambda got, w: float((got.double() - w).abs().max()) <= 1e-4 * (float(w.abs().max()) + 1.0)
    assert close(d_msg[:, :C], want[0]) and close(d_gate.reshape(-1, 1), want[1])
    assert close(d_tmsg[:, :C], want[2]) and close(d_tgate.reshape(-1, 1), want[3])
    if pad:
        assert float(d_tmsg[:, C:].min()) == 7.0 and float(d_msg[:, C:].min()) == 7.0


@pytest.mark.parametrize('act', [1, 2, 0])
def test_act_tangent_vjp_against_double_backward(hhost, act):
    g = torch.Generator().manual_seed(act)
    n = 501
    z, tz, dy, dty = [torch.randn(n, generator=g, dtype=torch.float64) for _ in range(4)]
    fn = {1: torch.relu, 2: torch.tanh, 0: lambda v: v * 1.0}[act]
    zz, tzz = z.clone().requires_grad_(True), tz.clone().requires_grad_(True)
    (ydot,) = torch.autograd.grad(fn(zz), zz, grad_outputs=tzz, create_graph=True)
    ((fn(zz) * dy).sum() + (ydot * dty).sum()).backward()
    dz, dtz = torch.empty(n), torch.empty(n)
    keep = [dy.float(), dty.float(), fn(z).float(), tz.float()]                                  # alive across the call
    hhost.host_act_tangent_bwd(*[_p(t) for t in keep], ctypes.c_int64(n), act, _p(dz), _p(dtz))
    assert torch.allclose(dz.double(), zz.grad, rtol=1e-5, atol=1e-5)
    assert torch.allclose(dtz.double(), tzz.grad, rtol=1e-5, atol=1e-5)


SD_CASES = [('DubinsCar', 12, 3, 2, 2.0, 31, False, 3.0), ('SimpleCar', 10, 0, 3, 1.5, 32, False, 8.0),
            ('SimpleDrone', 6, 6, 2, 0.9, 33, False, 8.0), ('DubinsCar', 12, 3, 1, 2.0, 34, True, 0.3),
            ('SimpleDrone', 6, 6, 1, 0.9, 35, True, 0.3)]


def _sd_inputs(env_name, n, obs, B, area, seed, on_goal, scale):
    sb = _case(env_name, n, obs, B, area, seed, on_goal)
    ob = oracle_batch(sb)
    p = O.ENV_PARAMS[env_name]
    g = torch.Generator().manual_seed(seed)
    action = (torch.randn(B * n, p['action_dim'], generator=g) * scale).contiguous()
    d_sdot = torch.randn(sb.states.shape[0], p['state_dim'], generator=g)
    return sb, ob, p, action, d_sdot


@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal,scale', SD_CASES)
def test_state_dot_vjp_against_autograd(hhost, env_name, n, obs, B, area, seed, on_goal, scale):
    """Clamp active (large actions) and inactive, the single-graph freeze, obstacle rows (which carry no action)."""
    sb, ob, p, action, d_sdot = _sd_inputs(env_name, n, obs, B, area, seed, on_goal, scale)
    a = action.clone().requires_grad_(True)
    sd = JO.closed_loop_state_dot(env_name, sb.states, sb.goals, a, B, n, sb.num_obs, K=ob['K'])
    (want,) = torch.autograd.grad((sd * d_sdot).sum(), a)
    got = torch.full_like(action, 7.0)
    f = ctypes.c_float
    st, goal = sb.states.contiguous(), sb.goals.contiguous()
    hhost.host_state_dot_bwd(ENV_ID[env_name], B, sb.nodes_per_graph, n, _p(st), st.shape[1], _p(action), _p(ob['u_ref'].contiguous()), _p(goal),
                             goal.shape[1], 0, f(p['action_lim']), f(p['dist2goal']), 1 if B == 1 else 0, _p(d_sdot.contiguous()), p['state_dim'],
                             _p(got), 0)
    assert torch.allclose(got, want, rtol=1e-6, atol=1e-6)
    if on_goal:
        assert float(got[1].abs().max()) == 0.0
    if scale > 1:
        assert float((want == 0).float().mean()) > 0.05


def test_state_dot_vjp_at_the_clamp_limits(hhost):
    """torch.clamp passes the gradient AT the limits (-lim <= x <= lim); so does the kernel."""
    sb, ob, p, action, d_sdot = _sd_inputs('SimpleCar', 10, 0, 2, 1.5, 38, False, 0.3)
    uref = ob['u_ref'].contiguous()
    action[0, 0] = p['action_lim'] - float(uref[0, 0])
    action[1, 1] = -p['action_lim'] - float(uref[1, 1])
    tot = action + uref
    assert float(tot[0, 0]) == p['action_lim'] and float(tot[1, 1]) == -p['action_lim']
    a = action.clone().requires_grad_(True)
    sd = JO.closed_loop_state_dot('SimpleCar', sb.states, sb.goals, a, 2, 10, 0, K=ob['K'])
    (want,) = torch.autograd.grad((sd * d_sdot).sum(), a)
    got = torch.empty_like(action)
    st, goal = sb.states.contiguous(), sb.goals.contiguous()
    hhost.host_state_dot_bwd(0, 2, 10, 10, _p(st), 4, _p(action), _p(uref), _p(goal), goal.shape[1], 0, ctypes.c_float(p['action_lim']),
                             ctypes.c_float(p['dist2goal']), 0, _p(d_sdot.contiguous()), 4, _p(got), 0)
    assert want[0, 0] != 0 and want[1, 1] != 0
    assert torch.allclose(got, want, rtol=1e-6, atol=1e-6)


# ---- 3. kernel bodies on the emulated grid ---------------------------------------------------------------------------------------------
GEOMETRIES = [(1, 1), (3, 7), (2, 256), (1056, 256)]


@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal,scale', SD_CASES)
def test_state_dot_bwd_kernel_on_an_emulated_grid(hhost, hgrid, env_name, n, obs, B, area, seed, on_goal, scale):
    sb, ob, p, action, d_sdot = _sd_inputs(env_name, n, obs, B, area, seed, on_goal, scale)
    sd, ad, f = p['state_dim'], p['action_dim'], ctypes.c_float
    st = torch.cat([sb.states, torch.full((sb.states.shape[0], 2), 9.0)], 1).contiguous()          # padded pitches
    ds = torch.cat([d_sdot, torch.full((d_sdot.shape[0], 3), 9.0)], 1).contiguous()
    goal, uref = sb.goals.contiguous(), ob['u_ref'].contiguous()
    args = lambda out, acc: (ENV_ID[env_name], B, sb.nodes_per_graph, n, _p(st), st.shape[1], _p(action), _p(uref), _p(goal), goal.shape[1], 0,
                             f(p['action_lim']), f(p['dist2goal']), 1 if B == 1 else 0, _p(ds), ds.shape[1], _p(out), acc)
    base = torch.randn(B * n, ad, generator=torch.Generator().manual_seed(seed))
    for acc in (0, 1):
        ref = base.clone()
        hhost.host_state_dot_bwd(*args(ref, acc))
        for grid, block in GEOMETRIES:
            got = base.clone()
            hgrid.grid_state_dot_bwd(grid, block, *args(got, acc))
            assert torch.equal(got, ref), (grid, block, acc)


@pytest.mark.parametrize('act', [0, 1, 2])
def test_act_tangent_bwd_kernel_on_an_emulated_grid(hhost, hgrid, act):
    g = torch.Generator().manual_seed(act + 3)
    n = 777
    dy, dty, y, tz = [torch.randn(n + 5, generator=g) for _ in range(4)]
    ref_z, ref_t = torch.full((n + 5,), 7.0), torch.full((n + 5,), 7.0)
    hhost.host_act_tangent_bwd(_p(dy), _p(dty), _p(y), _p(tz), ctypes.c_int64(n), act, _p(ref_z), _p(ref_t))
    for grid, block in GEOMETRIES:
        gz, gt = torch.full((n + 5,), 7.0), torch.full((n + 5,), 7.0)
        hgrid.grid_act_tangent_bwd(grid, block, _p(dy), _p(dty), _p(y), _p(tz), ctypes.c_int64(n), act, _p(gz), _p(gt))
        assert torch.equal(gz, ref_z) and torch.equal(gt, ref_t), (grid, block)
        assert float(gz[n:].min()) == 7.0 and float(gt[n:].min()) == 7.0                  # nothing past `count` is written


# ---- 4. argument checks ------------------------------------------------------------------------------------------------------------------
def test_new_entry_points_reject_bad_arguments_before_touching_the_gpu():
    from gcbf_b200 import _C
    lib = _C.lib()
    ok = 0x7f0000000000
    err = lambda: lib.gcbf_last_error().decode()
    assert lib.gcbf_attn_aggr_tangent_bwd(ok, 256, ok, 256, ok, ok, ok, 10, 256, ok, 255, ok, 256, ok, ok, 256, ok, 1, None) == -1
    assert 'gcbf_attn_aggr_tangent_bwd' in err()
    assert lib.gcbf_attn_aggr_tangent_bwd(ok, 256, ok, 256, ok, ok, None, 10, 256, ok, 256, ok, 256, ok, ok, 256, ok, 1, None) == -1
    assert lib.gcbf_act_tangent_bwd(ok, ok, ok, ok, 10, 3, ok, ok, None) == -1                          # unknown activation
    assert lib.gcbf_act_tangent_bwd(ok, ok, ok, None, 10, 2, ok, ok, None) == -1                        # tanh needs the tangent
    cfg = _C.EnvCfg(1, 2, 8, 6, 0.05, 0.8, 0.02, 0.03)
    assert lib.gcbf_state_dot_bwd(None, ok, 4, ok, ok, ok, 2, 0, 0, ok, 4, ok, 0, None) == -1
    assert lib.gcbf_state_dot_bwd(ctypes.byref(cfg), ok, 3, ok, ok, ok, 2, 0, 0, ok, 4, ok, 0, None) == -1     # ld < state_dim
    assert lib.gcbf_state_dot_bwd(ctypes.byref(cfg), ok, 4, ok, ok, None, 2, 0, 1, ok, 4, ok, 0, None) == -1   # freeze without goal
    assert lib.gcbf_edge_attr_bwd_ordered(5, ok, 4, ok, 10, 8, ok, ok, None) == -1
    assert lib.gcbf_edge_attr_bwd_ordered(1, ok, 4, None, 10, 8, ok, ok, None) == -1
    assert lib.gcbf_loss_partials_hdot(ok, None, ok, 2, ok, ok, 10, 1.0, 0.02, ok, None) == -1
    assert lib.gcbf_loss_grads_hdot(ok, ok, ok, 2, ok, ok, 10, 1.0, 0.02, 1.0, 1.0, 1.0, 1.0, ok, ok, None, ok, ok, None) == -1


def test_h_dot_mode_must_be_known():
    _, algo = seeded_algo('SimpleCar', 4, torch.device('cpu'), 0, {'num_obs': 0, 'area_size': 2.0})
    assert algo._h_dot_mode() == 'finite_difference'
    algo.params['h_dot'] = 'analytic'
    assert algo._h_dot_mode() == 'analytic'
    algo.params['h_dot'] = 'autodiff'
    with pytest.raises(ValueError):
        algo.train_step(None)
