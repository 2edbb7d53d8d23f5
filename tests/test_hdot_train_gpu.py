"""GPU tests of the analytic-h_dot training loss (GCBF.params['h_dot'] = 'analytic'): the backward kernels of the tangent pass against
float64 autograd, and the analytic train step against the CPU oracle (tests/hdot_train_oracle.py, pinned by a float64 finite difference in
tests/test_hdot_train_cpu.py)."""
import pytest
import torch

import gcbf_oracle as O
import hdot_train_oracle as HO
from gcbf_b200 import _C, ops, synth
from helpers import oracle_batch, product_batch, sd_clone, seeded_algo

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _p(t):
    return t.data_ptr() if t is not None else None


def _csr(g, Nn, deg_hi, empty=(2,), single=(5,)):
    deg = torch.randint(0, deg_hi + 1, (Nn,), generator=g)
    for i in empty:
        deg[i] = 0
    for i in single:
        deg[i] = 1
    dst = torch.repeat_interleave(torch.arange(Nn), deg)
    rowptr = torch.zeros(Nn + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).int()
    return dst, rowptr, int(deg.sum())


# the last case has more targets (20,000) than the launch has warps (at most 16 * 132 blocks of 8): the grid-stride loop runs twice
@pytest.mark.parametrize('C,deg_hi,pad,Nn', [(256, 9, 4, 37), (7, 30, 3, 37), (7, 4, 1, 20000)])
def test_attn_tangent_bwd_against_double_backward(C, deg_hi, pad, Nn):
    g = torch.Generator().manual_seed(C)
    dst, rowptr, E = _csr(g, Nn, deg_hi)
    msg, gate = torch.randn(E, C, generator=g, dtype=torch.float64), torch.randn(E, 1, generator=g, dtype=torch.float64)
    t_msg, t_gate = torch.randn(E, C, generator=g, dtype=torch.float64), torch.randn(E, 1, generator=g, dtype=torch.float64)
    tau = torch.randn(Nn, C, generator=g, dtype=torch.float64)
    d_msg0, d_gate0 = torch.randn(E, C, generator=g, dtype=torch.float64), torch.randn(E, 1, generator=g, dtype=torch.float64)
    # autograd of L = <tau, tangent(msg, gate; t_msg, t_gate)> in float64
    leaves = [t.clone().requires_grad_(True) for t in (msg, gate, t_msg, t_gate)]
    m, gt, tm, tg = leaves
    a = O.segment_softmax(gt, dst, Nn)
    gbar = torch.zeros(Nn, 1, dtype=torch.float64).index_add(0, dst, a * tg)
    tang = torch.zeros(Nn, C, dtype=torch.float64).index_add(0, dst, a * (tm + m * (tg - gbar[dst])))
    (tang * tau).sum().backward()
    w_dm, w_dg, w_dtm, w_dtg = [t.grad for t in leaves]
    # the kernel, float32, padded pitches, accumulating onto given primal gradients
    f = lambda t: t.float()
    att = f(O.segment_softmax(gate, dst, Nn)).reshape(-1).contiguous().to(DEV)
    ld = C + pad
    pad_buf = lambda t: torch.cat([f(t), torch.full((t.shape[0], pad), 7.0)], 1).contiguous().to(DEV)
    msg_d, tmsg_d, tau_d = pad_buf(msg), pad_buf(t_msg), pad_buf(tau)
    d_msg, d_tmsg = pad_buf(d_msg0), torch.full((E, ld), 7.0, device=DEV)
    d_gate, d_tgate = f(d_gate0).reshape(-1).contiguous().to(DEV), torch.full((E,), 7.0, device=DEV)
    tg_d, rp_d = f(t_gate).reshape(-1).contiguous().to(DEV), rowptr.to(DEV)
    _C.call('gcbf_attn_aggr_tangent_bwd', _p(msg_d), ld, _p(tmsg_d), ld, _p(att), _p(tg_d), _p(rp_d), Nn, C, _p(tau_d), ld,
            _p(d_tmsg), ld, _p(d_tgate), _p(d_msg), ld, _p(d_gate), 1)
    torch.cuda.synchronize()
    # the second-order terms are d(tangent)/d(msg, gate); autograd's grads of msg / gate are exactly those
    close = lambda got, want: float((got.double() - want).abs().max()) <= 1e-4 * (float(want.abs().max()) + 1.0)
    assert close(d_tmsg[:, :C].cpu(), w_dtm)
    assert close(d_tgate.cpu().reshape(-1, 1), w_dtg)
    assert close(d_msg[:, :C].cpu() - f(d_msg0), w_dm)
    assert close(d_gate.cpu().reshape(-1, 1) - f(d_gate0), w_dg)
    assert float(d_tmsg[:, C:].min()) == 7.0 and float(d_msg[:, C:].min()) == 7.0                  # pitch padding untouched


@pytest.mark.parametrize('act', [ops.ACT_RELU, ops.ACT_TANH, ops.ACT_NONE])
def test_act_tangent_bwd_against_double_backward(act):
    g = torch.Generator().manual_seed(act + 11)
    n = 3001
    z, tz, dy, dty = [torch.randn(n, generator=g, dtype=torch.float64) for _ in range(4)]
    fn = {ops.ACT_RELU: torch.relu, ops.ACT_TANH: torch.tanh, ops.ACT_NONE: lambda v: v}[act]
    zz, tzz = z.clone().requires_grad_(True), tz.clone().requires_grad_(True)
    y = fn(zz)
    (ydot,) = torch.autograd.grad(y, zz, grad_outputs=tzz, create_graph=True)       # act'(z) z_dot
    ((y * dy).sum() + (ydot * dty).sum()).backward()
    yv = fn(z).float().to(DEV)
    dz, dtz = torch.empty(n, device=DEV), torch.empty(n, device=DEV)
    dy_d, dty_d, tz_d = [t.float().to(DEV) for t in (dy, dty, tz)]          # alive until the kernel has run
    _C.call('gcbf_act_tangent_bwd', _p(dy_d), _p(dty_d), _p(yv), _p(tz_d), n, act, _p(dz), _p(dtz))
    torch.cuda.synchronize()
    assert torch.allclose(dz.cpu().double(), zz.grad, rtol=1e-5, atol=1e-5)
    assert torch.allclose(dtz.cpu().double(), tzz.grad, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal,scale', [('DubinsCar', 12, 3, 2, 2.0, 31, False, 3.0),
                                                                      ('SimpleCar', 10, 0, 3, 1.5, 32, False, 8.0),
                                                                      ('SimpleDrone', 6, 6, 2, 0.9, 33, False, 8.0),
                                                                      ('DubinsCar', 12, 3, 1, 2.0, 34, True, 0.3),
                                                                      ('SimpleDrone', 6, 6, 1, 0.9, 35, True, 0.3)])
def test_state_dot_bwd_against_autograd(env_name, n, obs, B, area, seed, on_goal, scale):
    """Clamp active and inactive (large and small actions), the single-graph freeze, obstacle rows."""
    from gcbf_b200 import jvp
    import jvp_oracle as JO
    sb = synth.make_states(env_name, n, obs, B, area, seed)
    if on_goal:
        pd = O.ENV_PARAMS[env_name]['pos_dim']
        sb.states[1, :pd] = sb.goals[1, :pd]
    env, _ = seeded_algo(env_name, n, DEV, 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    data = product_batch(env, sb, DEV)
    ob = oracle_batch(sb)
    p = O.ENV_PARAMS[env_name]
    g = torch.Generator().manual_seed(seed)
    action = torch.randn(B * n, p['action_dim'], generator=g) * scale
    d_sdot = torch.randn(sb.states.shape[0], p['state_dim'], generator=g)
    a = action.clone().requires_grad_(True)
    sd = JO.closed_loop_state_dot(env_name, sb.states, sb.goals, a, B, n, sb.num_obs, K=ob['K'])
    (want,) = torch.autograd.grad((sd * d_sdot).sum(), a)
    base = torch.randn(B * n, p['action_dim'], generator=g)
    got = base.clone().to(DEV)
    jvp.state_dot_bwd(env, data, action.to(DEV), d_sdot.to(DEV), got)
    torch.cuda.synchronize()
    assert torch.allclose(got.cpu() - base, want, rtol=1e-5, atol=1e-5)
    if on_goal:
        assert float(want[1].abs().max()) == 0.0
    if scale > 1:
        assert float((want == 0).float().mean()) > 0.05                 # the clamp is active somewhere


@pytest.mark.parametrize('env_name,seed', [('DubinsCar', 41), ('SimpleDrone', 42), ('SimpleCar', 43)])
def test_edge_attr_bwd_ordered_matches_the_atomic_vjp(env_name, seed):
    from gcbf_b200 import jvp
    sb = synth.make_states(env_name, 24, 4 if env_name != 'SimpleCar' else 0, 3, 2.0, seed)
    env, _ = seeded_algo(env_name, 24, DEV, 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    data = product_batch(env, sb, DEV)
    E = data.edge_index.shape[1]
    assert E > 0
    d_ea = torch.randn(E, env.edge_dim, generator=torch.Generator().manual_seed(seed)).to(DEV)
    a = jvp.edge_attr_bwd_ordered(env, data.states, data.edge_index, d_ea).clone()
    b = jvp.edge_attr_bwd_ordered(env, data.states, data.edge_index, d_ea).clone()
    ref = ops.edge_attr_bwd(ops.ENV_IDS[env_name], data.states, data.edge_index, d_ea)
    torch.cuda.synchronize()
    assert torch.equal(a, b)
    assert torch.allclose(a, ref, rtol=1e-5, atol=1e-5)


# ---- the train step -------------------------------------------------------------------------------------------------------------------
CASES = [('DubinsCar', 12, 3, 2, 2.0, 31, False), ('SimpleCar', 10, 0, 3, 1.5, 32, False), ('SimpleDrone', 6, 6, 2, 0.9, 33, False),
         ('DubinsCar', 12, 3, 1, 2.0, 34, True), ('SimpleCar', 4, 0, 2, 50.0, 36, False),      # B = 1 freeze; a batch without edges
         ('DubinsCar', 64, 8, 4, 3.0, 7, False)]                                                # the 2048-wide layers on the tensor cores


def _setup(env_name, n, obs, B, area, seed, on_goal, init_seed=0):
    # init_seed 0: the weights of test_zz_jvp_gpu.py's cases.  h_dot jumps where a hidden ReLU's pre-activation is within rounding of 0
    # and the 3xfp16 product and the CPU oracle decide its mask differently (one agent of DubinsCar n = 64 / B = 4 at init_seed 1)
    sb = synth.make_states(env_name, n, obs, B, area, seed)
    if on_goal:
        pd = O.ENV_PARAMS[env_name]['pos_dim']
        sb.states[1, :pd] = sb.goals[1, :pd]
    env, algo = seeded_algo(env_name, n, DEV, init_seed, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    algo.params['h_dot'] = 'analytic'
    data = product_batch(env, sb, DEV)
    return sb, env, algo, data


@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal', CASES)
def test_analytic_train_step_against_the_oracle(env_name, n, obs, B, area, seed, on_goal):
    sb, env, algo, data = _setup(env_name, n, obs, B, area, seed, on_goal)
    cbf, act = sd_clone(algo.cbf), sd_clone(algo.actor)
    ob = oracle_batch(sb)
    assert torch.equal(data.edge_index.cpu(), ob['edge_index'])
    if env_name == 'SimpleCar' and area == 50.0:
        assert ob['edge_index'].shape[1] == 0
    want = HO.analytic_update_step(env_name, cbf, act, {}, {}, sb.states, sb.goals, ob['edge_index'], ob['u_ref'], B, n, sb.num_obs,
                                   hp=algo.params, K=ob['K'])
    # raw gradients: a second product step on fresh copies, without the optimizer
    _, _, algo2, data2 = _setup(env_name, n, obs, B, area, seed, on_goal)
    algo2.train_step(data2, apply_optim=False)
    res = algo.train_step(data)
    torch.cuda.synchronize()
    assert 'h_next' not in res and 'h_next_new' not in res and 'edge_index_new' not in res
    assert float((res['h'].cpu() - want['h']).abs().max()) <= 1e-5
    assert float((res['actions'].cpu() - want['actions']).abs().max()) <= 1e-5
    hd_want = want['h_dot'].reshape(-1)
    hd_tol = 1e-4 * float(hd_want.abs().max()) + 1e-6
    assert float((res['hdot'].cpu() - hd_want).abs().max()) <= hd_tol
    s = res['scalars'].tolist()
    for got, key, tol in zip(s[:4], ('loss_unsafe', 'loss_safe', 'loss_h_dot', 'loss_action'), (1e-5, 1e-5, hd_tol + 1e-6, 1e-5)):
        assert abs(got - float(want[key])) <= tol, (key, got, float(want[key]))
    assert torch.equal(res['unsafe_mask'].cpu(), want['unsafe_mask']) and torch.equal(res['safe_mask'].cpu(), want['safe_mask'])
    assert abs(float(res['acc_h_dot']) - float(want['acc_h_dot'])) <= 1.5 / n / B
    for mod, ref in ((algo2.cbf, want['raw_grads']['cbf']), (algo2.actor, want['raw_grads']['actor'])):
        total = torch.sqrt(sum((g.double() ** 2).sum() for g in ref.values()))
        err = torch.sqrt(sum(((p.grad.cpu().double() - ref[k].double()) ** 2).sum() for k, p in mod.named_parameters()))
        assert total > 0 and err / total < 2e-2, (err.item(), total.item())
    for mod, ref_sd, lr in ((algo.cbf, cbf, 3e-4), (algo.actor, act, 1e-3)):          # the tolerances of test_train_step_against_live_oracle
        for k, v in mod.state_dict().items():
            diff = (v.cpu() - ref_sd[k]).abs()
            tol = 2e-5 + 1e-4 * ref_sd[k].abs()
            assert (diff > tol).float().mean().item() <= 0.10, (k, (diff > tol).float().mean().item())
            if k.endswith(('weight', 'bias', 'weight_orig')):
                assert diff.max().item() <= 2 * lr + 1e-6, (k, diff.max().item())


def _uv(module):
    return {k: v.detach().clone() for k, v in module.state_dict().items() if k.endswith(('weight_u', 'weight_v'))}


def _restore_uv(module, uv):
    sd = module.state_dict()
    for k, v in uv.items():
        sd[k].copy_(v)


@pytest.mark.parametrize('case', [0, 5])
def test_step_h_dot_is_h_dot_analytic(case):
    sb, env, algo, data = _setup(*CASES[case])
    uv = _uv(algo.cbf)
    res = algo.train_step(data, apply_optim=False)
    hdot = res['hdot'].clone()
    _restore_uv(algo.cbf, uv)
    h, want = algo.h_dot_analytic(data, res['actions'])
    torch.cuda.synchronize()
    assert torch.equal(hdot, want.reshape(-1))
    assert torch.equal(res['h'], h)


def test_three_analytic_steps_are_bit_reproducible():
    outs = []
    for _ in range(2):
        sb, env, algo, data = _setup(*CASES[0])
        rs = [algo.train_step(data) for _ in range(3)]
        torch.cuda.synchronize()
        outs.append(([torch.cat([r['scalars'], r['h'].reshape(-1), r['hdot'], r['actions'].reshape(-1)]).cpu() for r in rs],
                     algo._bucket.flat.cpu().clone()))
    for a, b in zip(outs[0][0], outs[1][0]):
        assert torch.equal(a, b)
    assert torch.equal(outs[0][1], outs[1][1])


def test_update_with_the_device_replay_ring():
    import random
    import numpy as np
    n, obs, area = 10, 4, 2.0
    sb, env, algo, data = _setup('DubinsCar', n, obs, 1, area, 61, False)
    algo.use_device_replay(capacity=8)
    for k in range(14):
        sbk = synth.make_states('DubinsCar', n, obs, 1, area, 300 + k)
        algo.buffer.append(env.graph_from_states(sbk.states.to(DEV)), is_safe=(k % 3 != 0))
    algo.batch_size = 20
    algo.params['inner_iter'] = 2
    np.random.seed(3), random.seed(3)
    info = algo.update(1, None)
    assert set(info) == {'acc/safe', 'acc/unsafe', 'acc/derivative'}
    assert all(np.isfinite(v) for v in info.values())
    assert algo.buffer.size == 0
