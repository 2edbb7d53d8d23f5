"""CPU tests of the MACBF path (SURVEY 8f-4):
  1. the port (oracle/macbf_oracle.py) against the golden fixtures generated from the reference-on-shim (oracle/make_golden.py macbf);
  2. the host build of the per-element functions the CUDA kernels are made of (csrc/macbf_core.h via tests/host_driver/macbf_host.cpp,
     compiled here with g++ -ffp-contract=off) against the fixtures / the port: top-k radius graph bit-exact, per-edge masks equal,
     max aggregation forward + backward against torch, losses and their gradients against autograd;
  3. the product-side host logic that needs no GPU (factories, state-dict keys, seeded initialisation, the reference's no-op apply).
"""
import copy
import ctypes
import os
import subprocess

import pytest
import torch

import gcbf_oracle as O
import macbf_oracle as MO
from conftest import ROOT, digest_close, load_golden, macbf_golden_cases
from helpers import case_inputs

CASES = macbf_golden_cases()


def _inputs(fix):
    meta = fix['meta']
    sb = case_inputs(meta)
    if meta['case'].endswith('single'):
        sb.states[0, :2] = sb.goals[0, :2]
    assert torch.equal(sb.states, fix['states']) and torch.equal(sb.goals, fix['goals'])
    return meta, sb


@pytest.fixture(scope='module')
def host():
    """tests/host_driver/macbf_host.cpp -> shared object (the kernels' arithmetic, serial)."""
    out = os.path.join(ROOT, 'tests', 'host_driver', '_build')
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, 'macbf_host.so')
    src = os.path.join(ROOT, 'tests', 'host_driver', 'macbf_host.cpp')
    subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-I', os.path.join(ROOT, 'gcbf-pytorch_b200', 'csrc'),
                           '-o', so, src])
    lib = ctypes.CDLL(so)
    lib.host_radius_graph_topk.restype = ctypes.c_int64
    return lib


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def host_topk(lib, env, states, B, N, n, k):
    p = O.ENV_PARAMS[env]
    st = states.contiguous()
    rowptr = torch.zeros(B * n + 1, dtype=torch.int32)
    args = (_p(st), ctypes.c_int(st.shape[1]), ctypes.c_int(p['pos_dim']), ctypes.c_int(B), ctypes.c_int(N), ctypes.c_int(n),
            ctypes.c_float(p['comm_radius']), ctypes.c_int(0 if env == 'SimpleCar' else 1), ctypes.c_int(k), _p(rowptr))
    E = lib.host_radius_graph_topk(*args, None, ctypes.c_int64(0))
    ei = torch.zeros(2, E, dtype=torch.int64)
    lib.host_radius_graph_topk(*args, _p(ei), ctypes.c_int64(E))
    return ei, rowptr


@pytest.mark.parametrize('case', CASES)
def test_port_matches_golden(case):
    fix = load_golden(case)
    meta, sb = _inputs(fix)
    env, n, o, B = sb.env, sb.num_agents, sb.num_obs, sb.num_graphs
    N = n + o
    ei = MO.batch_radius_graph_topk(env, sb.states, B, N, n)
    assert torch.equal(ei, fix['edge_index'])
    K = O.lqr_gain(env) if env != 'DubinsCar' else None
    x, am = O.make_graph_inputs(env, sb.states, B, n, o)
    ur = O.u_ref(env, sb.states if am is None else sb.states[am], sb.goals, K)
    assert torch.allclose(ur, fix['u_ref'], rtol=0, atol=1e-6)      # (the LQR matmul rounds differently per batch shape)
    ur = fix['u_ref']
    e_attr = O.edge_attr(env, sb.states, ei)
    assert torch.equal(e_attr, fix['edge_attr'])
    cbf, act = copy.deepcopy(fix['cbf_init']), copy.deepcopy(fix['actor_init'])
    with torch.no_grad():
        h = MO.cbf_net_forward(cbf, x, e_attr, ei)
        u = MO.controller_forward(act, x, e_attr, ei, am, ur)
    assert torch.allclose(h, fix['h_probe'], rtol=0, atol=1e-7) and torch.allclose(u, fix['u_probe'], rtol=0, atol=1e-7)
    sm, um = MO.edge_masks(env, e_attr)
    assert torch.equal(sm, fix['safe_mask']) and torch.equal(um, fix['unsafe_mask'])
    # MACBF.apply of the reference never moves the action (its leaf does not require grad): it returns the actor's output
    ei0 = ei[:, ei[1] < N]
    a0 = MO.apply_controller(env, cbf, act, sb.states[:N], sb.goals, ei0, ur[:n], n, o)
    assert torch.allclose(a0, fix['apply_action'], rtol=0, atol=1e-7)
    assert torch.equal(fix['apply_action'], fix['u_probe'][:n]) or torch.allclose(fix['apply_action'], fix['u_probe'][:n], atol=1e-6)
    oc, oa = {}, {}
    for gold in fix['steps']:
        st = MO.update_step(env, cbf, act, oc, oa, sb.states, sb.goals, ei, ur, B, n, o, K=K)
        for tag, key in (('loss/unsafe', 'loss_unsafe'), ('loss/safe', 'loss_safe'), ('loss/derivative', 'loss_h_dot'),
                         ('loss/action', 'loss_action'), ('acc/unsafe', 'acc_unsafe'), ('acc/safe', 'acc_safe'),
                         ('acc/derivative', 'acc_h_dot')):
            assert abs(float(st[key]) - gold['scalars'][tag]) <= 1e-6, (tag, float(st[key]), gold['scalars'][tag])
    assert not digest_close(cbf, fix['cbf_final'], 1e-6, 1e-6)
    assert not digest_close(act, fix['actor_final'], 1e-6, 1e-6)


@pytest.mark.parametrize('case', CASES)
def test_kernel_arithmetic_topk_and_edge_masks_bit_exact(host, case):
    fix = load_golden(case)
    meta, sb = _inputs(fix)
    env, n, o, B = sb.env, sb.num_agents, sb.num_obs, sb.num_graphs
    ei, rowptr = host_topk(host, env, sb.states, B, n + o, n, 12)
    assert torch.equal(ei, fix['edge_index'])
    assert int(rowptr[-1]) == ei.shape[1]
    ea = fix['edge_attr'].contiguous()
    E = ea.shape[0]
    safe, unsafe = torch.zeros(E, dtype=torch.uint8), torch.zeros(E, dtype=torch.uint8)
    host.host_edge_masks(_p(ea), ctypes.c_int(ea.shape[1]), ctypes.c_int(O.ENV_PARAMS[env]['pos_dim']), ctypes.c_int64(E),
                         ctypes.c_double(O.ENV_PARAMS[env]['radius']), _p(safe), _p(unsafe))
    assert torch.equal(safe.bool(), fix['safe_mask']) and torch.equal(unsafe.bool(), fix['unsafe_mask'])


@pytest.mark.parametrize('env,n,o,B,area,k', [('DubinsCar', 40, 10, 4, 1.2, 12), ('SimpleDrone', 30, 30, 3, 0.7, 12), ('SimpleCar', 50, 0, 3, 1.0, 12),
                                               ('DubinsCar', 16, 0, 2, 1.0, 3), ('SimpleCar', 9, 0, 2, 0.5, 2), ('SimpleDrone', 14, 14, 1, 5.0, 12)])
def test_kernel_arithmetic_topk_dense_random(host, env, n, o, B, area, k):
    """Very dense graphs (every agent has far more than k nodes in range) and tiny k against the port's torch.topk / cumsum."""
    from gcbf_b200 import synth
    sb = synth.make_states(env, n, o, B, area, 77)
    N = sb.nodes_per_graph
    want = MO.batch_radius_graph_topk(env, sb.states, B, N, n, k)
    got, _ = host_topk(host, env, sb.states, B, N, n, k)
    assert torch.equal(got, want)
    if k < N - 1 and area < 2:
        assert int(torch.bincount(want[1]).max()) >= k      # the filter is active in the dense cases


def test_kernel_arithmetic_edge_norm_matches_torch_on_strided_rows(host):
    """||edge_attr[:, :pos_dim]|| feeds two threshold tests: the fma-chain formula of macbf_core.h against torch.norm on the strided
    slice the reference takes, on 2e5 random rows and on rows placed within a few ulps of both thresholds."""
    g = torch.Generator().manual_seed(3)
    for env in ('SimpleCar', 'DubinsCar', 'SimpleDrone'):
        p = O.ENV_PARAMS[env]
        pd, R = p['pos_dim'], p['radius']
        ea = (torch.rand(200_000, p['edge_dim'], generator=g) - 0.5) * 0.6
        # rows scaled onto the thresholds, then nudged by a few ulps
        for thr in (4 * R, 2 * R):
            blk = ea[:20_000, :pd]
            blk *= (thr / blk.norm(dim=-1, keepdim=True))
            blk *= 1 + (torch.randint(-3, 4, (20_000, 1), generator=g).float() * 6e-8)
            ea = torch.cat([ea, torch.cat([blk, torch.zeros(20_000, p['edge_dim'] - pd)], dim=1)], dim=0)
        ea = ea.contiguous()
        E = ea.shape[0]
        safe, unsafe = torch.zeros(E, dtype=torch.uint8), torch.zeros(E, dtype=torch.uint8)
        host.host_edge_masks(_p(ea), ctypes.c_int(ea.shape[1]), ctypes.c_int(pd), ctypes.c_int64(E), ctypes.c_double(R), _p(safe), _p(unsafe))
        sm, um = MO.edge_masks(env, ea)
        assert int((safe.bool() != sm).sum()) == 0 and int((unsafe.bool() != um).sum()) == 0, env


@pytest.mark.parametrize('C,deg_hi', [(128, 13), (5, 40), (1, 3)])
def test_kernel_arithmetic_seg_max(host, C, deg_hi):
    g = torch.Generator().manual_seed(C)
    Nn = 57
    deg = torch.randint(0, deg_hi + 1, (Nn,), generator=g)
    deg[3] = 0
    deg[Nn - 1] = 0
    dst = torch.repeat_interleave(torch.arange(Nn), deg)
    E = int(deg.sum())
    rowptr = torch.zeros(Nn + 1, dtype=torch.int32)
    rowptr[1:] = torch.cumsum(deg, 0).int()
    ld = C + 3
    buf = torch.randn(E, ld, generator=g)
    msg = buf[:, :C]
    out, arg = torch.full((Nn, C), 7.0), torch.zeros(Nn, C, dtype=torch.int32)
    host.host_seg_max_fwd(_p(buf), ctypes.c_int(ld), _p(rowptr), ctypes.c_int(Nn), ctypes.c_int(C), _p(out), ctypes.c_int(C), _p(arg))
    m = msg.clone().requires_grad_(True)
    want = torch.zeros(Nn, C).scatter_reduce(0, dst.view(-1, 1).expand(E, C), m, reduce='amax', include_self=False)
    assert torch.equal(out, want.detach())
    assert bool((arg[deg == 0] == -1).all()) and bool((out[deg == 0] == 0).all())
    d_out = torch.randn(Nn, C, generator=g)
    want.backward(d_out)
    d_msg = torch.full((E, C), 3.0)
    host.host_seg_max_bwd(_p(d_out), ctypes.c_int(C), _p(arg), ctypes.c_int(Nn), ctypes.c_int(C), _p(d_msg), ctypes.c_int(C), ctypes.c_int64(E))
    assert torch.equal(d_msg, m.grad)          # no ties in random floats: one winner per cell


@pytest.mark.parametrize('E,M,ad,empty', [(500, 60, 2, None), (64, 10, 3, 'unsafe'), (33, 7, 2, 'safe'), (1, 1, 2, None)])
def test_kernel_arithmetic_losses_match_autograd(host, E, M, ad, empty):
    g = torch.Generator().manual_seed(E)
    h = (torch.randn(E, generator=g) * 0.05).requires_grad_(True)
    hn = (h.detach() + torch.randn(E, generator=g) * 0.002).requires_grad_(True)
    act = torch.randn(M, ad, generator=g).requires_grad_(True)
    safe = torch.rand(E, generator=g) < 0.6
    unsafe = (torch.rand(E, generator=g) < 0.2) & ~safe
    if empty == 'unsafe':
        unsafe[:] = False
    if empty == 'safe':
        safe[:] = False
    alpha, eps, dt, cu, cs, ch, ca = 1.0, 0.02, 0.03, 1.0, 0.7, 0.4, 0.05
    # macbf.py:140-177
    hu, hs = h[unsafe], h[safe]
    lu = torch.relu(hu + eps).mean() if hu.numel() else torch.tensor(0.0)
    ls = torch.relu(-hs + eps).mean() if hs.numel() else torch.tensor(0.0)
    h_dot = (hn - h) / dt
    lh = torch.relu(-h_dot - alpha * h + eps).mean()
    la = torch.square(act).sum(dim=1).mean()
    loss = cu * lu + cs * ls + ch * lh + ca * la
    loss.backward()
    acc = [(hu < 0).float().mean() if hu.numel() else 1.0, (hs >= 0).float().mean() if hs.numel() else 1.0, ((h_dot + alpha * h) >= 0).float().mean()]
    partial = torch.zeros(16, dtype=torch.float64)
    d_h, d_hn, d_act, sc = torch.zeros(E), torch.zeros(E), torch.zeros(M, ad), torch.zeros(8)
    hd, hnd, ad_ = h.detach().contiguous(), hn.detach().contiguous(), act.detach().contiguous()
    s8, u8 = safe.to(torch.uint8), unsafe.to(torch.uint8)
    f = ctypes.c_float
    host.host_macbf_loss_partials(_p(hd), _p(hnd), _p(s8), _p(u8), ctypes.c_int64(E), _p(ad_), ctypes.c_int(ad), ctypes.c_int64(M), f(alpha), f(eps),
                                  f(dt), _p(partial))
    host.host_macbf_loss_grads(_p(hd), _p(hnd), _p(s8), _p(u8), ctypes.c_int64(E), _p(ad_), ctypes.c_int(ad), ctypes.c_int64(M), f(alpha), f(eps), f(dt),
                               f(cu), f(cs), f(ch), f(ca), _p(partial), _p(d_h), _p(d_hn), _p(d_act), _p(sc))
    for got, want in zip(sc.tolist(), [lu, ls, lh, la, acc[0], acc[1], loss, acc[2]]):
        assert abs(got - float(torch.as_tensor(want).detach())) <= 1e-6
    assert torch.allclose(d_h, h.grad, rtol=1e-5, atol=1e-9)
    assert torch.allclose(d_hn, hn.grad, rtol=1e-5, atol=1e-9)
    assert torch.allclose(d_act, act.grad, rtol=1e-6, atol=1e-9)
    assert partial[7] == E and partial[10] == M


# ---- the product's Python on a host emulation of the C ABI (tests/fake_device.py) ------------------------------------------------
def _product_algo(fix, sb, monkeypatch, host):
    import fake_device
    from gcbf_b200.algo import make_algo
    from gcbf_b200.env import make_env
    fd = fake_device.install(monkeypatch, host)
    dev = torch.device('cpu')
    env = make_env(sb.env, sb.num_agents, dev)
    params = env.default_params
    params.update({'num_obs': sb.num_obs, 'area_size': sb.area_size})
    env = make_env(sb.env, sb.num_agents, dev, params=params, max_neighbors=12)       # train.py:30
    algo = make_algo('macbf', env, sb.num_agents, env.node_dim, env.edge_dim, env.action_dim, dev, 512, MO.HYPERPARAMS[sb.env])
    algo.cbf.load_state_dict(fix['cbf_init'])
    algo.actor.load_state_dict(fix['actor_init'])
    return fd, env, algo


@pytest.mark.parametrize('into_param', [True, False])
@pytest.mark.parametrize('case', CASES)
def test_product_python_wiring_on_the_fake_device(host, monkeypatch, case, into_param):
    """algo/macbf.py + the autograd Functions + env glue + flat bucket / optimiser glue, executed on the host emulation of the C ABI,
    against the reference-on-shim fixture: top-k edges, per-edge h, actions, masks, two train steps (losses, accuracies) and the
    post-step weights."""
    from gcbf_b200 import synth
    fix = load_golden(case)
    meta, sb = _inputs(fix)
    fd, env, algo = _product_algo(fix, sb, monkeypatch, host)
    algo.GRAD_INTO_PARAM = into_param
    data = synth.product_batch(env, sb, torch.device('cpu'))
    assert torch.equal(data.edge_index, fix['edge_index'])
    assert torch.allclose(data.u_ref, fix['u_ref'], rtol=0, atol=1e-6)
    assert torch.allclose(data.edge_attr, fix['edge_attr'], rtol=0, atol=0)
    with torch.no_grad():
        h, u = algo.cbf(data), algo.act(data)
    assert torch.allclose(h, fix['h_probe'], rtol=0, atol=1e-6) and torch.allclose(u, fix['u_probe'], rtol=0, atol=1e-6)
    assert torch.equal(env.safe_mask(data, return_edge=True), fix['safe_mask'])
    assert torch.equal(env.unsafe_mask(data, return_edge=True), fix['unsafe_mask'])
    n = sb.num_agents
    one = synth.product_batch(env, synth.SynthBatch(sb.env, n, sb.num_obs, 1, sb.area_size, sb.states[:sb.nodes_per_graph], sb.goals, sb.obs),
                              torch.device('cpu'))
    assert torch.allclose(algo.apply(one), fix['apply_action'], rtol=0, atol=1e-6)
    for gold in fix['steps']:
        res = algo.train_step(data)
        s = res['scalars'].tolist()
        for i, tag in enumerate(('loss/unsafe', 'loss/safe', 'loss/derivative', 'loss/action', 'acc/unsafe', 'acc/safe')):
            assert abs(s[i] - gold['scalars'][tag]) <= 2e-6, (tag, s[i], gold['scalars'][tag])
        assert abs(s[7] - gold['scalars']['acc/derivative']) <= 1e-6
    assert not digest_close({k: v for k, v in algo.cbf.state_dict().items()}, fix['cbf_final'], 1e-5, 1e-5, flip=3e-6)
    assert not digest_close({k: v for k, v in algo.actor.state_dict().items()}, fix['actor_final'], 1e-5, 1e-5, flip=3e-6)
    for name in ('gcbf_radius_graph_topk_count', 'gcbf_radius_graph_topk_fill', 'gcbf_edge_masks', 'gcbf_seg_max_fwd', 'gcbf_seg_max_bwd',
                 'gcbf_macbf_loss_partials', 'gcbf_macbf_loss_grads', 'gcbf_mlp_forward', 'gcbf_mlp_backward', 'gcbf_clip_adam', 'gcbf_step_bwd',
                 'gcbf_edge_attr_bwd'):
        assert name in fd.calls, name


def test_product_train_step_on_a_batch_without_edges(host, monkeypatch):
    """Agents out of each other's range: no edges, so no per-edge CBF values; the step must still run (action loss only; the
    reference would produce NaN from the mean over an empty h_dot)."""
    from gcbf_b200 import synth
    fix = load_golden('macbf_simplecar_n20_b3')
    sb = synth.make_states('SimpleCar', 20, 0, 2, 500.0, 3)
    fd, env, algo = _product_algo(fix, sb, monkeypatch, host)
    data = synth.product_batch(env, sb, torch.device('cpu'))
    assert data.edge_index.shape[1] == 0
    before = {k: v.clone() for k, v in algo.cbf.state_dict().items()}
    res = algo.train_step(data)
    s = res['scalars'].tolist()
    want_la = float(torch.square(res['actions']).sum(dim=1).mean())
    assert s[0] == 0.0 and s[1] == 0.0 and s[2] == 0.0 and abs(s[3] - want_la) <= 1e-7 and s[4] == 1.0 and s[5] == 1.0 and s[7] == 1.0
    assert res['h'].shape == (0, 1) and all(torch.equal(v, before[k]) for k, v in algo.cbf.state_dict().items())      # zero CBF gradient
    assert 'gcbf_mlp_backward' in fd.calls and 'gcbf_clip_adam' in fd.calls


def test_factories_and_state_dict_contract():
    """make_env(max_neighbors) / make_algo('macbf' | 'nominal') exist with the reference's signatures; the MACBF networks carry the
    reference's state-dict keys and, seeded like the reference (GCBF nets drawn first), its initial weights."""
    from gcbf_b200.algo import MACBF, Nominal, make_algo
    from gcbf_b200.env import make_env
    from gcbf_b200.trainer.utils import read_params
    fix = load_golden('macbf_dubins_n24_o6_b3')
    dev = torch.device('cpu')
    env = make_env('DubinsCar', 24, dev, max_neighbors=12)
    assert env._max_neighbors == 12
    with pytest.raises(ValueError):
        make_env('DubinsCar', 24, dev, max_neighbors=0)
    torch.manual_seed(0)
    algo = make_algo('macbf', env, 24, env.node_dim, env.edge_dim, env.action_dim, dev, 512, read_params('DubinsCar', 'macbf'))
    assert isinstance(algo, MACBF) and algo.params['loss_h_dot_coef'] == 1.0 and algo.params['loss_action_coef'] == 0.0005
    for mod, key in ((algo.cbf, 'cbf_init'), (algo.actor, 'actor_init')):
        sd = mod.state_dict()
        assert list(sd.keys()) == list(fix[key].keys())
        for k, v in sd.items():
            assert torch.allclose(v, fix[key][k], rtol=0, atol=1e-6), k      # bit-equal on the same host; LAPACK's QR differs across CPUs
    fast = MACBF(env, 24, env.node_dim, env.edge_dim, env.action_dim, dev, reference_rng=False)
    assert list(fast.actor.state_dict().keys()) == list(fix['actor_init'].keys())
    with pytest.raises(NotImplementedError):
        algo.use_device_replay()
    nom = make_algo('nominal', env, 24, env.node_dim, env.edge_dim, env.action_dim, dev)
    assert isinstance(nom, Nominal)
    with pytest.raises(NotImplementedError):
        make_algo('ppo', env, 24, env.node_dim, env.edge_dim, env.action_dim, dev)
    for e in ('SimpleCar', 'SimpleDrone', 'DubinsCar'):
        assert read_params(e, 'macbf') == MO.HYPERPARAMS[e]


def test_macbf_still_has_no_cpu_fallback():
    from gcbf_b200.algo import MACBF
    from gcbf_b200.env import make_env
    dev = torch.device('cpu')
    env = make_env('SimpleCar', 8, dev, max_neighbors=12)
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        env.graph_from_states(torch.rand(8, 4), with_u_ref=False)
    algo = MACBF(env, 8, 4, 4, 2, dev, reference_rng=False)
    from gcbf_b200.data import Data
    d = Data(x=torch.zeros(8, 4), states=torch.rand(8, 4), edge_index=torch.tensor([[1, 0], [0, 1]]), edge_attr=torch.rand(2, 4), u_ref=torch.zeros(8, 2))
    with pytest.raises(RuntimeError, match='no CPU fallback'):
        algo.cbf(d)


def test_ctypes_signatures_match_the_header():
    """Every prototype of include/gcbf_b200.h against the ctypes signature the Python binding registers for it: same number of
    parameters, same kind (pointer / int32 / int64 / float / double / size_t) in every position, same return kind.  A mismatch would
    not fail at import -- it would silently shift arguments on the GPU box."""
    import re
    from gcbf_b200 import _C, native  # noqa: F401  (native registers the chain-level signatures)
    text = open(os.path.join(ROOT, 'include', 'gcbf_b200.h')).read()
    text = re.sub(r'/\*.*?\*/', ' ', text, flags=re.S)
    protos = re.findall(r'^\s*((?:const\s+)?[\w ]+?\**)\s+(gcbf_\w+)\s*\(([^;{}]*)\)\s*;', text, flags=re.M)
    assert len(protos) >= 60

    def c_kind(decl):
        d = decl.strip()
        if '*' in d or '[' in d:
            return 'ptr'
        d = re.sub(r'\b\w+$', '', d).strip() if len(d.split()) > 1 else d      # drop the parameter name
        d = d.replace('const', '').strip()
        return {'int': 'i32', 'int32_t': 'i32', 'int64_t': 'i64', 'long long': 'i64', 'unsigned long long': 'i64', 'float': 'f32',
                'double': 'f64', 'size_t': 'size', 'void': 'void', 'char': 'i8'}[d]

    def py_kind(t):
        if t is None:
            return 'void'
        if t in (ctypes.c_void_p, ctypes.c_char_p) or issubclass(t, ctypes._Pointer):
            return 'ptr'
        return {ctypes.c_int: 'i32', ctypes.c_int32: 'i32', ctypes.c_int64: 'i64', ctypes.c_longlong: 'i64', ctypes.c_ulonglong: 'i64',
                ctypes.c_float: 'f32', ctypes.c_double: 'f64', ctypes.c_size_t: 'size'}[t]

    seen = set()
    for ret, name, params in protos:
        assert name in _C._SIGS, f'{name} is declared in the header but has no ctypes signature'
        seen.add(name)
        res, args = _C._SIGS[name]
        want = [] if params.strip() in ('', 'void') else [c_kind(p) for p in params.split(',')]
        got = [py_kind(a) for a in args]
        assert got == want, f'{name}: header {want} vs ctypes {got}'
        assert py_kind(res) == c_kind(ret + ' x'), name
    assert set(_C._SIGS) <= seen, set(_C._SIGS) - seen


# ---- data-parallel MACBF step: two gloo ranks on the fake device == one process ---------------------------------------------------
class _Setter:
    def setattr(self, obj, name, value):
        setattr(obj, name, value)


def _dp_worker(rank, world, port, so_path, case, out_dir):
    import torch.distributed as dist
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        import fake_device
        from gcbf_b200 import synth
        from gcbf_b200.algo import make_algo
        from gcbf_b200.distributed import shard_range
        from gcbf_b200.env import make_env
        torch.set_num_threads(1)
        lib = ctypes.CDLL(so_path)
        lib.host_radius_graph_topk.restype = ctypes.c_int64
        fake_device.install(_Setter(), lib)
        fix = load_golden(case)
        meta, sb = _inputs(fix)
        dev = torch.device('cpu')
        env = make_env(sb.env, sb.num_agents, dev)
        params = env.default_params
        params.update({'num_obs': sb.num_obs, 'area_size': sb.area_size})
        env = make_env(sb.env, sb.num_agents, dev, params=params, max_neighbors=12)
        algo = make_algo('macbf', env, sb.num_agents, env.node_dim, env.edge_dim, env.action_dim, dev, 512, MO.HYPERPARAMS[sb.env])
        algo.cbf.load_state_dict(fix['cbf_init'])
        algo.actor.load_state_dict(fix['actor_init'])
        lo, hi = shard_range(sb.num_graphs, world, rank)            # 3 graphs on 2 ranks: unequal shares
        N = sb.nodes_per_graph
        mine = synth.SynthBatch(sb.env, sb.num_agents, sb.num_obs, hi - lo, sb.area_size, sb.states[lo * N:hi * N].contiguous(), sb.goals, sb.obs)
        data = synth.product_batch(env, mine, dev)
        scal = [algo.train_step(data)['scalars'].tolist() for _ in fix['steps']]
        torch.save(dict(scalars=scal, cbf={k: v.clone() for k, v in algo.cbf.state_dict().items()},
                        actor={k: v.clone() for k, v in algo.actor.state_dict().items()}, share=(lo, hi)), os.path.join(out_dir, f'r{rank}.pt'))
    finally:
        dist.destroy_process_group()


def test_two_gloo_ranks_equal_one_process(host, tmp_path):
    """Environment-parallel MACBF: each rank steps its own graphs, the 16 partial sums are all-reduced before the loss gradients are
    formed and the flat gradient bucket after the backward, so both ranks must report the single-process losses / accuracies (= the
    reference's, from the fixture) and end with identical weights equal to the single-process ones."""
    import socket
    import torch.multiprocessing as mp
    case = 'macbf_dubins_n24_o6_b3'
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    so_path = os.path.join(ROOT, 'tests', 'host_driver', '_build', 'macbf_host.so')
    mp.spawn(_dp_worker, args=(2, port, so_path, case, str(tmp_path)), nprocs=2, join=True)
    fix = load_golden(case)
    r0, r1 = (torch.load(os.path.join(tmp_path, f'r{r}.pt'), weights_only=False) for r in (0, 1))
    assert r0['share'] == (0, 2) and r1['share'] == (2, 3)
    for res in (r0, r1):
        for s, gold in zip(res['scalars'], fix['steps']):
            for i, tag in enumerate(('loss/unsafe', 'loss/safe', 'loss/derivative', 'loss/action', 'acc/unsafe', 'acc/safe')):
                assert abs(s[i] - gold['scalars'][tag]) <= 2e-6, (tag, s[i], gold['scalars'][tag])
            assert abs(s[7] - gold['scalars']['acc/derivative']) <= 1e-6
        assert not digest_close(res['cbf'], fix['cbf_final'], 1e-5, 1e-5, flip=3e-6)
        assert not digest_close(res['actor'], fix['actor_final'], 1e-5, 1e-5, flip=3e-6)
    for k in r0['cbf']:
        assert torch.equal(r0['cbf'][k], r1['cbf'][k]), k               # replicas stay bit-identical
    for k in r0['actor']:
        assert torch.equal(r0['actor'][k], r1['actor'][k]), k


@pytest.mark.parametrize('env,seed', [(e, s) for e in ('SimpleCar', 'DubinsCar', 'SimpleDrone') for s in range(4)])
def test_kernel_arithmetic_topk_properties(host, env, seed):
    """Size-independent properties of the filtered graph: a subset of the unfiltered radius graph, sorted (target, source), in-degree
    capped at k (k + 1 for torch_cluster's rule when the target itself is not among the first hits), identical to the unfiltered
    graph once k covers every node, and monotone in k."""
    from gcbf_b200 import synth
    g = torch.Generator().manual_seed(100 + seed)
    n = int(torch.randint(5, 40, (1,), generator=g))
    o = 0 if env == 'SimpleCar' else (n if env == 'SimpleDrone' else int(torch.randint(0, 9, (1,), generator=g)))
    B = int(torch.randint(1, 4, (1,), generator=g))
    area = float(torch.rand(1, generator=g)) * 2.5 + 0.4
    sb = synth.make_states(env, n, o, B, area, 500 + seed)
    N = sb.nodes_per_graph
    full = O.batch_radius_graph(env, sb.states, B, N, n)
    full_set = set(map(tuple, full.t().tolist()))
    prev = None
    for k in (1, 2, 5, 12, N + 1):
        ei, rowptr = host_topk(host, env, sb.states, B, N, n, k)
        pairs = list(map(tuple, ei.t().tolist()))
        assert set(pairs) <= full_set
        assert pairs == sorted(pairs, key=lambda p: (p[1], p[0]))
        deg = torch.bincount(ei[1], minlength=B * N) if ei.numel() else torch.zeros(1, dtype=torch.long)
        assert int(deg.max()) <= (k + 1 if env == 'SimpleCar' else k)
        assert torch.equal(torch.diff(rowptr.long()), deg[torch.arange(B * N).reshape(B, N)[:, :n].reshape(-1)]) if ei.numel() else True
        if prev is not None:
            assert prev <= set(pairs)                       # a larger k never drops an edge
        prev = set(pairs)
    assert prev == full_set


# ---- the kernel bodies themselves on an emulated grid (tests/host_driver/cuda_emu.h) ---------------------------------------------
@pytest.fixture(scope='module')
def grid():
    out = os.path.join(ROOT, 'tests', 'host_driver', '_build')
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, 'macbf_grid.so')
    subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-I', os.path.join(ROOT, 'gcbf-pytorch_b200', 'csrc'),
                           '-I', os.path.join(ROOT, 'include'), '-I', os.path.join(ROOT, 'tests', 'host_driver'), '-o', so,
                           os.path.join(ROOT, 'tests', 'host_driver', 'macbf_grid.cpp')])
    return ctypes.CDLL(so)


STRIDE_GEOMETRIES = [(1, 1), (3, 7), (2, 256), (1056, 256)]      # one thread striding over everything ... more threads than work


@pytest.mark.parametrize('case', CASES)
def test_kernel_bodies_on_an_emulated_grid(host, grid, case):
    """csrc/macbf_kernels.cuh compiled as C++ and run thread by thread: bit-equal to the per-element driver / the fixture in every launch
    geometry (indexing, pitches, grid-stride loops, untouched padding).  The library launches the top-k kernel with 128-thread blocks,
    one thread per target; the others as grid-stride loops over at most 8 x 132 blocks of 256."""
    fix = load_golden(case)
    meta, sb = _inputs(fix)
    env, n, o, B = sb.env, sb.num_agents, sb.num_obs, sb.num_graphs
    N, p = n + o, O.ENV_PARAMS[env]
    f, i64 = ctypes.c_float, ctypes.c_int64
    metric = 0 if env == 'SimpleCar' else 1
    st = torch.cat([sb.states, torch.full((B * N, 3), 9.0)], dim=1).contiguous()           # a pitch larger than the state width
    want_ei = fix['edge_index']
    E = want_ei.shape[1]
    for blocks, threads in ((-(-B * n // 128), 128), (B * n, 1), (1, 1024)):
        if blocks * threads < B * n:
            continue
        rowptr = torch.zeros(B * n + 1, dtype=torch.int32)
        grid.grid_radius_topk_count(blocks, threads, _p(st), st.shape[1], p['pos_dim'], B, N, n, f(p['comm_radius']), metric, 12, _p(rowptr))
        rowptr[1:] = torch.cumsum(rowptr[:-1].clone(), 0).int()
        rowptr[0] = 0
        assert int(rowptr[-1]) == E
        ei = torch.full((2, E), -1, dtype=torch.int64)
        grid.grid_radius_topk_fill(blocks, threads, _p(st), st.shape[1], p['pos_dim'], B, N, n, f(p['comm_radius']), metric, 12, _p(rowptr), _p(ei), i64(E))
        assert torch.equal(ei, want_ei), (blocks, threads)
    ea = torch.cat([fix['edge_attr'], torch.full((E, 2), 9.0)], dim=1).contiguous()
    R = p['radius']
    for g_, b_ in STRIDE_GEOMETRIES:
        safe, unsafe = torch.full((E,), 7, dtype=torch.uint8), torch.full((E,), 7, dtype=torch.uint8)
        grid.grid_edge_masks(g_, b_, _p(ea), ea.shape[1], p['pos_dim'], i64(E), f(4 * R), f(2 * R), _p(safe), _p(unsafe))
        assert torch.equal(safe.bool(), fix['safe_mask']) and torch.equal(unsafe.bool(), fix['unsafe_mask']) and int(safe.max()) <= 1, (g_, b_)
    # max aggregation on this graph's CSR with random messages (padded pitches), against the per-element driver
    gen = torch.Generator().manual_seed(1)
    C, Nn = 37, B * N
    rp = torch.searchsorted(want_ei[1].contiguous(), torch.arange(Nn + 1)).int()
    msg = torch.randn(E, C + 3, generator=gen)
    ref_out, ref_arg = torch.full((Nn, C + 1), 7.0), torch.zeros(Nn, C, dtype=torch.int32)
    host.host_seg_max_fwd(_p(msg), C + 3, _p(rp), Nn, C, _p(ref_out), C + 1, _p(ref_arg))
    d_out = torch.randn(Nn, C + 1, generator=gen)
    ref_dmsg = torch.full((E, C + 2), 3.0)
    host.host_seg_max_bwd(_p(d_out), C + 1, _p(ref_arg), Nn, C, _p(ref_dmsg), C + 2, i64(E))
    for g_, b_ in STRIDE_GEOMETRIES:
        out, arg = torch.full((Nn, C + 1), 7.0), torch.zeros(Nn, C, dtype=torch.int32)
        grid.grid_seg_max_fwd(g_, b_, _p(msg), C + 3, _p(rp), Nn, C, _p(out), C + 1, _p(arg))
        assert torch.equal(out, ref_out) and torch.equal(arg, ref_arg), (g_, b_)
        d_msg = torch.zeros(E, C + 2)                                   # (the entry point zero-fills before the launch)
        grid.grid_seg_max_bwd(g_, b_, _p(d_out), C + 1, _p(arg), Nn, C, _p(d_msg), C + 2)
        assert torch.equal(d_msg, ref_dmsg), (g_, b_)
    # loss gradients + scalars from given partial sums
    M, ad = B * n, p['action_dim']
    h, hn = (torch.randn(E, generator=gen) * 0.05).contiguous(), (torch.randn(E, generator=gen) * 0.05).contiguous()
    act = torch.randn(M, ad, generator=gen).contiguous()
    s8, u8 = fix['safe_mask'].to(torch.uint8).contiguous(), fix['unsafe_mask'].to(torch.uint8).contiguous()
    partial = torch.zeros(16, dtype=torch.float64)
    host.host_macbf_loss_partials(_p(h), _p(hn), _p(s8), _p(u8), i64(E), _p(act), ad, i64(M), f(1.0), f(0.02), f(0.03), _p(partial))
    ref = [torch.zeros(E), torch.zeros(E), torch.zeros(M, ad), torch.zeros(8)]
    host.host_macbf_loss_grads(_p(h), _p(hn), _p(s8), _p(u8), i64(E), _p(act), ad, i64(M), f(1.0), f(0.02), f(0.03), f(1.0), f(0.7), f(0.4), f(0.05),
                               _p(partial), *[_p(t) for t in ref])
    for g_, b_ in STRIDE_GEOMETRIES:
        got = [torch.full((E,), 7.0), torch.full((E,), 7.0), torch.full((M, ad), 7.0), torch.full((8,), 7.0)]
        grid.grid_macbf_loss_grads(g_, b_, _p(h), _p(hn), _p(s8), _p(u8), i64(E), _p(act), ad, i64(M), f(1.0), f(0.02), f(0.03), f(1.0), f(0.7), f(0.4),
                                   f(0.05), _p(partial), *[_p(t) for t in got])
        assert all(torch.equal(a, b) for a, b in zip(got, ref)), (g_, b_)
