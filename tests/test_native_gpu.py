"""(Run with GCBF_EPI_H=0 the two sequencings use the very same kernels and the forward outputs are bit-identical; by default the
library path lets the GEMM epilogues emit tile-scaled companions between tensor-core layers -- a different, slightly more accurate
rounding of the same products -- so the comparison allows 2e-6.)

The chain-level entry points (gcbf_net_forward / _backward, gcbf_mlp_*, gcbf_step_*: host sequencing inside the library,
csrc/net.cu + csrc/step.cu) against the per-kernel Python sequencing of round 1 (ops.net_forward / net_backward, GCBF._train_step):
same kernels in the same order, so outputs must agree to atomics-reordering noise.  (Parity against the ORACLE is in
test_parity_gpu.py / test_fullsize_gpu.py, which run through the chain-level path by default.)"""
import os

import pytest
import torch

from gcbf_b200 import _C, native, ops, synth
from gcbf_b200.data import agent_row_index
from gcbf_b200.nn.gnn import cached_rowptr
from helpers import product_batch, seeded_algo

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0') if torch.cuda.is_available() else None


def _setup(env_name, n, obs, B, area, seed):
    sb = synth.make_states(env_name, n, obs, B, area, seed)
    env, algo = seeded_algo(env_name, n, DEV, 0, {'num_obs': sb.num_obs, 'area_size': area})
    return sb, env, algo, product_batch(env, sb, DEV)


EMIT = os.environ.get('GCBF_EPI_H', '1') != '0'
GTOL = 3e-4 if EMIT else 1e-5        # gradients: a rounding-level ReLU flip moves a layer's gradient by ~1/sqrt(#units) of one row


def _close(a, b):
    if not EMIT:
        return torch.equal(a, b)
    return torch.allclose(a, b, rtol=0, atol=2e-6 * max(1.0, float(b.abs().max())))


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-300)).item()


@pytest.mark.parametrize('env_name,n,obs,B,area,impl', [('DubinsCar', 96, 6, 3, 3.0, 0), ('SimpleCar', 24, 0, 3, 1.5, 0),
                                                        ('SimpleDrone', 12, 12, 2, 1.0, 1), ('SimpleCar', 4, 0, 2, 50.0, 0)])
def test_net_pass_matches_python_sequencing(env_name, n, obs, B, area, impl):
    """CBF and actor pass, forward + backward (weight grads, bias grads, d_edge_attr), native vs Python sequencing; the last case
    is an edge-less batch (E = 0)."""
    outs = []
    old = ops.GEMM_IMPL
    ops.GEMM_IMPL = impl
    try:
        for nat in (False, True):
            sb, env, algo, data = _setup(env_name, n, obs, B, area, 81)
            ops.NATIVE = nat
            ea = data.edge_attr.detach().clone().requires_grad_(True)
            g = data
            from gcbf_b200.data import Data
            fields = dict(x=g.x, edge_index=g.edge_index, edge_attr=ea, u_ref=g.u_ref, states=g.states)
            if hasattr(g, 'agent_mask'):
                fields['agent_mask'] = g.agent_mask
            d2 = Data(**fields)
            h = algo.cbf(d2)
            u = algo.actor(d2)
            gen = torch.Generator().manual_seed(5)
            dh, du = torch.randn(h.shape, generator=gen).to(DEV), torch.randn(u.shape, generator=gen).to(DEV)
            torch.autograd.backward([h, u], [dh, du])
            torch.cuda.synchronize()
            outs.append(dict(h=h.detach().clone(), u=u.detach().clone(), dea=ea.grad.clone(),
                             gc=[p.grad.clone() for p in algo.cbf.parameters()], ga=[p.grad.clone() for p in algo.actor.parameters()],
                             uv=[v.clone() for k, v in algo.cbf.state_dict().items() if k.endswith(('_u', '_v'))]))
    finally:
        ops.NATIVE = True
        ops.GEMM_IMPL = old
    a, b = outs
    assert _close(a['h'], b['h']) and _close(a['u'], b['u'])          # forward: no atomics -> bit-identical without emission
    for x, y in zip(a['uv'], b['uv']):
        assert torch.equal(x, y)
    if a['dea'].numel():
        assert rel(b['dea'], a['dea']) < GTOL
    # per tensor, relative to the whole net's gradient norm (the last gate bias has an exactly-zero gradient -- softmax is shift
    # invariant -- so its entries are pure atomics-order noise)
    for key in ('gc', 'ga'):
        total = torch.sqrt(sum((g.double() ** 2).sum() for g in a[key]))
        for ga, gb in zip(a[key], b[key]):
            assert (gb.double() - ga.double()).norm() <= GTOL * ga.double().norm() + GTOL * 1e-2 * total, (ga.shape, rel(gb, ga))


@pytest.mark.parametrize('limit_lip', [False, True])
def test_bare_mlp_matches_python_sequencing(limit_lip):
    from gcbf_b200.nn import MLP
    outs = []
    try:
        for nat in (False, True):
            torch.manual_seed(3)
            mlp = MLP(260, 64, (2048, 512), limit_lip=limit_lip).to(DEV)
            ops.NATIVE = nat
            x = torch.randn(700, 260, generator=torch.Generator().manual_seed(1)).to(DEV).requires_grad_(True)
            y = mlp(x)
            y.backward(torch.randn(y.shape, generator=torch.Generator().manual_seed(2)).to(DEV))
            outs.append((y.detach().clone(), x.grad.clone(), [p.grad.clone() for p in mlp.parameters()]))
    finally:
        ops.NATIVE = True
    (ya, dxa, ga), (yb, dxb, gb) = outs
    assert _close(ya, yb)
    assert rel(dxb, dxa) < GTOL
    for p, q in zip(ga, gb):
        assert rel(q, p) < GTOL


@pytest.mark.parametrize('two_streams', ['0', '1'])
@pytest.mark.parametrize('env_name,n,obs,B,area', [('DubinsCar', 64, 8, 6, 4.0), ('SimpleCar', 48, 0, 4, 2.5), ('SimpleDrone', 16, 16, 3, 1.2),
                                                   ('DubinsCar', 16, 4, 1, 2.0)])
def test_train_step_matches_python_sequencing(monkeypatch, env_name, n, obs, B, area, two_streams):
    """gcbf_step_forward / _relink / _backward (+ clip / Adam) against the Python-sequenced train step: losses, outputs, re-linked
    edges, spectral-norm state, accumulated gradients (one step, before the optimizer) and the weights after the optimizer."""
    monkeypatch.setenv('GCBF_TWO_STREAMS', two_streams)
    outs = []
    try:
        for nat in (False, True):
            sb, env, algo, data = _setup(env_name, n, obs, B, area, 83)
            ops.NATIVE = nat
            res = algo.train_step(data, apply_optim=False)
            torch.cuda.synchronize()
            o = dict(s=res['scalars'].clone(), h=res['h'].clone(), u=res['actions'].clone(), hn=res['h_next'].clone(),
                     hnn=res['h_next_new'].clone().reshape(-1), ei=res['edge_index_new'].clone(), acc=float(res['acc_h_dot']),
                     hdot=res['hdot'].clone(), safe=res['safe_mask'].clone(), unsafe=res['unsafe_mask'].clone(),
                     g=algo._bucket.grad.clone(), uv=[v.clone() for k, v in algo.cbf.state_dict().items() if k.endswith(('_u', '_v'))])
            algo.optim_step()
            torch.cuda.synchronize()
            o['w'] = algo._bucket.flat.clone()
            outs.append(o)
    finally:
        ops.NATIVE = True
    a, b = outs
    assert torch.equal(a['ei'], b['ei']) and torch.equal(a['safe'], b['safe']) and torch.equal(a['unsafe'], b['unsafe'])
    for k in ('h', 'u', 'hn', 'hnn'):
        assert _close(a[k].reshape(-1), b[k].reshape(-1)), k
    assert torch.allclose(a['hdot'], b['hdot'], rtol=0, atol=(2e-6 / 0.03 if EMIT else 0.0))
    M = a['h'].numel()
    assert torch.allclose(a['s'], b['s'], rtol=0, atol=2e-6 if EMIT else 1e-7) and abs(a['acc'] - b['acc']) <= (2.0 / M if EMIT else 1e-12)
    for x, y in zip(a['uv'], b['uv']):
        assert torch.equal(x, y)
    assert a['g'].norm() > 0 and (a['g'] - b['g']).norm() <= (2e-2 if EMIT else 1e-5) * a['g'].norm()
    # clipped Adam's first step is +-lr per entry: entries whose gradient is rounding noise may flip, nothing moves further
    assert ((a['w'] - b['w']).abs() > 1e-7).float().mean().item() < (0.10 if EMIT else 0.02)


def test_step_workspace_grows_for_a_denser_relinked_graph():
    """gcbf_step_relink reports GCBF_E_WORKSPACE (+ the needed size) BEFORE launching when the re-linked graph does not fit, and
    the retry gives the same result as a roomy first attempt."""
    sb, env, algo, data = _setup('DubinsCar', 64, 8, 6, 4.0, 84)
    res = algo.train_step(data, apply_optim=False)
    want = res['h_next_new'].clone()
    sb, env, algo2, data = _setup('DubinsCar', 64, 8, 6, 4.0, 84)
    algo2._native_ws = (native.GrowBuffer(), native.GrowBuffer())
    algo2._native_ws[1].buf = native.workspace(4096, DEV)                # far too small: forces the retry path
    res2 = algo2.train_step(data, apply_optim=False)
    assert torch.equal(res2['h_next_new'], want)
    assert algo2._native_ws[1].buf.numel() > 4096


def test_abi_struct_mirrors_match_the_library():
    import ctypes
    mirrors = [_C.EnvCfg, native.LinearDesc, native.NetDesc, native.StepDesc, native.StepBatch, native.StepOut, native.NetCtx,
               native.MlpCtx, native.StepCtx, native.TimeRec, _C.SnLayer, _C.SplitDesc, native.H16Desc]
    for i, m in enumerate(mirrors):
        assert ctypes.sizeof(m) == _C.lib().gcbf_abi_struct_size(i), m.__name__


@pytest.mark.parametrize('env_name,n,obs,area,rand,max_iter', [('DubinsCar', 16, 4, 2.0, 0, 30), ('SimpleCar', 8, 0, 1.5, 0, 30),
                                                               ('SimpleDrone', 8, 8, 1.0, 0, 30), ('DubinsCar', 16, 4, 2.0, 30, 2),
                                                               ('SimpleCar', 4, 0, 50.0, 0, 5)])
def test_apply_matches_python_sequencing(env_name, n, obs, area, rand, max_iter):
    """gcbf_apply (csrc/apply.cu: the whole refinement loop + the per-agent Adam kernel in the library) against the Python-sequenced
    controller (autograd over the per-kernel ops), same weights, same noise draw.  Adam's normalised step amplifies rounding
    where a gradient component is ~0, hence the tolerance; with noise only a few rounds are compared.  Last case: no edges."""
    outs = []
    try:
        for nat in (False, True):
            sb, env, algo, data = _setup(env_name, n, obs, 1, area, 91)
            ops.NATIVE = nat
            single = env.graph_from_states(sb.states[:sb.nodes_per_graph].to(DEV))
            torch.manual_seed(7)
            a = algo.apply(single, rand=rand, max_iter=max_iter)
            torch.cuda.synchronize()
            outs.append((a.clone(), [v.clone() for k, v in algo.cbf.state_dict().items() if k.endswith(('_u', '_v'))],
                         getattr(algo, 'last_apply_rounds', None)))
    finally:
        ops.NATIVE = True
    (pa, puv, _), (na, nuv, rounds) = outs
    assert rounds is not None and 0 <= rounds <= max_iter + 1
    assert na.shape == pa.shape
    assert (na - pa).abs().max().item() <= 2e-3 * max(1.0, pa.abs().max().item()), (na - pa).abs().max().item()
    if rounds > 0:
        assert na.abs().max().item() > 0                 # somebody violated: the refined action is not the nominal zero
    for x, y in zip(puv, nuv):                           # the same number of CBF passes -> the same number of power iterations
        assert torch.allclose(x, y, atol=1e-5)


@pytest.mark.parametrize('env_name,n,obs,B,area,two_streams', [('DubinsCar', 64, 8, 4, 3.0, '0'), ('SimpleCar', 16, 0, 1, 4.0, '1'),
                                                              ('SimpleDrone', 24, 24, 3, 1.0, '1')])
def test_train_step_is_bit_reproducible(monkeypatch, env_name, n, obs, B, area, two_streams):
    """Two runs of three train steps from the same seeded weights on the same batch give bit-identical results and weights:
    reductions over blocks (split-K weight gradients, column sums, the edge-feature VJP) are summed in a fixed order, so the
    result does not depend on block scheduling.  The cases cover the tensor-core layers (with emission), the few-rows kernels
    of a single 16-agent graph, and the side stream."""
    monkeypatch.setenv('GCBF_TWO_STREAMS', two_streams)
    runs = []
    for _ in range(2):
        sb, env, algo, data = _setup(env_name, n, obs, B, area, 17)
        for _ in range(3):
            res = algo.train_step(data)
        torch.cuda.synchronize()
        out = {k: v.detach().clone() for k, v in res.items() if torch.is_tensor(v)}
        out.update({'cbf.' + k: v.detach().clone() for k, v in algo.cbf.state_dict().items()})
        out.update({'actor.' + k: v.detach().clone() for k, v in algo.actor.state_dict().items()})
        runs.append(out)
    assert runs[0].keys() == runs[1].keys()
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k
