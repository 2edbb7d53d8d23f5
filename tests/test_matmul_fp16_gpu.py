"""The one-product tensor-core mode (gcbf_linear_*_h with products = 1; GCBF.params['matmul'] = 'fp16') on the GPU.

  * per product: every product kind, both tile widths, ragged shapes, split-K, per-tensor and tile-scaled operands, strided outputs
    and accumulation, each element within the bound derived in tests/matmul_fp16_model.py against float64 of the fp32 operands;
  * emission: the companion a one-product launch writes is split_tiled(its own fp32 output), bit for bit; column sums and the
    hi-plane ReLU mask against float64;
  * the train step: bit-identical to fp32 mode where no layer reaches the tensor cores (C1), within the stated bounds at C2 against
    the oracle and against fp32 mode (h, u, losses, per-net gradient cosine), bit-reproducible, and a short vectorised training run.
"""
import ctypes
import math

import numpy as np
import pytest
import torch

import fp16x3_model as F16
import gcbf_oracle as O
import matmul_fp16_model as F1
from gcbf_b200 import _C, native, ops, synth
from helpers import oracle_batch, per_tensor, product_batch, sd_clone, seeded_algo, tiled_buffers

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0') if torch.cuda.is_available() else None
L_MAX = 256          # the longest promotion chunk (data-grad with a per-tensor weight: 8 k-blocks of 32)


def _g(seed):
    return torch.Generator().manual_seed(seed)


def strided(rows, cols, extra=5):
    """[rows, cols] output view inside a NaN-filled buffer of pitch cols + extra."""
    buf = torch.full((rows, cols + extra), float('nan'), device=DEV)
    return buf, buf[:, :cols], cols + extra


def _np(t):
    return t.detach().cpu().double().numpy()


def _assert_bound(got, ref, bd, what):
    err = np.abs(_np(got) - ref)
    ratio = float((err / np.maximum(bd, 1e-300)).max())
    assert np.all(err <= bd), f'{what}: max err / bound = {ratio:.3f}'
    return ratio


def _conservative(Kc):
    """(chunk, chunks, splits) that over-count every schedule: chunks and splits are at most the number of 32-element k-blocks."""
    kb = math.ceil(Kc / 32)
    return L_MAX, kb, kb


def fwd_h(X, W, b, alpha, act, y, ldy, Yh, M, N, K, products=1):
    native.check(native.fn('gcbf_linear_fwd_h')(ctypes.byref(X), ctypes.byref(W), _C.ptr(b), _C.ptr(alpha), act, _C.ptr(y), ldy,
                                                 ctypes.byref(Yh) if Yh is not None else None, None, M, N, K, _C.stream(), products),
                 'gcbf_linear_fwd_h')


# ---- per-product bound ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M,N,K,bias', [(777, 260, 300, True), (513, 128, 200, False), (300, 2048, 1000, True), (256, 97, 2048, False)])
def test_forward_within_bound(M, N, K, bias):
    g = _g(M + N + K)
    x = torch.randn(M, K, generator=g) * torch.logspace(0, -5, M).unsqueeze(1)
    W = torch.randn(N, K, generator=g) / math.sqrt(K)
    b = torch.randn(N, generator=g) if bias else None
    xd, Wd = x.to(DEV), W.to(DEV)
    bd = b.to(DEV) if bias else None
    alpha = torch.tensor([0.7], device=DEV)
    X, k0 = per_tensor(xd)
    Wh, k1 = per_tensor(Wd)
    buf, y, ldy = strided(M, N)
    fwd_h(X, Wh, bd, alpha, ops.ACT_NONE, buf, ldy, None, M, N, K)
    torch.cuda.synchronize()
    a, bm = x.numpy(), W.t().contiguous().numpy()
    ref = 0.7 * (a.astype(np.float64) @ bm.astype(np.float64)) + (b.double().numpy()[None, :] if bias else 0.0)
    L, n, s = _conservative(K)
    bd_ = F1.bound(a, bm, F1.tensor_scales(a), F1.tensor_scales(bm), L, n, s, alpha=0.7, bias=b.numpy() if bias else None)
    r = _assert_bound(y, ref, bd_, 'forward')
    assert torch.isnan(buf[:, N:]).all(), 'padding written'
    print(f'fwd {M}x{N}x{K}: max err / bound {r:.3f}')


@pytest.mark.parametrize('M,N,K,accumulate,mask', [(777, 300, 260, 0, True), (513, 200, 128, 1, False), (1000, 2048, 2048, 0, True)])
def test_data_grad_within_bound(M, N, K, accumulate, mask):
    g = _g(M * 7 + N + K)
    dz = torch.randn(M, N, generator=g) * torch.logspace(-3, 0, M).unsqueeze(1)
    W = torch.randn(N, K, generator=g) / math.sqrt(N)
    src = torch.randn(M, K, generator=g)
    src[::7] = 0.0                                                   # exact zeros: masked
    prev = torch.randn(M, K, generator=g)
    dzd, Wd, srcd = dz.to(DEV), W.to(DEV), src.to(DEV)
    DZ, k0 = per_tensor(dzd)
    Wh, k1 = per_tensor(Wd)
    buf, dx, ld = strided(M, K)
    if accumulate:
        dx.copy_(prev.to(DEV))
    native.check(native.fn('gcbf_linear_bwd_data_h')(ctypes.byref(DZ), ctypes.byref(Wh), None, _C.ptr(srcd) if mask else None, K, None,
                                                      _C.ptr(buf), ld, accumulate, None, None, None, M, N, K, _C.stream(), 1), 'dgrad')
    torch.cuda.synchronize()
    a, bm = dz.numpy(), W.numpy()
    m = (src.numpy() > 0) if mask else np.ones((M, K), bool)
    ref = (a.astype(np.float64) @ bm.astype(np.float64)) * m + (prev.double().numpy() if accumulate else 0.0)
    L, n, s = _conservative(N)
    bd_ = F1.bound(a, bm, F1.tensor_scales(a), F1.tensor_scales(bm), L, n, s, prev=prev.numpy() if accumulate else None)
    r = _assert_bound(dx, ref, bd_ * m + (F1.gamma(n + s + 4) * np.abs(prev.double().numpy()) if accumulate else 0.0), 'data-grad')
    assert torch.isnan(buf[:, K:]).all()
    print(f'dgrad {M}x{N}x{K}: max err / bound {r:.3f}')


@pytest.mark.parametrize('M,N,K,accumulate', [(4100, 130, 300, 0), (2000, 256, 128, 1), (9000, 2048, 2048, 0)])
def test_weight_grad_within_bound(M, N, K, accumulate):
    """Split-K at the first shape (17 contraction splits), BN 128 at the second, the C-sized layer at the third."""
    g = _g(M + 3 * N + K)
    dz = torch.randn(M, N, generator=g) * torch.logspace(-2, 0, M).unsqueeze(1)
    x = torch.relu(torch.randn(M, K, generator=g))
    prev = torch.randn(N, K, generator=g)
    DZ, k0 = per_tensor(dz.to(DEV))
    X, k1 = per_tensor(x.to(DEV))
    buf, dW, ld = strided(N, K)
    if accumulate:
        dW.copy_(prev.to(DEV))
    native.check(native.fn('gcbf_linear_bwd_weight_h')(ctypes.byref(DZ), ctypes.byref(X), None, _C.ptr(buf), ld, accumulate, M, N, K,
                                                        _C.stream(), 1), 'wgrad')
    torch.cuda.synchronize()
    a, bm = dz.t().contiguous().numpy(), x.numpy()
    ref = a.astype(np.float64) @ bm.astype(np.float64) + (prev.double().numpy() if accumulate else 0.0)
    L, n, s = _conservative(M)
    bd_ = F1.bound(a, bm, F1.tensor_scales(a), F1.tensor_scales(bm), L, n, s, prev=prev.numpy() if accumulate else None)
    r = _assert_bound(dW, ref, bd_, 'weight-grad')
    assert torch.isnan(buf[:, K:]).all()
    print(f'wgrad {M}x{N}x{K}: max err / bound {r:.3f}')


# ---- tile-scaled operands and emission ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('M,N,K', [(1000, 2048, 2048), (700, 512, 300), (2500, 256, 1024)])
def test_emission_and_tile_scaled_operands(M, N, K):
    """y1 = relu(x W1^T) emitted by a one-product forward: its companion is split_tiled(y1) bit for bit.  Then the three products
    read tile-scaled operands: forward from y1's companion, data-grad with the ReLU mask from y1's hi plane, emitting dx with column
    sums, and weight-grads with one and with both operands tile-scaled -- each within the bound."""
    g = _g(M * 3 + N + K)
    x = torch.randn(M, K, generator=g) * torch.logspace(-1, 1, M).unsqueeze(1)
    W1, W2 = torch.randn(K, K, generator=g) / math.sqrt(K), torch.randn(N, K, generator=g) / math.sqrt(K)
    dz = torch.randn(M, N, generator=g) * torch.logspace(-4, -2, M).unsqueeze(1)
    xd, W1d, W2d, dzd = x.to(DEV), W1.to(DEV), W2.to(DEV), dz.to(DEV)
    X, k0 = per_tensor(xd)
    W1h, k1 = per_tensor(W1d)
    W2h, k2 = per_tensor(W2d)
    y1 = torch.empty(M, K, device=DEV)
    y1d, y1buf, y1amax = tiled_buffers(M, K)
    fwd_h(X, W1h, torch.zeros(K, device=DEV), None, ops.ACT_RELU, y1, K, y1d, M, K, K)
    torch.cuda.synchronize()
    hi, lo, amax = F16.split_tiled(y1.cpu())
    assert torch.equal(y1amax.view(torch.float32).cpu(), amax)
    assert torch.equal(y1buf[0, :, :K].cpu(), hi) and torch.equal(y1buf[1, :, :K].cpu(), lo)
    a1 = y1.cpu().numpy()
    s1 = F1.tile_scales(a1)
    # forward from the emitted (tile-scaled) companion
    y2 = torch.empty(M, N, device=DEV)
    fwd_h(y1d, W2h, None, None, ops.ACT_NONE, y2, N, None, M, N, K)
    w2t = W2.t().contiguous().numpy()
    L, n, s = _conservative(K)
    _assert_bound(y2, a1.astype(np.float64) @ w2t.astype(np.float64), F1.bound(a1, w2t, s1, F1.tensor_scales(w2t), L, n, s), 'forward (tiled A)')
    # data-grad: mask from y1's hi plane, dx emitted + fp32, column sums
    DZ, k3 = per_tensor(dzd)
    dx = torch.empty(M, K, device=DEV)
    dxd, dxbuf, dxamax = tiled_buffers(M, K)
    colsum = torch.zeros(K, device=DEV)
    native.check(native.fn('gcbf_linear_bwd_data_h')(ctypes.byref(DZ), ctypes.byref(W2h), None, None, 0, ctypes.byref(y1d), _C.ptr(dx), K, 0,
                                                      ctypes.byref(dxd), _C.ptr(colsum), None, M, N, K, _C.stream(), 1), 'dgrad')
    torch.cuda.synchronize()
    mask = a1 > 0
    a, bm = dz.numpy(), W2.numpy()
    L, n, s = _conservative(N)
    bdx = F1.bound(a, bm, F1.tensor_scales(a), F1.tensor_scales(bm), L, n, s) * mask
    _assert_bound(dx, (a.astype(np.float64) @ bm.astype(np.float64)) * mask, bdx, 'data-grad (hi-plane mask)')
    hi, lo, amax = F16.split_tiled(dx.cpu())
    assert torch.equal(dxamax.view(torch.float32).cpu(), amax)
    assert torch.equal(dxbuf[0, :, :K].cpu(), hi) and torch.equal(dxbuf[1, :, :K].cpu(), lo)
    dx64 = _np(dx)
    cs_bound = F1.gamma(M + 8) * np.abs(dx64).sum(0)                                   # an M-term fp32 sum of the kernel's own values
    assert np.all(np.abs(_np(colsum) - dx64.sum(0)) <= cs_bound)
    # weight-grads: both operands tile-scaled (dx, y1), and a per-tensor dZ with the tile-scaled y1
    dW = torch.empty(K, K, device=DEV)
    native.check(native.fn('gcbf_linear_bwd_weight_h')(ctypes.byref(dxd), ctypes.byref(y1d), None, _C.ptr(dW), K, 0, M, K, K, _C.stream(), 1),
                 'wgrad')
    dW2 = torch.empty(N, K, device=DEV)
    native.check(native.fn('gcbf_linear_bwd_weight_h')(ctypes.byref(DZ), ctypes.byref(y1d), None, _C.ptr(dW2), K, 0, M, N, K, _C.stream(), 1),
                 'wgrad2')
    torch.cuda.synchronize()
    dxf = dx.cpu().numpy()
    L, n, s = _conservative(M)
    _assert_bound(dW, dxf.T.astype(np.float64) @ a1.astype(np.float64),
                  F1.bound(np.ascontiguousarray(dxf.T), a1, F1.tile_scales(dxf).T, s1, L, n, s), 'weight-grad (both tiled)')
    dzt = np.ascontiguousarray(dz.numpy().T)
    _assert_bound(dW2, dzt.astype(np.float64) @ a1.astype(np.float64), F1.bound(dzt, a1, F1.tensor_scales(dzt), s1, L, n, s),
                  'weight-grad (tiled B)')


def test_products_argument_is_checked():
    x = torch.randn(256, 128, device=DEV)
    X, k0 = per_tensor(x)
    W, k1 = per_tensor(torch.randn(128, 128, device=DEV))
    y = torch.empty(256, 128, device=DEV)
    for bad in (0, 2, 4, -1):
        rc = native.fn('gcbf_linear_fwd_h')(ctypes.byref(X), ctypes.byref(W), None, None, 0, _C.ptr(y), 128, None, None, 256, 128, 128,
                                            _C.stream(), bad)
        assert rc != 0
    # products = 3 is the default (3xFP16) path, bit for bit
    fwd_h(X, W, None, None, 0, y, 128, None, 256, 128, 128, products=3)
    y3 = ops.linear_fwd_h(k0, k1, None, None, 0)
    assert torch.equal(y, y3)


# ---- the train step ---------------------------------------------------------------------------------------------------------------
def _case(cfg, matmul):
    c = dict(synth.CONFIGS[cfg])
    sb = synth.make_states(**c)
    from gcbf_b200.trainer.utils import read_params
    hp = dict(read_params(sb.env, 'gcbf'), matmul=matmul)
    env, algo = seeded_algo(sb.env, sb.num_agents, DEV, 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size}, hyperparams=hp)
    return sb, env, algo, product_batch(env, sb, DEV)


def _grads(algo):
    return {name: torch.cat([p.grad.reshape(-1).double() for p in m.parameters()]) for name, m in (('cbf', algo.cbf), ('actor', algo.actor))}


def _step(cfg, matmul):
    sb, env, algo, data = _case(cfg, matmul)
    res = algo.train_step(data, apply_optim=False)
    torch.cuda.synchronize()
    out = {k: v.detach().clone() for k, v in res.items() if torch.is_tensor(v)}
    return sb, out, _grads(algo), algo, data


def test_c1_is_bit_identical_in_both_modes():
    """C1 (16 agents, one graph): no layer reaches the tensor cores, so the step, apply, apply_batch and cbf_field give the same bits."""
    runs = []
    for mode in ('fp32', 'fp16'):
        sb, out, grads, algo, data = _step('C1', mode)
        assert not ops.use_h(int(data.edge_index.shape[1]), 2048, 2048)
        single = data
        a = algo.apply(single, rand=0)
        from gcbf_b200.data import Batch
        ab = algo.apply_batch(Batch.from_data_list([single, single]), rand=0)
        lims = (single.states.min(0).values, single.states.max(0).values)
        xs, ys, h = algo.cbf_field(single, agents=[0], n_mesh=4, lims=lims)
        assert not ops.use_h(algo.last_field_edges, 2048, 2048)         # 16 probes: the field's passes stay off the tensor cores too
        torch.cuda.synchronize()
        runs.append((out, grads, a.clone(), ab.clone(), h.clone()))
    (o0, g0, a0, ab0, h0), (o1, g1, a1, ab1, h1) = runs
    for k in o0:
        assert torch.equal(o0[k], o1[k]), k
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    assert torch.equal(a0, a1) and torch.equal(ab0, ab1) and torch.equal(h0, h1)


# Stated bounds of the fp16 mode at C2 (SimpleCar, 32 graphs x 256 agents, seeded weights), each >= 4x the maximum measured on an
# H100 80GB HBM3 (700 W), one run: |dh| 1.95e-6 against the oracle and against fp32 mode, |du| 3.06e-4, losses 3.2e-6 (loss_action;
# total 1.3e-7), gradient cosine 1 - 6.2e-5 (CBF) and 1 - 2.5e-7 (actor)
C2_TOL_H = 1e-5
C2_TOL_U = 2e-3
C2_TOL_LOSS = 2e-5
C2_COS = 0.999


def test_c2_step_against_oracle_and_fp32_mode():
    _reset_counts()
    sb, o16, g16, algo, data = _step('C2', 'fp16')
    assert native.tc_launch_count(3) == 0 and native.tc_launch_count(1) > 0      # every tensor-core launch of the step: one product
    _, o32, g32, _, _ = _step('C2', 'fp32')
    sb2, env, algo_o, data_o = _case('C2', 'fp32')
    cbf, act = sd_clone(algo_o.cbf), sd_clone(algo_o.actor)
    ob = oracle_batch(sb2)
    want = O.update_step(sb2.env, cbf, act, {}, {}, sb2.states, sb2.goals, ob['edge_index'], ob['u_ref'], sb2.num_graphs, sb2.num_agents,
                         sb2.num_obs, K=ob['K'], apply_optim=False)
    md = lambda a, b: (a.detach().cpu().double().reshape(-1) - b.detach().cpu().double().reshape(-1)).abs().max().item()
    rec = dict(dh_oracle=md(o16['h'], want['h']), du_oracle=md(o16['actions'], want['actions']),
               dh_fp32=md(o16['h'], o32['h']), du_fp32=md(o16['actions'], o32['actions']),
               dloss=abs(float(o16['scalars'][6]) - float(want['loss'])),
               dlosses=[abs(float(o16['scalars'][i]) - float(o32['scalars'][i])) for i in range(4)])
    for k in g16:
        rec['cos_' + k] = float(torch.nn.functional.cosine_similarity(g16[k], g32[k], dim=0))
    print('c2-fp16', rec)
    assert rec['dh_oracle'] <= C2_TOL_H and 0 < rec['dh_fp32'] <= C2_TOL_H, rec
    assert rec['du_fp32'] > 0 and min(rec['cos_cbf'], rec['cos_actor']) < 1.0, rec                 # the step did change
    assert rec['du_oracle'] <= C2_TOL_U and rec['du_fp32'] <= C2_TOL_U, rec
    assert rec['dloss'] <= C2_TOL_LOSS and max(rec['dlosses']) <= C2_TOL_LOSS, rec
    assert rec['cos_cbf'] >= C2_COS and rec['cos_actor'] >= C2_COS, rec


def test_fp16_steps_are_bit_reproducible():
    runs = []
    for _ in range(2):
        sb, env, algo, data = _case('C2', 'fp16')
        for _ in range(3):
            res = algo.train_step(data)
        torch.cuda.synchronize()
        out = {k: v.detach().clone() for k, v in res.items() if torch.is_tensor(v)}
        out.update({'cbf.' + k: v.detach().clone() for k, v in algo.cbf.state_dict().items()})
        out.update({'actor.' + k: v.detach().clone() for k, v in algo.actor.state_dict().items()})
        runs.append(out)
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k


def test_short_vectorised_training_run_in_fp16(tmp_path):
    from gcbf_b200.env import make_env
    from gcbf_b200.trainer import Trainer
    from gcbf_b200.trainer.utils import read_params, set_seed
    set_seed(0)
    hp = dict(read_params('SimpleCar', 'gcbf'), matmul='fp16')
    env, algo = seeded_algo('SimpleCar', 16, DEV, 0, None, hyperparams=hp)
    env_test = make_env('SimpleCar', 16, DEV, params=env._params)
    algo.batch_size = 64
    scalars = []
    step = algo.train_step

    def recorded(*a, **k):
        res = step(*a, **k)
        scalars.append(res['scalars'].detach().clone())
        return res

    algo.train_step = recorded
    tr = Trainer(env, env_test, algo, str(tmp_path / 'fp16'), num_envs=8, seed=0)
    native.tc_launch_count(1, True), native.tc_launch_count(3, True)
    tr.train(64, 64, 2)
    assert scalars and all(bool(torch.isfinite(s).all()) for s in scalars)
    assert native.tc_launch_count(1) > 0 and native.tc_launch_count(3) == 0      # the updates' tensor-core layers ran one-product kernels


def _reset_counts():
    native.tc_launch_count(1, True)
    native.tc_launch_count(3, True)


def _counts():
    return native.tc_launch_count(3), native.tc_launch_count(1)


def test_mode_set_after_construction_reaches_the_modules():
    """params['matmul'] changed on the dict after construction: the next algo.actor(data) -- no GCBF entry point in between, as in
    VectorRollout -- already runs the one-product kernels, and back."""
    sb = synth.make_states('DubinsCar', 64, 8, 2, 3.0, 7)
    env, algo = seeded_algo('DubinsCar', 64, DEV, 0, {'num_obs': 8, 'area_size': 3.0})
    data = product_batch(env, sb, DEV)
    assert ops.use_h(int(data.edge_index.shape[1]), 2048, 2048)
    with torch.no_grad():
        for mode, want in (('fp16', 1), ('fp32', 3), ('fp16', 1)):
            algo.params['matmul'] = mode
            _reset_counts()
            algo.actor(data)
            algo.cbf(data)
            torch.cuda.synchronize()
            n3, n1 = _counts()
            assert (n1 > 0 and n3 == 0) if want == 1 else (n3 > 0 and n1 == 0), (mode, n3, n1)


# ---- net level: gcbf_net_forward / _backward of both nets against a float64 replica ------------------------------------------------
# Bounds, fp16 mode against float64 (>= 4x the maximum measured on an H100 80GB HBM3, 700 W, one run: |dh| 1.3e-6, |du| 1.4e-6, largest
# relative error of a 2048-wide weight gradient 2.3e-2, of a whole net's gradient 8.8e-3 -- fp32 mode: 1.1e-8, 1.3e-8, 4.3e-5, 3.7e-5)
NET_TOL_H = 1e-5
NET_TOL_U = 1e-5
NET_TOL_GRAD_WIDE = 0.1      # per 2048-wide weight, ||g - g64|| / ||g64||
NET_TOL_GRAD_NET = 4e-2      # per net, over all its parameters


def test_net_passes_run_one_product_kernels_and_match_float64():
    """CBF and actor forward + backward through the module API (gcbf_net_forward / gcbf_net_backward) on a graph whose phi / gate / gamma
    layers run on the wgmma kernels (E ~ 2.3 k): in fp16 mode every tensor-core launch of the passes is a one-product launch -- as many
    as fp32 mode issues three-product ones -- and h, u and every parameter gradient are within the stated bounds of a float64 replica
    (oracle/gcbf_oracle.py in float64 on the same weights and spectral-norm state), further from it than fp32 mode is."""
    from gcbf_b200.data import agent_row_index
    from gcbf_b200.trainer.utils import read_params
    sb = synth.make_states('DubinsCar', 64, 8, 2, 3.0, 31)
    res = {}
    for mode in ('fp32', 'fp16'):
        hp = dict(read_params('DubinsCar', 'gcbf'), matmul=mode)
        env, algo = seeded_algo('DubinsCar', 64, DEV, 0, {'num_obs': 8, 'area_size': 3.0}, hyperparams=hp)
        data = product_batch(env, sb, DEV)
        assert ops.use_h(int(data.edge_index.shape[1]), 2048, 2048)
        sds = {'cbf': sd_clone(algo.cbf), 'actor': sd_clone(algo.actor)}          # the spectral-norm state the pass starts from
        g = torch.Generator().manual_seed(5)
        _reset_counts()
        h, u = algo.cbf(data), algo.actor(data)
        wh, wu = torch.randn(h.shape, generator=g).to(DEV), torch.randn(u.shape, generator=g).to(DEV)
        ((h * wh).sum() + (u * wu).sum()).backward()
        torch.cuda.synchronize()
        counts = _counts()
        grads = {n + '.' + k: p.grad.detach().double().cpu() for n, m in (('cbf', algo.cbf), ('actor', algo.actor)) for k, p in m.named_parameters()}
        res[mode] = (h.detach().double().cpu(), u.detach().double().cpu(), grads, counts)
    (n3_32, n1_32), (n3_16, n1_16) = res['fp32'][3], res['fp16'][3]
    assert n3_32 > 0 and n1_32 == 0, res['fp32'][3]
    assert n3_16 == 0 and n1_16 == n3_32, res['fp16'][3]
    # float64 replica
    rows = agent_row_index(data)
    x, ea, ei = data.x.double().cpu(), data.edge_attr.detach().double().cpu(), data.edge_index.cpu()
    rows = rows.cpu() if rows is not None else None
    sd64 = {}
    for n, m in (('cbf', algo.cbf), ('actor', algo.actor)):
        names = {k for k, _ in m.named_parameters()}
        sd64[n] = {k: v.double().requires_grad_(k in names) for k, v in sds[n].items()}
    h64 = O.cbf_forward(sd64['cbf'], x, ea, ei, rows)
    u64 = O.actor_forward(sd64['actor'], x, ea, ei, rows, data.u_ref.detach().double().cpu())
    ((h64 * wh.double().cpu()).sum() + (u64 * wu.double().cpu()).sum()).backward()
    g64 = {n + '.' + k: v.grad for n in ('cbf', 'actor') for k, v in sd64[n].items() if v.grad is not None}
    rec = {}
    wide = [k for k in g64 if g64[k].dim() == 2 and min(g64[k].shape) >= 2048]
    for mode in ('fp32', 'fp16'):
        h_, u_, gr, _ = res[mode]
        net_rel = {}
        for n in ('cbf', 'actor'):
            ks = [k for k in g64 if k.startswith(n + '.')]
            d = torch.cat([(gr[k] - g64[k]).reshape(-1) for k in ks])
            net_rel[n] = (d.norm() / torch.cat([g64[k].reshape(-1) for k in ks]).norm()).item()
        rec[mode] = dict(dh=(h_ - h64.detach()).abs().max().item(), du=(u_ - u64.detach()).abs().max().item(),
                         grad_rel_net=max(net_rel.values()),
                         grad_rel_wide=max(((gr[k] - g64[k]).norm() / g64[k].norm()).item() for k in wide))
    print('net-fp16', rec)
    r16, r32 = rec['fp16'], rec['fp32']
    assert r16['dh'] <= NET_TOL_H and r16['du'] <= NET_TOL_U, r16
    assert r16['grad_rel_wide'] <= NET_TOL_GRAD_WIDE and r16['grad_rel_net'] <= NET_TOL_GRAD_NET, r16
    # the one-product arithmetic is visible in the results, not only in the counters
    assert r16['dh'] > 4 * r32['dh'] and r16['du'] > 4 * r32['du'] and r16['grad_rel_wide'] > 4 * r32['grad_rel_wide'], (r16, r32)


# ---- one C3 share and trained-like weights -----------------------------------------------------------------------------------------
def _two_mode_step(algo, data):
    """One train step in each mode from the same weights and spectral-norm state: {mode: (h, u, scalars, grads, counts)}."""
    snap = {n: {k: v.clone() for k, v in m.state_dict().items()} for n, m in (('cbf', algo.cbf), ('actor', algo.actor))}
    out = {}
    for mode in ('fp32', 'fp16'):
        algo.cbf.load_state_dict(snap['cbf'])
        algo.actor.load_state_dict(snap['actor'])
        algo.set_matmul(mode)
        _reset_counts()
        r = algo.train_step(data, apply_optim=False)
        torch.cuda.synchronize()
        out[mode] = (r['h'].detach().double().cpu(), r['actions'].detach().double().cpu(), r['scalars'].double().cpu(), _grads(algo), _counts())
    return out


def _compare_modes(out):
    (h32, u32, s32, g32, c32), (h16, u16, s16, g16, c16) = out['fp32'], out['fp16']
    assert c32[1] == 0 and c16[0] == 0 and c16[1] == c32[0] > 0, (c32, c16)
    return dict(dh=(h16 - h32).abs().max().item(), du=(u16 - u32).abs().max().item(), u_absmax=u32.abs().max().item(),
                h_absmax=h32.abs().max().item(), dloss=(s16[:4] - s32[:4]).abs().max().item(),
                cos_cbf=float(torch.nn.functional.cosine_similarity(g16['cbf'], g32['cbf'], dim=0)),
                cos_actor=float(torch.nn.functional.cosine_similarity(g16['actor'], g32['actor'], dim=0)))


# one GPU's C3 share (DubinsCar, 64 graphs x 1024 agents, 206 k edges, seeded weights): >= 4x the maximum measured on an H100 80GB HBM3
# (700 W), one run: |dh| 1.0e-5, |du| 1.7e-4, losses 1.1e-6, gradient cosine 1 - 1.4e-5 / 1 - 1.8e-6.  fp32 mode is itself within 1e-5
# of the oracle on this share (tests/test_fullsize_gpu.py).
C3_TOL_H = 5e-5
C3_TOL_U = 1e-3
C3_TOL_LOSS = 1e-5
C3_COS = 0.999


def test_c3_share_step_against_fp32_mode():
    sb, env, algo, data = _case('C3', 'fp32')
    rec = _compare_modes(_two_mode_step(algo, data))
    print('c3-fp16', rec)
    assert 0 < rec['dh'] <= C3_TOL_H and 0 < rec['du'] <= C3_TOL_U and rec['dloss'] <= C3_TOL_LOSS, rec
    assert rec['cos_cbf'] >= C3_COS and rec['cos_actor'] >= C3_COS, rec


# C2 with trained-like weights (tests/golden/pretrained_stats.pt statistics, as tests/test_fullsize_gpu.py builds them), >= 4x the maximum
# measured on an H100 80GB HBM3 (700 W), one run: |dh| 4.6e-7 (|h| <= 0.017), |du| 3.3e-4 (|u| <= 0.43), losses 5.6e-7, gradient
# cosine 1 - 6.0e-6 / 1 - 1.9e-7 -- far inside the 1e-2 the mode was aimed at.  u is compared relative to max(1, max|u|).
TRAINED_TOL_H = 2e-6
TRAINED_TOL_U_REL = 1.5e-3
TRAINED_TOL_LOSS = 5e-6
TRAINED_COS = 0.999


def test_c2_step_with_trained_like_weights():
    import os
    from conftest import GOLDEN_DIR
    from test_fullsize_gpu import _trained_like
    stats = torch.load(os.path.join(GOLDEN_DIR, 'pretrained_stats.pt'), weights_only=False)['SimpleCar']
    sb, env, algo, data = _case('C2', 'fp32')
    algo.cbf.load_state_dict({k: v.to(DEV) for k, v in _trained_like(sd_clone(algo.cbf), stats['cbf'], 5).items()})
    algo.actor.load_state_dict({k: v.to(DEV) for k, v in _trained_like(sd_clone(algo.actor), stats['actor'], 6).items()})
    rec = _compare_modes(_two_mode_step(algo, data))
    rec['du_rel'] = rec['du'] / max(1.0, rec['u_absmax'])
    print('c2-trained-like-fp16', rec)
    assert rec['dh'] <= TRAINED_TOL_H and rec['du_rel'] <= TRAINED_TOL_U_REL and rec['dloss'] <= TRAINED_TOL_LOSS, rec
    assert rec['cos_cbf'] >= TRAINED_COS and rec['cos_actor'] >= TRAINED_COS, rec
