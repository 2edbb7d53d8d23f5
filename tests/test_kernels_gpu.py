"""GPU unit tests: every C-ABI kernel against the CPU oracle (oracle/gcbf_oracle.py) or a plain torch fp32/fp64
restatement of the same op, on seeded inputs.  Integer / index outputs must be bit-exact; floating point within the
tolerance written next to each assert."""
import ctypes
import math

import pytest
import torch

import gcbf_oracle as O
from gcbf_b200 import _C, ops, synth
from helpers import oracle_batch, product_batch, seeded_algo

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0') if torch.cuda.is_available() else None


def _g(seed):
    g = torch.Generator(device='cpu')
    g.manual_seed(seed)
    return g


# ------------------------------------------------------------------------------------------------------
# K1 radius graph
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('env,n,obs,B,area', [('SimpleCar', 16, 0, 3, 2.0), ('SimpleCar', 67, 0, 2, 4.0),
                                              ('DubinsCar', 33, 7, 3, 3.0), ('SimpleDrone', 20, 20, 2, 1.2),
                                              ('DubinsCar', 256, 16, 2, 8.0), ('SimpleCar', 5, 0, 4, 100.0)])
def test_radius_graph_bit_exact(env, n, obs, B, area):
    sb = synth.make_states(env, n, obs, B, area, 77)
    ob = oracle_batch(sb)
    pd = O.ENV_PARAMS[env]['pos_dim']
    N = sb.nodes_per_graph
    ei, rowptr = ops.radius_graph(sb.states.to(DEV), pd, B, N, n, O.ENV_PARAMS[env]['comm_radius'],
                                  0 if env == 'SimpleCar' else 1)
    assert ei.dtype == torch.int64 and ei.shape == ob['edge_index'].shape, (ei.shape, ob['edge_index'].shape)
    assert torch.equal(ei.cpu(), ob['edge_index'])
    assert int(rowptr[-1]) == ei.shape[1]
    # CSR over all nodes agrees with a bincount of the targets
    rp = ops.rowptr_from_edge_index(ei, B * N).cpu()
    counts = torch.bincount(ob['edge_index'][1], minlength=B * N)
    assert torch.equal(rp[1:] - rp[:-1], counts.int())


@pytest.mark.parametrize('metric', [0, 1])
def test_radius_graph_boundary_ulps(metric):
    """Pairs placed within a few ulps of the radius: the compare must round exactly like the CPU reference
    (metric 0: unfused dx*dx+dy*dy < r*r; metric 1: sqrt(fma chain) < r)."""
    g = _g(5)
    n = 64
    base = torch.rand(n // 2, 2, generator=g) * 50 + torch.arange(n // 2).unsqueeze(1) * 10.0   # far apart pairs
    ang = torch.rand(n // 2, generator=g) * 2 * math.pi
    r = 1.0
    delta = (torch.randint(-3, 4, (n // 2,), generator=g).float()) * 6e-8
    other = base + torch.stack([torch.cos(ang), torch.sin(ang)], 1) * (r + delta).unsqueeze(1)
    pos = torch.cat([base, other], 0)
    env = 'SimpleCar' if metric == 0 else 'DubinsCar'
    states = torch.cat([pos, torch.zeros(n, 2)], 1)
    want = O.radius_graph(env, pos, n)
    got, _ = ops.radius_graph(states.to(DEV), 2, 1, n, n, r, metric)
    assert torch.equal(got.cpu(), want), (got.shape, want.shape)
    assert 0 < want.shape[1] < n   # the construction really straddles the boundary


def test_rowptr_rejects_unsorted():
    ei = torch.tensor([[0, 1, 2], [2, 0, 1]], device=DEV)
    with pytest.raises(ValueError):
        ops.rowptr_from_edge_index(ei, 3)


# ------------------------------------------------------------------------------------------------------
# K2 edge features
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('env', ['SimpleCar', 'DubinsCar', 'SimpleDrone'])
def test_edge_attr_fwd_bwd(env):
    sb = synth.make_states(env, 24, 6, 2, 2.0, 3)
    ob = oracle_batch(sb)
    ei = ob['edge_index']
    st = sb.states.clone().requires_grad_(True)
    want = O.edge_attr(env, st, ei)
    w = torch.randn(want.shape, generator=_g(1))
    (want * w).sum().backward()
    st_d = sb.states.to(DEV).requires_grad_(True)
    got = ops.EdgeAttrFunction.apply(st_d, ei.to(DEV), ops.ENV_IDS[env])
    (got * w.to(DEV)).sum().backward()
    assert torch.allclose(got.detach().cpu(), want.detach(), rtol=0, atol=2e-6)      # sin/cos ulps (Dubins)
    assert torch.allclose(st_d.grad.cpu(), st.grad, rtol=1e-5, atol=1e-5)


# ------------------------------------------------------------------------------------------------------
# K3 linear layers (fp32 SIMT path), odd shapes included
# ------------------------------------------------------------------------------------------------------
SHAPES = [(1, 1, 1), (7, 5, 3), (130, 2048, 13), (300, 256, 2048), (257, 1, 128), (64, 128, 256), (513, 130, 260),
          (1000, 32, 1026), (129, 2048, 2048)]


@pytest.mark.parametrize('M,N,K', SHAPES)
@pytest.mark.parametrize('act', [ops.ACT_NONE, ops.ACT_RELU, ops.ACT_TANH])
def test_linear_fwd(M, N, K, act):
    g = _g(M * 7 + N)
    x, W, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    inv_sigma = torch.tensor([0.7])
    want = (x.double() @ W.double().t()) * 0.7 + b.double()
    want = torch.relu(want) if act == ops.ACT_RELU else (torch.tanh(want) if act == ops.ACT_TANH else want)
    old = ops.GEMM_IMPL
    ops.GEMM_IMPL = 1
    try:
        got = ops.linear_fwd(x.to(DEV), W.to(DEV), b.to(DEV), inv_sigma.to(DEV), act)
    finally:
        ops.GEMM_IMPL = old
    err = (got.cpu().double() - want).abs().max().item()
    assert err < 2e-5 * max(1.0, want.abs().max().item()), err


@pytest.mark.parametrize('M,N,K', SHAPES)
def test_linear_bwd(M, N, K):
    g = _g(M + N * 3 + K)
    x, W = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K)
    dz = torch.randn(M, N, generator=g)
    relu_src = torch.randn(M, K, generator=g)
    old = ops.GEMM_IMPL
    ops.GEMM_IMPL = 1
    try:
        dx = ops.linear_bwd_data(dz.to(DEV), W.to(DEV), None, relu_src.to(DEV))
        dx_acc = torch.ones(M, K, device=DEV)
        ops.linear_bwd_data(dz.to(DEV), W.to(DEV), None, None, out=dx_acc, accumulate=True)
        dW, db = ops.linear_bwd_weight(dz.to(DEV), x.to(DEV), None)
    finally:
        ops.GEMM_IMPL = old
    want_dx = (dz.double() @ W.double())
    assert (dx.cpu().double() - want_dx * (relu_src > 0)).abs().max() < 2e-5 * max(1.0, want_dx.abs().max().item())
    assert (dx_acc.cpu().double() - (want_dx + 1)).abs().max() < 2e-5 * max(1.0, want_dx.abs().max().item())
    want_dW = dz.double().t() @ x.double()
    assert (dW.cpu().double() - want_dW).abs().max() < 3e-5 * max(1.0, want_dW.abs().max().item())
    assert (db.cpu().double() - dz.double().sum(0)).abs().max() < 3e-5 * max(1.0, dz.double().sum(0).abs().max().item())


TC_SHAPES = [(256, 256, 96), (384, 128, 96), (1000, 2048, 2048), (2500, 256, 2048), (777, 2048, 260), (4096, 512, 1024),
             (300, 130, 100), (70000, 128, 256)]


@pytest.mark.parametrize('M,N,K', TC_SHAPES)
def test_linear_tcgen05_3xfp16(M, N, K):
    """wgmma path (forced) against fp64: forward with fused bias+ReLU, data grad with ReLU mask and accumulate, weight
    grad + bias grad (fused into the split of dZ).  Tolerance 1e-5 of the output scale: the [hi|lo] fp16 companions carry
    22 significand bits and K is accumulated in 256-wide chunks promoted to fp32 registers (measured 1-2e-6)."""
    if not _C.lib().gcbf_has_wgmma():
        pytest.skip('library built without the wgmma path')
    g = _g(M + N + K)
    x, W, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    dz, rs = torch.randn(M, N, generator=g), torch.randn(M, K, generator=g)
    xd, Wd, bd, dzd, rsd = x.to(DEV), W.to(DEV), b.to(DEV), dz.to(DEV), rs.to(DEV)
    alpha = torch.tensor([1.3], device=DEV)
    old = ops.GEMM_IMPL
    ops.GEMM_IMPL = 2
    try:
        assert ops.use_h(M, N, K)
        y = ops.linear_fwd(xd, Wd, bd, alpha, ops.ACT_RELU)
        dx = ops.linear_bwd_data(dzd, Wd, alpha, rsd)
        dx_acc = torch.ones(M, K, device=DEV)
        ops.linear_bwd_data(dzd, Wd, None, None, out=dx_acc, accumulate=True)
        dW, db = ops.linear_bwd_weight(dzd, xd, alpha)
    finally:
        ops.GEMM_IMPL = old
    x64, W64, dz64 = xd.double(), Wd.double(), dzd.double()
    e = lambda a, r: ((a.double() - r).abs().max() / r.abs().max()).item()
    assert e(y, torch.relu(1.3 * (x64 @ W64.t()) + bd.double())) < 1e-5
    assert e(dx, 1.3 * (dz64 @ W64) * (rsd > 0)) < 1e-5
    assert e(dx_acc, dz64 @ W64 + 1) < 1e-5
    assert e(dW, 1.3 * (dz64.t() @ x64)) < 1e-5
    assert e(db, dz64.sum(0)) < 1e-5


def _split_reference(x: torch.Tensor):
    """(amax_bits, hi, lo, s) from the CPU model of the companion format (oracle/fp16x3_model.py)."""
    import fp16x3_model as F16
    hi, lo, s = F16.split(x)
    return x.abs().max().view(torch.int32).item(), hi, lo, s


@pytest.mark.parametrize('rows,cols,scale', [(300, 260, 1.0), (1000, 2048, 3e-7), (257, 129, 1e4), (64, 8, 1.0), (5, 1027, 2.5e-3)])
def test_amax_and_fp16_split_bit_exact(rows, cols, scale):
    """The fp16 [hi | lo] companion is integer-like work: bit-exact against the restatement, including odd column
    counts (scalar tail), a padded pitch, fused column sums, and the 22-bit reconstruction bound."""
    x = (torch.randn(rows, cols, generator=_g(rows + cols)) * scale)
    x[0, 0] = 0.0
    bits, hi, lo, s = _split_reference(x)
    xd = x.to(DEV)
    colsum = torch.empty(cols, device=DEV)
    h = ops.split_h(xd, colsum=colsum)
    assert h.amax.item() == bits
    assert h.ld % 8 == 0 and h.buf.shape == (2, rows, h.ld)
    assert torch.equal(h.buf[0, :, :cols].cpu(), hi)
    assert torch.equal(h.buf[1, :, :cols].cpu(), lo)
    rec = (h.buf[0, :, :cols].double() + h.buf[1, :, :cols].double()).cpu() / s
    assert ((rec - x.double()).abs() <= x.abs().double() * 2.0 ** -21 + x.abs().max().item() * 2.0 ** -39).all()
    assert torch.allclose(colsum.cpu().double(), x.double().sum(0), rtol=0, atol=1e-5 * scale * math.sqrt(rows) + 1e-30)
    # a strided view (leading dimension > cols) gives the same companion
    big = torch.zeros(rows, cols + 5, device=DEV)
    big[:, :cols] = xd
    h2 = ops.split_h(big[:, :cols])
    assert h2.amax.item() == bits and torch.equal(h2.buf[:, :, :cols], h.buf[:, :, :cols])


@pytest.mark.parametrize('M,N,K', [(5000, 2048, 13), (129, 256, 12), (24196, 2048, 14), (1000, 70, 16), (64, 64, 1)])
def test_linear_skinny_k(M, N, K):
    """In-features <= 16 (first phi layer): dedicated HBM-streaming kernels, exact fp32 FFMA."""
    g = _g(M + N + K)
    x, W, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g), torch.randn(N, generator=g)
    dz, rs = torch.randn(M, N, generator=g), torch.randn(M, K, generator=g)
    xd, Wd, bd, dzd, rsd = x.to(DEV), W.to(DEV), b.to(DEV), dz.to(DEV), rs.to(DEV)
    alpha = torch.tensor([0.9], device=DEV)
    assert ops.GEMM_IMPL == 0
    am = torch.zeros(1, device=DEV, dtype=torch.int32)
    y = ops.linear_fwd(xd, Wd, bd, alpha, ops.ACT_RELU, out_amax=am)
    assert _C.lib().gcbf_last_gemm_impl() == (3 if N >= 64 and M >= 64 else (4 if N <= 32 and K <= 256 else 1))
    assert am.view(torch.float32).item() == y.abs().max().item()
    dx = ops.linear_bwd_data(dzd, Wd, alpha, rsd)
    dx_acc = torch.ones(M, K, device=DEV)
    ops.linear_bwd_data(dzd, Wd, None, None, out=dx_acc, accumulate=True)
    dW, db = ops.linear_bwd_weight(dzd, xd, alpha)
    x64, W64, dz64 = xd.double(), Wd.double(), dzd.double()
    e = lambda a, r: ((a.double() - r).abs().max() / r.abs().max()).item()
    assert e(y, torch.relu(0.9 * (x64 @ W64.t()) + bd.double())) < 2e-6
    assert e(dx, 0.9 * (dz64 @ W64) * (rsd > 0)) < 1e-5
    assert e(dx_acc, dz64 @ W64 + 1) < 1e-5
    assert e(dW, 0.9 * (dz64.t() @ x64)) < 1e-5
    assert e(db, dz64.sum(0)) < 1e-5


@pytest.mark.parametrize('M,N,K', [(24196, 1, 128), (8192, 32, 128), (8192, 1, 32), (8192, 2, 32), (777, 7, 200), (50, 32, 256), (3, 5, 17)])
def test_linear_tiny_n(M, N, K):
    """Out-features <= 32 (gate / head tails): row-streaming fwd and dgrad kernels, narrow column sums; exact fp32 FFMA."""
    g = _g(M + N + K)
    x, W, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    dz, rs = torch.randn(M, N, generator=g), torch.randn(M, K, generator=g)
    xd, Wd, bd, dzd, rsd = x.to(DEV), W.to(DEV), b.to(DEV), dz.to(DEV), rs.to(DEV)
    alpha = torch.tensor([1.1], device=DEV)
    assert ops.GEMM_IMPL == 0 and not ops.use_h(M, N, K)
    am = torch.zeros(1, device=DEV, dtype=torch.int32)
    y = ops.linear_fwd(xd, Wd, bd, alpha, ops.ACT_TANH, out_amax=am)
    assert _C.lib().gcbf_last_gemm_impl() == 4
    dx = ops.linear_bwd_data(dzd, Wd, alpha, rsd)
    assert _C.lib().gcbf_last_gemm_impl() == 4
    dx_acc = torch.ones(M, K, device=DEV)
    ops.linear_bwd_data(dzd, Wd, None, None, out=dx_acc, accumulate=True)
    dW, db = ops.linear_bwd_weight(dzd, xd, alpha)
    x64, W64, dz64 = xd.double(), Wd.double(), dzd.double()
    e = lambda a, r: ((a.double() - r).abs().max() / r.abs().max()).item()
    assert e(y, torch.tanh(1.1 * (x64 @ W64.t()) + bd.double())) < 2e-6
    assert am.view(torch.float32).item() == y.abs().max().item()
    assert e(dx, 1.1 * (dz64 @ W64) * (rsd > 0)) < 2e-6
    assert e(dx_acc, dz64 @ W64 + 1) < 2e-6
    assert e(dW, 1.1 * (dz64.t() @ x64)) < 1e-5
    assert e(db, dz64.sum(0)) < 1e-5


def test_sn_power_iter_batched_bit_identical():
    """The batched power iteration (all layers of a net in four launches) must reproduce the per-layer kernels bit for bit."""
    shapes = [(2048, 13), (2048, 2048), (256, 2048), (128, 256), (1, 128), (512, 1026), (32, 128)]
    g = _g(5)
    specs_a, specs_b = [], []
    for N, K in shapes:
        W = (torch.randn(N, K, generator=g) / math.sqrt(K)).to(DEV)
        u = torch.nn.functional.normalize(torch.randn(N, generator=g), dim=0).to(DEV)
        v = torch.nn.functional.normalize(torch.randn(K, generator=g), dim=0).to(DEV)
        specs_a.append(ops.LinearSpec(W, torch.zeros(N, device=DEV), u.clone(), v.clone()))
        specs_b.append(ops.LinearSpec(W, torch.zeros(N, device=DEV), u.clone(), v.clone()))
    specs_b.insert(2, ops.LinearSpec(torch.randn(4, 4, device=DEV), torch.zeros(4, device=DEV)))   # a layer without spectral norm
    for _ in range(2):
        want = [ops.sn_power_iter(L.W, L.u, L.v) for L in specs_a]
        got, _ = ops.sn_power_iter_batched(specs_b)
        assert got[2] is None
        got = [x for x in got if x is not None]
        for La, Lb, a, b in zip(specs_a, [L for L in specs_b if L.sn], want, got):
            assert torch.equal(La.u, Lb.u) and torch.equal(La.v, Lb.v) and torch.equal(a, b)


def test_batched_weight_companions_bit_identical():
    """ops.prepare_weights (all stale weight companions of a net in two launches) against the per-matrix amax + split."""
    shapes = [(2048, 2048), (256, 2048), (128, 256), (2048, 260), (512, 1027), (1024, 2048), (128, 128)]
    g = _g(11)
    specs = [ops.LinearSpec((torch.randn(N, K, generator=g) * 10 ** float(torch.randint(-6, 3, (1,), generator=g))).to(DEV),
                            torch.zeros(N, device=DEV)) for N, K in shapes]
    specs.append(ops.LinearSpec(torch.randn(16, 2048, device=DEV), torch.zeros(16, device=DEV)))      # N < 96: not a tensor-core layer
    ops.prepare_weights([(L, 4096) for L in specs])
    assert getattr(specs[-1].W, '_gcbf_h16', None) is None
    for L in specs[:-1]:
        got = L.W._gcbf_h16[1]
        want = ops.split_h(L.W)
        assert got.amax.item() == want.amax.item() and got.ld == want.ld
        assert torch.equal(got.buf[:, :, :got.cols], want.buf[:, :, :want.cols])
        assert ops.weight_h(L.W) is got                      # the cache entry is current: no second split
    specs[0].W.mul_(2.0)                                      # an in-place update invalidates exactly that entry
    ops.prepare_weights([(L, 4096) for L in specs])
    assert torch.equal(specs[0].W._gcbf_h16[1].buf, ops.split_h(specs[0].W).buf)


def test_linear_strided_views():
    """Kernels take leading dimensions: column slices of wider buffers must work without copies."""
    g = _g(9)
    big = torch.randn(50, 300, generator=g).to(DEV)
    W = torch.randn(40, 260, generator=g).to(DEV)
    out = torch.zeros(50, 64, device=DEV)
    ops.linear_fwd(big[:, :260], W, None, None, ops.ACT_NONE, out=out[:, 8:48])
    want = big[:, :260].cpu().double() @ W.cpu().double().t()
    assert (out[:, 8:48].cpu().double() - want).abs().max() < 1e-4
    assert out[:, :8].abs().max() == 0 and out[:, 48:].abs().max() == 0


# ------------------------------------------------------------------------------------------------------
# K4 attention aggregation
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('deg_hi', [4, 90])
def test_attention_aggregation_fwd_bwd(deg_hi):
    g = _g(deg_hi)
    N, C = 37, 256
    deg = torch.randint(0, deg_hi + 1, (N,), generator=g)
    deg[3] = 0
    dst = torch.repeat_interleave(torch.arange(N), deg)
    E = int(dst.numel())
    msg = torch.randn(E, C, generator=g, requires_grad=True)
    gate = (torch.randn(E, 1, generator=g) * 3).requires_grad_(True)
    att = O.segment_softmax(gate, dst, N)
    want = torch.zeros(N, C).index_add(0, dst, att * msg)
    w = torch.randn(N, C, generator=g)
    (want * w).sum().backward()
    rowptr = torch.zeros(N + 1, dtype=torch.int32)
    rowptr[1:] = deg.cumsum(0).int()
    msg_d, gate_d, rowptr_d = msg.detach().to(DEV), gate.detach().to(DEV), rowptr.to(DEV)
    out = torch.full((N, C + 4), 7.0, device=DEV)
    att_d = torch.empty(E, device=DEV)
    _C.call('gcbf_attn_aggr_fwd', _C.ptr(msg_d), C, _C.ptr(gate_d), _C.ptr(rowptr_d), N, C, _C.ptr(att_d), _C.ptr(out), C + 4)
    assert torch.allclose(out[:, :C].cpu(), want.detach(), rtol=1e-5, atol=1e-5)
    assert (out[:, C:] == 7.0).all()
    assert torch.allclose(att_d.cpu(), att.detach().reshape(-1), rtol=1e-5, atol=1e-6)
    d_msg = torch.empty(E, C, device=DEV)
    d_gate = torch.empty(E, device=DEV)
    d_aggr = torch.zeros(N, C + 4, device=DEV)
    d_aggr[:, :C] = w.to(DEV)
    _C.call('gcbf_attn_aggr_bwd', _C.ptr(msg_d), C, _C.ptr(att_d), _C.ptr(rowptr_d), N, C, _C.ptr(d_aggr), C + 4,
            _C.ptr(d_msg), C, _C.ptr(d_gate), 0)
    assert torch.allclose(d_msg.cpu(), msg.grad, rtol=1e-4, atol=1e-5)
    assert torch.allclose(d_gate.cpu(), gate.grad.reshape(-1), rtol=1e-3, atol=2e-5)


# ------------------------------------------------------------------------------------------------------
# K5 / K6 environment kernels
# ------------------------------------------------------------------------------------------------------
ENV_CASES = [('SimpleCar', 24, 0, 3, 1.5), ('DubinsCar', 24, 6, 3, 1.5), ('SimpleDrone', 12, 12, 2, 0.8),
             ('DubinsCar', 24, 6, 1, 1.5), ('SimpleDrone', 12, 12, 1, 0.8)]


def _env_setup(env_name, n, obs, B, area, seed=21):
    sb = synth.make_states(env_name, n, obs, B, area, seed)
    if env_name == 'SimpleCar':
        sb.states[:, 2:] *= 3          # some over-speed agents -> penalty branch of u_ref
    if env_name == 'SimpleDrone':
        sb.states[:n, 3:] *= 3
    if env_name == 'DubinsCar':
        sb.states[:n // 2, 3] += 0.5   # some v > speed_limit
    if B == 1 and env_name != 'SimpleCar':
        sb.states[1, :O.ENV_PARAMS[env_name]['pos_dim']] = sb.goals[1, :O.ENV_PARAMS[env_name]['pos_dim']]   # reached
    env, algo = seeded_algo(env_name, n, DEV, 0, {'num_obs': sb.num_obs, 'area_size': area})
    data = product_batch(env, sb, DEV)
    return sb, env, algo, data, oracle_batch(sb)


@pytest.mark.parametrize('env_name,n,obs,B,area', ENV_CASES)
def test_u_ref_step_masks(env_name, n, obs, B, area):
    sb, env, _, data, ob = _env_setup(env_name, n, obs, B, area)
    assert torch.equal(data.edge_index.cpu(), ob['edge_index'])
    assert torch.allclose(data.u_ref.cpu(), ob['u_ref'], rtol=1e-5, atol=2e-6), (data.u_ref.cpu() - ob['u_ref']).abs().max()
    N = sb.nodes_per_graph
    sm = O.safe_mask(env_name, sb.states, B, N, n)
    um = O.unsafe_mask(env_name, sb.states, B, N, n)
    assert torch.equal(env.safe_mask(data).cpu(), sm)
    assert torch.equal(env.unsafe_mask(data).cpu(), um)
    assert um.any() and sm.any() and not (um & sm).any()
    # finite-difference step + VJP to the action
    a_dim = O.ENV_PARAMS[env_name]['action_dim']
    act = (torch.randn(B * n, a_dim, generator=_g(4)) * (4.0 if env_name != 'DubinsCar' else 1.5)).requires_grad_(True)
    want = O.forward_states(env_name, sb.states, ob['agent_mask'], act, sb.goals, ob['K'], N)
    w = torch.randn(want.shape, generator=_g(6))
    (want * w).sum().backward()
    act_d = act.detach().to(DEV).requires_grad_(True)
    got = env.next_states(data, act_d)
    (got * w.to(DEV)).sum().backward()
    assert torch.allclose(got.detach().cpu(), want.detach(), rtol=0, atol=2e-6), (got.detach().cpu() - want.detach()).abs().max()
    assert torch.allclose(act_d.grad.cpu(), act.grad, rtol=1e-5, atol=1e-7)
    if B == 1 and env_name != 'SimpleCar':
        assert torch.equal(got.detach().cpu()[1], sb.states[1]) and act.grad[1].abs().sum() == 0   # frozen agent


def test_loss_kernels_match_reference_formulas():
    g = _g(8)
    M, a = 301, 2
    h = torch.randn(M, 1, generator=g) * 0.05
    hn = h + torch.randn(M, 1, generator=g) * 0.002
    hnn = hn + torch.randn(M, 1, generator=g) * 0.001
    act = torch.randn(M, a, generator=g)
    safe = torch.rand(M, generator=g) < 0.4
    unsafe = (torch.rand(M, generator=g) < 0.2) & ~safe
    alpha, eps, dt = 1.0, 0.02, 0.03
    cu, cs, ch, ca = 1.0, 1.0, 0.5, 0.05
    hr, hnr, ar = h.clone().requires_grad_(True), hn.clone().requires_grad_(True), act.clone().requires_grad_(True)
    lu = torch.relu(hr[unsafe] + eps).mean()
    ls = torch.relu(-hr[safe] + eps).mean()
    hd = (hnr.reshape(-1) - hr.reshape(-1)) / dt
    hdn = (hnn.reshape(-1) - hr.reshape(-1)) / dt
    hd = (hdn - hd).clone().detach() + hd
    lh = torch.relu(-hd - alpha * hr.reshape(-1) + eps).mean()
    la = torch.square(ar).sum(dim=1).mean()
    (cu * lu + cs * ls + ch * lh + ca * la).backward()
    acc = O.acc_h_dot_broadcast(hd.detach(), h, alpha)
    hD, hnD, hnnD, actD = h.to(DEV).contiguous(), hn.to(DEV).contiguous(), hnn.to(DEV).contiguous(), act.to(DEV).contiguous()
    partial = torch.empty(16, device=DEV, dtype=torch.float64)
    hdot = torch.empty(M, device=DEV)
    su8, uu8 = safe.to(torch.uint8).to(DEV), unsafe.to(torch.uint8).to(DEV)
    _C.call('gcbf_loss_partials', _C.ptr(hD), _C.ptr(hnD), _C.ptr(hnnD), _C.ptr(actD), a, _C.ptr(su8), _C.ptr(uu8), M,
            alpha, eps, dt, _C.ptr(partial), _C.ptr(hdot))
    dh, dhn, da, sc = torch.empty(M, device=DEV), torch.empty(M, device=DEV), torch.empty(M, a, device=DEV), torch.empty(8, device=DEV)
    _C.call('gcbf_loss_grads', _C.ptr(hD), _C.ptr(hnD), _C.ptr(hnnD), _C.ptr(actD), a, _C.ptr(su8), _C.ptr(uu8), M,
            alpha, eps, dt, cu, cs, ch, ca, _C.ptr(partial), _C.ptr(dh), _C.ptr(dhn), _C.ptr(da), _C.ptr(sc))
    sc = sc.cpu()
    for got, want in zip(sc[:4].tolist(), [lu.item(), ls.item(), lh.item(), la.item()]):
        assert abs(got - want) < 1e-6, (got, want)
    assert abs(sc[4].item() - (h[unsafe] < 0).float().mean().item()) < 1e-6
    assert abs(sc[5].item() - (h[safe] >= 0).float().mean().item()) < 1e-6
    assert torch.equal(hdot.cpu(), hd.detach())
    assert torch.allclose(dh.cpu(), hr.grad.reshape(-1), rtol=1e-5, atol=1e-8)
    assert torch.allclose(dhn.cpu(), hnr.grad.reshape(-1), rtol=1e-5, atol=1e-8)
    assert torch.allclose(da.cpu(), ar.grad, rtol=1e-5, atol=1e-8)
    cnt = torch.empty(1, device=DEV, dtype=torch.int64)
    _C.call('gcbf_pair_count', _C.ptr(hdot), M, _C.ptr(hD), M, alpha, _C.ptr(cnt))
    assert abs(cnt.item() / (M * M) - acc.item()) < 1e-7
    # empty masks: loss 0, accuracy 1 (gcbf.py:175-177, 187-189)
    z = torch.zeros(M, dtype=torch.uint8, device=DEV)
    _C.call('gcbf_loss_partials', _C.ptr(hD), _C.ptr(hnD), _C.ptr(hnnD), _C.ptr(actD), a, _C.ptr(z), _C.ptr(z), M,
            alpha, eps, dt, _C.ptr(partial), None)
    sc2 = torch.empty(8, device=DEV)
    _C.call('gcbf_loss_grads', _C.ptr(hD), _C.ptr(hnD), _C.ptr(hnnD), _C.ptr(actD), a, _C.ptr(z), _C.ptr(z), M,
            alpha, eps, dt, cu, cs, ch, ca, _C.ptr(partial), _C.ptr(dh), _C.ptr(dhn), _C.ptr(da), _C.ptr(sc2))
    assert sc2[0].item() == 0 and sc2[1].item() == 0 and sc2[4].item() == 1 and sc2[5].item() == 1


# ------------------------------------------------------------------------------------------------------
# K7 spectral norm, K8 clip + Adam
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('N,K', [(2048, 13), (256, 2048), (2048, 260), (1024, 2048)])
def test_spectral_norm_power_iteration_and_grad(N, K):
    g = _g(N + K)
    W = torch.randn(N, K, generator=g) / math.sqrt(K)
    u0 = torch.nn.functional.normalize(torch.randn(N, generator=g), dim=0)
    v0 = torch.nn.functional.normalize(torch.randn(K, generator=g), dim=0)
    sd = {'l.weight_orig': W.clone().requires_grad_(True), 'l.weight_u': u0.clone(), 'l.weight_v': v0.clone()}
    W_eff = O._sn_weight(sd, 'l')
    G = torch.randn(N, K, generator=g)
    (W_eff * G).sum().backward()
    Wd, ud, vd = W.to(DEV), u0.to(DEV), v0.to(DEV)
    inv_sigma = ops.sn_power_iter(Wd, ud, vd)
    assert torch.allclose(ud.cpu(), sd['l.weight_u'], rtol=1e-4, atol=1e-6)
    assert torch.allclose(vd.cpu(), sd['l.weight_v'], rtol=1e-4, atol=1e-6)
    sigma_ref = (W / W_eff.detach())[0, 0].item()
    assert abs(1.0 / inv_sigma.item() - sigma_ref) < 1e-5 * sigma_ref
    dW = (G.to(DEV) * inv_sigma).contiguous()            # what bwd_weight delivers: dL/dW_eff / sigma
    ops.sn_grad_fixup(dW, Wd, ud, vd, inv_sigma)
    assert torch.allclose(dW.cpu(), sd['l.weight_orig'].grad, rtol=1e-3, atol=1e-5 * G.abs().max().item())


def test_clip_adam_matches_torch():
    g = _g(2)
    n = 100003
    p0 = torch.randn(n, generator=g)
    ref_p = torch.nn.Parameter(p0.clone())
    opt = torch.optim.Adam([ref_p], lr=3e-4)
    p = p0.clone().to(DEV)
    m, v = torch.zeros(n, device=DEV), torch.zeros(n, device=DEV)
    sumsq = torch.zeros(1, device=DEV, dtype=torch.float64)
    for step in range(1, 4):
        grad = torch.randn(n, generator=g) * (1e-2 if step != 2 else 1e-7)    # step 2: below the clip threshold
        ref_p.grad = grad.clone()
        torch.nn.utils.clip_grad_norm_([ref_p], 1e-3)
        opt.step()
        gd = grad.to(DEV)
        sumsq.zero_()
        _C.call('gcbf_grad_sumsq', _C.ptr(gd), n, _C.ptr(sumsq))
        assert abs(math.sqrt(sumsq.item()) - grad.double().norm().item()) < 1e-9 + 1e-7 * grad.norm().item()
        _C.call('gcbf_clip_adam', _C.ptr(p), _C.ptr(gd), _C.ptr(m), _C.ptr(v), n, _C.ptr(sumsq), 1e-3, 3e-4, 0.9, 0.999, 1e-8, step)
        assert torch.allclose(p.cpu(), ref_p.detach(), rtol=0, atol=2e-7), (step, (p.cpu() - ref_p.detach()).abs().max())


# ------------------------------------------------------------------------------------------------------
# modules: MLP and GNN layer, forward + backward against the oracle under autograd
# ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('limit_lip', [False, True])
def test_mlp_module_forward_backward(limit_lip):
    from gcbf_b200.nn import MLP
    torch.manual_seed(3)
    mlp = MLP(13, 5, (64, 32), output_activation=torch.nn.Tanh(), limit_lip=limit_lip)
    sd = {'m.' + k: v.clone() for k, v in mlp.state_dict().items()}
    for k in sd:
        if k.endswith(('weight', 'bias', 'weight_orig')):
            sd[k].requires_grad_(True)
    x = torch.randn(50, 13, generator=_g(1))
    want = O.mlp_forward(sd, 'm', x, 3, limit_lip, 'tanh')
    w = torch.randn(want.shape, generator=_g(2))
    (want * w).sum().backward()
    mlp = mlp.to(DEV)
    xd = x.to(DEV).requires_grad_(True)
    got = mlp(xd)
    (got * w.to(DEV)).sum().backward()
    assert torch.allclose(got.detach().cpu(), want.detach(), rtol=0, atol=1e-6)
    for name, p in mlp.named_parameters():
        ref = sd['m.' + name].grad
        assert torch.allclose(p.grad.cpu(), ref, rtol=1e-3, atol=1e-6), (name, (p.grad.cpu() - ref).abs().max())
    if limit_lip:   # buffers advanced by exactly one power iteration
        assert torch.allclose(mlp.net[0].weight_u.cpu(), sd['m.net.0.weight_u'], rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize('env_name,n,obs,B,area', ENV_CASES[:3])
def test_cbf_and_actor_forward_backward(env_name, n, obs, B, area):
    sb, env, algo, data, ob = _env_setup(env_name, n, obs, B, area, seed=31)
    cbf_sd = {k: v.detach().cpu().clone() for k, v in algo.cbf.state_dict().items()}
    act_sd = {k: v.detach().cpu().clone() for k, v in algo.actor.state_dict().items()}
    for sdd in (cbf_sd, act_sd):
        for k in O.trainable_keys(sdd):
            sdd[k].requires_grad_(True)
    ea = O.edge_attr(env_name, sb.states, ob['edge_index']).requires_grad_(True)
    h = O.cbf_forward(cbf_sd, ob['x'], ea, ob['edge_index'], ob['agent_mask'])
    u = O.actor_forward(act_sd, ob['x'], ea, ob['edge_index'], ob['agent_mask'], ob['u_ref'])
    wh, wu = torch.randn(h.shape, generator=_g(1)), torch.randn(u.shape, generator=_g(2))
    ((h * wh).sum() + (u * wu).sum()).backward()
    data.edge_attr = data.edge_attr.detach().requires_grad_(True)
    hg, ug = algo.cbf(data), algo.actor(data)
    ((hg * wh.to(DEV)).sum() + (ug * wu.to(DEV)).sum()).backward()
    assert torch.allclose(hg.detach().cpu(), h.detach(), rtol=0, atol=1e-5), (hg.detach().cpu() - h.detach()).abs().max()
    assert torch.allclose(ug.detach().cpu(), u.detach(), rtol=0, atol=1e-5), (ug.detach().cpu() - u.detach()).abs().max()
    # gradients: relative to each net's gradient norm.  A single ReLU decision flipped by rounding costs ~0.3 % of a
    # layer's gradient (1/sqrt(#hidden units)); exactness given identical masks is asserted in the next test.
    rel = lambda a, b: ((a.double() - b.double()).norm() / b.double().norm()).item()
    assert rel(data.edge_attr.grad.cpu(), ea.grad) < 2e-2
    for mod, sdd in ((algo.cbf, cbf_sd), (algo.actor, act_sd)):
        tot = torch.sqrt(sum((sdd[name].grad.double() ** 2).sum() for name, _ in mod.named_parameters()))
        for name, p in mod.named_parameters():
            err = (p.grad.cpu().double() - sdd[name].grad.double()).norm() / tot
            assert err < 1e-2, (name, err.item())


@pytest.mark.parametrize('impl,tol', [(1, 2e-5), (0, 3e-4)])
def test_net_backward_exact_given_same_relu_masks(impl, tol):
    """impl 1 = fp32 SIMT GEMMs (exact to fp32 round-off), impl 0 = wgmma 3xFP16 where the shape qualifies (22-bit
    operands; measured 1-2e-6 per GEMM, the tolerance below is the one the 3xTF32 predecessor needed).
    The whole fused backward (head -> gamma -> row scatter -> attention aggregation -> gate -> phi -> edge_attr,
    incl. the spectral-norm sigma term) against torch autograd in fp64 ON THE SAME ReLU MASKS (taken from the
    kernels' saved activations), so rounding-level mask flips cannot blur the comparison: tolerance 1e-5 relative."""
    from gcbf_b200.data import agent_row_index
    from gcbf_b200.nn.gnn import cached_rowptr
    sb, env, algo, data, ob = _env_setup('DubinsCar', 24 if impl == 1 else 96, 6, 3, 1.5 if impl == 1 else 3.0, seed=51)
    old_impl, ops.GEMM_IMPL = ops.GEMM_IMPL, impl
    try:
        _net_backward_check(algo, data, tol)
    finally:
        ops.GEMM_IMPL = old_impl


def _net_backward_check(algo, data, tol):
    from gcbf_b200.data import agent_row_index
    from gcbf_b200.nn.gnn import cached_rowptr
    layer = algo.cbf.feat_transformer.module_0
    spec = layer.net_spec(algo.cbf.feat_2_CBF)
    rowptr = cached_rowptr(data.edge_index, data.x.shape[0])
    ridx = agent_row_index(data)
    ea_in = data.edge_attr.detach()
    out, ctx = ops.net_forward(spec, data.x, ea_in, data.edge_index, rowptr, ridx, None, True)
    c_phi, c_gate, c_gamma, c_head, msg, att, Nn, E = ctx
    d_out = torch.randn(out.shape, generator=_g(3)).to(DEV)
    d_ea, grads = ops.net_backward(spec, ctx, d_out, rowptr, ridx, True)

    dd = lambda t: t.detach().double()
    leaves = []

    def chain(x, layers, mctx):
        for i, L in enumerate(layers):
            W = dd(L.W).requires_grad_(True)
            b = dd(L.b).requires_grad_(True)
            leaves.append((W, b))
            Weff = W
            if L.sn:
                u, v = mctx.uv[i]
                Weff = W / torch.dot(dd(u), W @ dd(v))
            x = torch.nn.functional.linear(x, Weff, b)
            if L.act == ops.ACT_RELU:
                x = x * (mctx.acts[i + 1] > 0).double()       # the kernels' own mask
            elif L.act == ops.ACT_TANH:
                x = torch.tanh(x)
        return x
    ea64 = dd(ea_in).requires_grad_(True)
    ei = data.edge_index
    x64 = dd(data.x)
    m = chain(torch.cat([x64[ei[1]], x64[ei[0]], ea64], 1), spec.phi, c_phi)
    gate = chain(m, spec.gate, c_gate)
    gmax = torch.full((Nn, 1), float('-inf'), dtype=torch.float64, device=DEV).scatter_reduce(
        0, ei[1].view(-1, 1), gate.detach(), reduce='amax', include_self=True)
    ex = (gate - gmax[ei[1]]).exp()
    den = torch.zeros(Nn, 1, dtype=torch.float64, device=DEV).index_add(0, ei[1], ex) + 1e-16
    aggr = torch.zeros(Nn, 256, dtype=torch.float64, device=DEV).index_add(0, ei[1], ex / den[ei[1]] * m)
    feat = chain(torch.cat([aggr, x64], 1)[ridx], spec.gamma, c_gamma)
    h = chain(feat, spec.head, c_head)
    assert rel_err(out, h) < tol
    (h * d_out.double()).sum().backward()
    assert rel_err(d_ea, ea64.grad) < tol, rel_err(d_ea, ea64.grad)
    names = ['phi'] * 3 + ['gate'] * 3 + ['gamma'] * 3 + ['head'] * 4
    for i, ((dW, db), (W, b)) in enumerate(zip(grads, leaves)):
        assert rel_err(dW, W.grad) < tol, (names[i], i, rel_err(dW, W.grad))
        # (the last gate bias has an exactly-zero gradient -- softmax is shift invariant -- so allow an fp32 noise floor)
        assert (db.double() - b.grad).norm() <= tol * b.grad.norm() + 1e-5 * dW.double().norm(), (names[i], i)


def rel_err(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-300)).item()


@pytest.mark.parametrize('M,N,K', [(16, 2048, 2048), (44, 2048, 260), (1, 512, 1024), (64, 128, 32), (45, 256, 2048), (16, 1024, 1027), (33, 70, 130),
                                   (64, 2048, 2048), (57, 1024, 520), (3, 256, 128), (44, 2052, 516)])
def test_linear_few_rows(M, N, K):
    """M <= 64 (rollout-time single-graph passes, config C1): weight-streaming kernels (gemm_fewrows.cu) instead of a 128 x 128 tile
    grid; exact fp32 FFMA, forward with fused bias / activation, data-grad with ReLU mask and accumulate, weight-grad + bias grad."""
    g = _g(M + 3 * N + K)
    x, W, b = torch.randn(M, K, generator=g), torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(N, generator=g)
    dz, rs = torch.randn(M, N, generator=g), torch.randn(M, K, generator=g)
    xd, Wd, bd, dzd, rsd = x.to(DEV), W.to(DEV), b.to(DEV), dz.to(DEV), rs.to(DEV)
    alpha = torch.tensor([1.2], device=DEV)
    assert ops.GEMM_IMPL == 0 and not ops.use_h(M, N, K)
    am = torch.zeros(1, device=DEV, dtype=torch.int32)
    y = ops.linear_fwd(xd, Wd, bd, alpha, ops.ACT_RELU, out_amax=am)
    assert _C.lib().gcbf_last_gemm_impl() == 5
    assert am.view(torch.float32).item() == y.abs().max().item()
    dx = ops.linear_bwd_data(dzd, Wd, alpha, rsd)
    assert _C.lib().gcbf_last_gemm_impl() == (5 if (K >= 64 and N >= 32) or (K <= 32 and N >= 64) else 1)      # (output width K, contraction N)
    dx_acc = torch.ones(M, K, device=DEV)
    ops.linear_bwd_data(dzd, Wd, None, None, out=dx_acc, accumulate=True)
    dW, db = ops.linear_bwd_weight(dzd, xd, alpha)
    assert _C.lib().gcbf_last_gemm_impl() == 5
    dW_acc = torch.ones(N, K, device=DEV)
    db_acc = torch.ones(N, device=DEV)
    ops.linear_bwd_weight(dzd, xd, None, out_w=dW_acc, out_b=db_acc)
    x64, W64, dz64 = xd.double(), Wd.double(), dzd.double()
    e = lambda a, r: ((a.double() - r).abs().max() / r.abs().max()).item()
    assert e(y, torch.relu(1.2 * (x64 @ W64.t()) + bd.double())) < 2e-6
    assert e(dx, 1.2 * (dz64 @ W64) * (rsd > 0)) < 2e-6
    assert e(dx_acc, dz64 @ W64 + 1) < 2e-6
    assert e(dW, 1.2 * (dz64.t() @ x64)) < 2e-6
    assert e(dW_acc, dz64.t() @ x64 + 1) < 2e-6
    assert e(db, dz64.sum(0)) < 1e-5 and e(db_acc, dz64.sum(0) + 1) < 1e-5


@pytest.mark.parametrize('M,N,K', [(44, 2048, 13), (16, 2048, 12), (64, 512, 32), (2, 64, 3)])
def test_linear_few_rows_narrow_input_grad(M, N, K):
    """d(input) of a layer with <= 32 inputs on <= 64 rows (d edge_attr of one small graph: the first phi layer in GCBF.apply): one block
    per row instead of the single-block tile kernel (213 us in the launch list of one apply round)."""
    g = _g(M + N + K)
    W, dz, rs = torch.randn(N, K, generator=g) / math.sqrt(K), torch.randn(M, N, generator=g), torch.randn(M, K, generator=g)
    Wd, dzd, rsd = W.to(DEV), dz.to(DEV), rs.to(DEV)
    alpha = torch.tensor([0.7], device=DEV)
    dx = ops.linear_bwd_data(dzd, Wd, alpha, rsd)
    assert _C.lib().gcbf_last_gemm_impl() == 5
    dx_acc = torch.ones(M, K, device=DEV)
    ops.linear_bwd_data(dzd, Wd, None, None, out=dx_acc, accumulate=True)
    want = dzd.double() @ Wd.double()
    e = lambda a, r: ((a.double() - r).abs().max() / r.abs().max()).item()
    assert e(dx, 0.7 * want * (rsd > 0)) < 2e-6
    assert e(dx_acc, want + 1) < 2e-6
