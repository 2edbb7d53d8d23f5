"""The opt-in fp16 tensor-core mode (GCBF.params['matmul'] = 'fp16') without a GPU: parameter parsing and refusals, the descriptor
field that carries the mode, and the rounding model whose bound tests/test_matmul_fp16_gpu.py asserts on the kernel."""
import ctypes
import math

import numpy as np
import pytest
import torch

import matmul_fp16_model as F1
from gcbf_b200 import native, ops
from gcbf_b200.synth import seeded_algo

CPU = torch.device('cpu')


def _algo(hp_extra=None, name='SimpleCar'):
    from gcbf_b200.trainer.utils import read_params
    hp = dict(read_params(name, 'gcbf'))
    if hp_extra:
        hp.update(hp_extra)
    return seeded_algo(name, 4, CPU, 0, {'area_size': 4.0}, hyperparams=hp)


# ---- parameter parsing and refusals -------------------------------------------------------------------------------------------
def test_default_is_fp32_and_puts_three_products_on_both_modules():
    env, algo = _algo()
    assert 'matmul' not in algo.params and algo._matmul_mode() == 'fp32'
    for m in (algo.cbf, algo.actor):
        assert m.feat_transformer.module_0.net_spec().tc_products == 3


def test_fp16_via_make_algo_hyperparams_reaches_the_net_descriptors():
    env, algo = _algo({'matmul': 'fp16'})
    for m, head in ((algo.cbf, algo.cbf.feat_2_CBF), (algo.actor, algo.actor.feat_2_action)):
        spec = m.feat_transformer.module_0.net_spec(head)
        assert spec.tc_products == 1
        assert native.make_net_desc(spec, 0, None).tc_products == 1
    algo.set_matmul('fp32')
    assert algo.cbf.feat_transformer.module_0.net_spec().tc_products == 3


@pytest.mark.parametrize('bad', ['bf16', 'FP16', 'tf32', 16, None])
def test_other_values_raise(bad):
    with pytest.raises(ValueError, match='matmul'):
        _algo({'matmul': bad})
    env, algo = _algo()
    with pytest.raises(ValueError, match='matmul'):
        algo.set_matmul(bad)
    assert algo._matmul_mode() == 'fp32'                # a refused switch leaves the mode as it was


def test_python_sequenced_paths_refuse_fp16():
    env, algo = _algo({'matmul': 'fp16'})
    data = None                                            # refused before the graph is looked at
    with pytest.raises(ValueError, match='h_dot_analytic'):
        algo.h_dot_analytic(data)
    with pytest.raises(ValueError, match='cbf_condition_field'):
        algo.cbf_condition_field(data)
    algo.params['h_dot'] = 'analytic'
    with pytest.raises(ValueError, match='analytic'):
        algo.train_step(data)
    # the per-kernel Python sequencing of a GNN pass
    spec = algo.cbf.feat_transformer.module_0.net_spec(algo.cbf.feat_2_CBF)
    with pytest.raises(ValueError, match='fp16'):
        ops.net_forward(spec, None, None, None, None, None, None, False)


def test_gcbf_native_0_refuses_fp16(monkeypatch):
    monkeypatch.setattr(ops, 'NATIVE', False)
    with pytest.raises(ValueError, match='GCBF_NATIVE'):
        _algo({'matmul': 'fp16'})
    env, algo = _algo()
    with pytest.raises(ValueError, match='GCBF_NATIVE'):
        algo.set_matmul('fp16')


def test_macbf_refuses_fp16():
    from gcbf_b200.algo import make_algo
    from gcbf_b200.env import make_env
    from gcbf_b200.trainer.utils import read_params
    env = make_env('DubinsCar', 8, CPU, max_neighbors=12)
    hp = dict(read_params('DubinsCar', 'macbf'), matmul='fp16')
    with pytest.raises(ValueError, match='MACBF'):
        make_algo('macbf', env, 8, env.node_dim, env.edge_dim, env.action_dim, CPU, 512, hp)
    hp['matmul'] = 'fp32'
    make_algo('macbf', env, 8, env.node_dim, env.edge_dim, env.action_dim, CPU, 512, hp)


# ---- the descriptor -----------------------------------------------------------------------------------------------------------
def test_tc_products_sits_where_pad_was():
    fields = [f[0] for f in native.NetDesc._fields_]
    assert fields[-1] == 'tc_products' and 'pad_' not in fields
    assert native.NetDesc.tc_products.offset == native.NetDesc.refresh_weights.offset + 4
    # size unchanged: 4 x 4 linear descriptors + 10 int32 (the last one was pad_)
    assert ctypes.sizeof(native.NetDesc) == 16 * ctypes.sizeof(native.LinearDesc) + 10 * 4
    assert native.NetDesc().tc_products == 0                # zero-initialised descriptors keep the 3xFP16 default


def test_tensor_core_entry_points_take_products_after_the_stream():
    for name in ('gcbf_linear_fwd', 'gcbf_linear_bwd_data', 'gcbf_linear_bwd_weight'):
        rt, args = native.SIGS[name + '_h']
        assert rt is ctypes.c_int and args[-2:] == [native.P, ctypes.c_int]
        assert args[:2] == [ctypes.POINTER(native.H16Desc)] * 2
        assert name + '_t' not in native.SIGS and name + '_tp' not in native.SIGS      # one generation of the three products


# ---- the rounding model ---------------------------------------------------------------------------------------------------------
def _check_model(a, b, sa, sb, chunk):
    got = F1.gemm_p1(a, b, sa, sb, chunk).astype(np.float64)
    ref = a.astype(np.float64) @ b.astype(np.float64)
    bd = F1.bound(a, b, sa, sb, chunk)
    err = np.abs(got - ref)
    assert np.all(err <= bd), float((err / np.maximum(bd, 1e-300)).max())
    return float((err / np.maximum(bd, 1e-300)).max())


@pytest.mark.parametrize('M,K,N,chunk', [(33, 128, 17, 128), (64, 300, 40, 128), (17, 517, 9, 256), (5, 1000, 3, 128), (40, 96, 130, 256)])
def test_model_within_bound_random_ragged(M, K, N, chunk):
    rng = np.random.default_rng(M * 1000 + K + N)
    a = rng.standard_normal((M, K)).astype(np.float32)
    b = rng.standard_normal((K, N)).astype(np.float32)
    ratio = _check_model(a, b, F1.tensor_scales(a), F1.tensor_scales(b), chunk)
    assert ratio > 1e-3                                    # the bound is not vacuous: errors reach a visible fraction of it


@pytest.mark.parametrize('e', [-30, -12, 0, 12, 30])
def test_model_within_bound_across_magnitudes(e):
    """Operands whose max spans 2^-30 .. 2^30, rows spread over six decades (small rows land in fp16 subnormals after scaling)."""
    rng = np.random.default_rng(100 + e)
    M, K, N = 48, 384, 24
    a = (rng.uniform(-1, 1, (M, K)) * np.logspace(0, -6, M)[:, None] * 2.0 ** e).astype(np.float32)
    b = (rng.uniform(-1, 1, (K, N)) * 2.0 ** (-e // 2)).astype(np.float32)
    b[:, 0] = 0.0
    _check_model(a, b, F1.tensor_scales(a), F1.tensor_scales(b), 128)


def test_model_within_bound_tile_scaled():
    """A tile-scaled along rows and contraction (K-major emitted activations), B tile-scaled along the contraction rows (MN-major
    emitted operand of the weight-grad): per-chunk descale, chunks inside one scale tile."""
    rng = np.random.default_rng(7)
    M, K, N = 300, 512, 70
    a = (rng.standard_normal((M, K)) * np.repeat(np.array([1.0, 2.0 ** -9]), 256)[None, :] * np.logspace(0, -3, M)[:, None]).astype(np.float32)
    b = (rng.standard_normal((K, N)) * np.repeat(np.array([2.0 ** 5, 1.0, 2.0 ** -7, 1.0]), 128)[:, None]).astype(np.float32)
    sa = F1.tile_scales(a)
    # b as an MN-major operand: one scale per 128-row block of the contraction (constant over each chunk)
    sb = np.repeat(np.array([F1.scale_for(float(np.abs(b[k:k + 128]).max())) for k in range(0, K, 128)]), 128)[:, None] * np.ones((1, N))
    _check_model(a, b, sa, sb, 128)


@pytest.mark.parametrize('L', [128, 256])
def test_model_truncation_within_the_accumulation_term(L):
    """Operands that are fp16 values after scaling (no representation error), all products positive so that the truncated
    in-chunk sums lose the most: the model's error is bounded by the accumulation terms alone, and the truncation shows."""
    rng = np.random.default_rng(L)
    M, K, N = 24, 4 * L, 16
    a = rng.uniform(0.5, 1.0, (M, K)).astype(np.float16).astype(np.float32)
    b = rng.uniform(0.5, 1.0, (K, N)).astype(np.float16).astype(np.float32)
    sa, sb = F1.tensor_scales(a), F1.tensor_scales(b)
    a = (a.astype(np.float64) * sa).astype(np.float16).astype(np.float64) / sa            # exactly representable in the companion
    b = (b.astype(np.float64) * sb).astype(np.float16).astype(np.float64) / sb
    a, b = a.astype(np.float32), b.astype(np.float32)
    got = F1.gemm_p1(a, b, sa, sb, L).astype(np.float64)
    ref = a.astype(np.float64) @ b.astype(np.float64)
    bd = F1.bound(a, b, sa, sb, L, exact_operands=True)
    err = np.abs(got - ref)
    assert np.all(err <= bd), float((err / bd).max())
    assert np.all(got <= ref) and float((err / bd).max()) > 1e-3       # truncation: every result below the exact sum, visibly


def test_mode_change_on_the_params_dict_reaches_the_modules():
    env, algo = _algo()
    algo.params['matmul'] = 'fp16'                         # no entry point in between: the next pass reads the key
    for m in (algo.cbf, algo.actor):
        assert m.feat_transformer.module_0.net_spec().tc_products == 1
    algo.params['matmul'] = 'fp32'
    assert algo.actor.feat_transformer.module_0.net_spec().tc_products == 3
    algo.params['matmul'] = 'half'
    with pytest.raises(ValueError, match='matmul'):
        algo.actor.feat_transformer.module_0.net_spec()


def test_attention_refuses_fp16():
    env, algo = _algo({'matmul': 'fp16'})
    with pytest.raises(ValueError, match='attention'):
        algo.cbf.attention(None)


def test_kappa_matches_the_chunk_length():
    # L = 128-element chunks over K = 2048 (16 chunks): kappa ~ L + 3 + (16 + 1 + 3) / 2
    k = F1.kappa(128, 16)
    assert abs(k - (128 + 1 + 2 + (16 + 1 + 3) / 2)) < 1.0
    assert F1.kappa(256, 8) > F1.kappa(128, 16)
    assert math.isclose(F1.bound(np.ones((1, 1), np.float32), np.ones((1, 1), np.float32), np.ones((1, 1)) * 2.0 ** 14,
                                 np.ones((1, 1)) * 2.0 ** 14, 128)[0, 0],
                        2.0 ** -10 + F1.kappa(128, 1) * 2.0 ** -23, rel_tol=1e-3)
