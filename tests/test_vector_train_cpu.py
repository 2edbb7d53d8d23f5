"""CPU tests of the vectorised training loop's pieces:
  1. the Philox4x32-10 of csrc/reset_core.h (through tests/host_driver/reset_host.cpp, g++ -ffp-contract=off) equals CUDA's own
     curand_Philox4x32_10 compiled for the host, and the numpy replica (tests/reset_replica.py) equals both;
  2. the acceptance rule equals the numpy fp32 replica, including squared distances within 3 ulps of the threshold;
  3. the replica sampler satisfies the constraints of every env's reset();
  4. gcbf_env_reset_batch rejects bad arguments before any launch;
  5. the vectorised Trainer's glue, driven with stubs: exploration, update / checkpoint cadence, env-major staging, RNG states
     around eval, refusals.
"""
import ctypes
import os
import random
import subprocess

import numpy as np
import pytest
import torch

import reset_replica as RR
from conftest import ROOT
from gcbf_b200 import _C


def _build(name):
    out = os.path.join(ROOT, 'tests', 'host_driver', '_build')
    os.makedirs(out, exist_ok=True)
    so = os.path.join(out, name + '.so')
    cuda_inc = os.path.join(os.environ.get('CUDA_HOME', '/usr/local/cuda'), 'include')
    subprocess.check_call(['g++', '-O2', '-ffp-contract=off', '-shared', '-fPIC', '-I', os.path.join(ROOT, 'gcbf-pytorch_b200', 'csrc'),
                           '-I', os.path.join(ROOT, 'include'), '-I', cuda_inc, '-o', so,
                           os.path.join(ROOT, 'tests', 'host_driver', name + '.cpp')])
    lib = ctypes.CDLL(so)
    lib.host_draw4.argtypes = [ctypes.c_uint64, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_uint32, ctypes.c_void_p]
    lib.host_dist2.restype = ctypes.c_float
    lib.host_dist2.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int]
    lib.host_too_close.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_float]
    lib.host_heading.restype = ctypes.c_float
    lib.host_heading.argtypes = [ctypes.c_float]
    return lib


@pytest.fixture(scope='module')
def rhost():
    return _build('reset_host')


def _philox(fn, ctr, key):
    c, k, o = np.ascontiguousarray(ctr, np.uint32), np.ascontiguousarray(key, np.uint32), np.zeros(4, np.uint32)
    fn(c.ctypes.data, k.ctypes.data, o.ctypes.data)
    return o


# ---- 1. Philox --------------------------------------------------------------------------------------------------------------------
def test_philox_equals_curand_and_the_known_answer(rhost):
    zero = [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]        # Random123's known-answer vector for counter 0, key 0
    assert _philox(rhost.host_philox, [0] * 4, [0, 0]).tolist() == zero
    assert _philox(rhost.curand_philox, [0] * 4, [0, 0]).tolist() == zero
    rng = np.random.default_rng(3)
    for _ in range(2000):
        ctr, key = rng.integers(0, 2 ** 32, 4, dtype=np.uint64), rng.integers(0, 2 ** 32, 2, dtype=np.uint64)
        want = _philox(rhost.curand_philox, ctr, key)
        assert np.array_equal(_philox(rhost.host_philox, ctr, key), want)
        got = RR.philox(*[int(x) for x in ctr], int(key[0]), int(key[1]))
        assert [int(x) for x in got] == want.tolist()


def test_uniforms_and_headings_equal_the_replica(rhost):
    rng = np.random.default_rng(4)
    u = np.zeros(4, np.float32)
    for _ in range(500):
        seed, env, ep, tag, k = int(rng.integers(0, 2 ** 63)), int(rng.integers(0, 1000)), int(rng.integers(0, 50)), int(rng.integers(0, 4)), \
            int(rng.integers(0, 2 ** 31))
        rhost.host_draw4(seed, env, ep, tag, k, u.ctypes.data)
        want = RR.uniforms(seed, env, ep, tag, [k])[0]
        assert np.array_equal(u, want) and (u >= 0).all() and (u < 1).all()
        h = np.float32(rhost.host_heading(float(u[0])))
        assert h == u[0] * RR.TWO_PI - RR.PI
    top = np.float32(1 - 2 ** -24)                                      # the largest uniform stays inside [-pi, pi)
    assert -RR.PI <= np.float32(rhost.host_heading(0.0)) and np.float32(rhost.host_heading(float(top))) < RR.PI


# ---- 2. acceptance rule -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('dim', [2, 3])
def test_acceptance_equals_fp32_replica_near_the_threshold(rhost, dim):
    rng = np.random.default_rng(dim)
    for _ in range(400):
        p = rng.uniform(0, 4, dim).astype(np.float32)
        c = (p + rng.normal(0, 0.2, dim)).astype(np.float32)
        d2 = RR.dist2(p[None], c)[0]
        assert np.float32(rhost.host_dist2(p.ctypes.data, c.ctypes.data, dim)) == d2
        for ulps in range(-3, 4):
            md2 = d2
            for _ in range(abs(ulps)):
                md2 = np.nextafter(md2, np.float32(np.inf if ulps > 0 else -np.inf), dtype=np.float32)
            got = rhost.host_too_close(p.ctypes.data, c.ctypes.data, dim, float(md2))
            assert got == int(d2 <= md2) == int(ulps >= 0)


# ---- 3. the replica sampler ---------------------------------------------------------------------------------------------------------
def _spec(name, n, **params):
    from gcbf_b200.env import make_env
    from gcbf_b200.env.device_reset import reset_spec
    env = make_env(name, n, torch.device('cpu'))
    if params:
        env = make_env(name, n, torch.device('cpu'), params={**env.default_params, **params})
    return env, reset_spec(env)


@pytest.mark.parametrize('name,n,params', [('SimpleCar', 16, {}), ('SimpleCar', 64, {}), ('DubinsCar', 16, {'num_obs': 8}),
                                           ('DubinsCar', 8, {}), ('SimpleDrone', 12, {})])
def test_replica_sampler_satisfies_the_reset_constraints(name, n, params):
    env, spec = _spec(name, n, **params)
    assert spec['num_obs'] == env.num_obstacles
    for e in range(6):
        states, goals, failed = RR.reset_env(name, spec, n, 1234, e, e % 3)
        assert failed == 0
        assert states.shape == (env.nodes_per_graph, env.state_dim) and goals.shape == (n, env.RESET_GOAL_DIM)
        assert RR.check_constraints(name, spec, n, states, goals) == []
    a = RR.reset_env(name, spec, n, 1234, 0, 0)
    b = RR.reset_env(name, spec, n, 1234, 0, 1)
    c = RR.reset_env(name, spec, n, 1234, 1, 0)
    assert not np.array_equal(a[0], b[0]) and not np.array_equal(a[0], c[0])   # episode and env id select the stream


def test_replica_sampler_reports_an_impossible_set():
    _, spec = _spec('SimpleCar', 400)
    _, _, failed = RR.reset_env('SimpleCar', spec, 400, 0, 0, 0, max_tries=2000)
    assert failed == 1


def test_env_constants_keep_the_host_draws(monkeypatch):
    """reset() reads its spacings from the class attributes; its draws are sample_separated's with the literal constants."""
    from gcbf_b200.env import make_env
    from gcbf_b200.env._sampling import sample_separated
    from gcbf_b200.env.base import MultiAgentEnv
    from gcbf_b200.trainer.utils import set_seed
    monkeypatch.setattr(MultiAgentEnv, 'add_communication_links', lambda self, data: data)     # the graph build needs the GPU
    env = make_env('SimpleCar', 8, torch.device('cpu'))
    set_seed(11)
    data = env.reset()
    set_seed(11)
    pos = sample_separated(8, 2, 4.0, 4 * 0.05)
    goal = sample_separated(8, 2, 4.0, 4 * 0.05)
    assert torch.equal(data.states[:, :2], pos) and torch.equal(env._goal, goal)
    env = make_env('DubinsCar', 8, torch.device('cpu'), params={**make_env('DubinsCar', 8, torch.device('cpu')).default_params, 'num_obs': 4})
    set_seed(12)
    data = env.reset()
    set_seed(12)
    obs = torch.rand(4, 4)
    obs[:, :2] *= 4.0
    pos = sample_separated(8, 2, 4.0, 4 * 0.05, obs[:, :2], 2 * 0.05 + 2 * 0.05)
    goal = sample_separated(8, 2, 4.0, 5 * 0.05, obs[:, :2], 2 * 0.05 + 2 * 0.05)
    assert torch.equal(data.states[:8, :2], pos) and torch.equal(env._goal[:, :2], goal)


# ---- 4. C entry point ---------------------------------------------------------------------------------------------------------------
def _desc(**over):
    d = _C.ResetDesc()
    fake = 0x7f0000000000
    d.seed = 1
    d.states = d.goals = d.step_count = d.episode = d.failed = fake
    d.reach = None
    d.env, d.num_envs, d.num_agents, d.num_obs = 0, 4, 16, 0
    d.ld_state, d.ld_goal, d.goal_dim, d.max_steps, d.max_tries, d.first_env = 4, 2, 2, 500, 1000, 0
    d.area, d.agent_dist2, d.goal_dist2, d.clear2, d.obs_speed_limit = 4.0, 0.04, 0.04, 0.0, 0.0
    for k, v in over.items():
        setattr(d, k, v)
    return d


def test_abi_struct_14_is_the_reset_descriptor():
    assert ctypes.sizeof(_C.ResetDesc) == _C.lib().gcbf_abi_struct_size(14)


@pytest.mark.parametrize('over,msg', [({'env': 3}, 'unknown env'), ({'num_envs': 0}, 'bad sizes'), ({'num_agents': 0}, 'bad sizes'),
                                      ({'num_obs': 2}, 'no obstacles'), ({'states': None}, 'null pointer'),
                                      ({'failed': None}, 'null pointer'), ({'ld_state': 3}, 'ld_state'), ({'goal_dim': 1}, 'goal_dim'),
                                      ({'ld_goal': 1}, 'goal_dim'), ({'max_tries': 0}, 'max_tries'), ({'area': 0.0}, 'area'),
                                      ({'agent_dist2': float('nan')}, 'area'), ({'first_env': -1}, 'first_env'),
                                      ({'env': 2, 'num_agents': 9000, 'num_obs': 9000, 'ld_state': 6, 'goal_dim': 6, 'ld_goal': 6},
                                       'shared memory')])
def test_reset_batch_rejects_bad_arguments_before_any_launch(over, msg):
    lib = _C.lib()
    d = _desc(**over)
    assert lib.gcbf_env_reset_batch(ctypes.byref(d), None) == -1
    assert msg in lib.gcbf_last_error().decode()
    assert lib.gcbf_env_reset_batch(None, None) == -1


def test_reset_failure_message_names_env_and_constraint():
    from gcbf_b200.env.device_reset import raise_on_failure
    env, _ = _spec('DubinsCar', 16, num_obs=4)
    raise_on_failure(env, np.zeros(3, np.int32))
    with pytest.raises(RuntimeError, match=r'env 5 .*16 goals with spacing 0.25 and clearance 0.2 from 4 obstacles'):
        raise_on_failure(env, np.array([0, 2, 1], np.int32), first_env=4)


# ---- 5. the vectorised Trainer's glue ----------------------------------------------------------------------------------------------
class _Env:
    num_agents, nodes_per_graph = 2, 3


class _Ring:
    def __init__(self):
        self.size, self.appended = 0, []

    def append_batch(self, states, u_ref, is_safe, goals):
        self.appended.append((states.clone(), u_ref.clone(), is_safe.clone(), goals.clone()))
        self.size += int(states.shape[0])


class _Algo:
    def __init__(self, batch_size=12):
        self.batch_size, self.process_group, self.device_replay = batch_size, None, False
        self.buffer, self.memory = _Ring(), _Ring()
        self.updates, self.saved, self.ring_at_update = [], [], []
        self._env = None

    def use_device_replay(self):
        self.device_replay = True
        self.buffer, self.memory = _Ring(), _Ring()
        return self

    def update(self, step, writer):
        self.updates.append(step)
        self.ring_at_update.append(len(self.buffer.appended))
        return {'acc/safe': 1.0}

    def save(self, path):
        self.saved.append(os.path.basename(path))


class _Rollout:
    """Env e's k-th step has states filled with 1000 k + e (and u_ref / goals derived from it)."""

    def __init__(self, B):
        self.B, self.k, self.probs, self.checks = B, 0, [], 0

    def step(self, prob, store):
        assert store is False
        self.probs.append(prob)
        B, k = self.B, self.k
        tag = (1000.0 * k + torch.arange(B, dtype=torch.float32))
        self.k += 1
        return dict(states=tag.repeat_interleave(3).unsqueeze(1).repeat(1, 4), u_ref=tag.repeat_interleave(2).unsqueeze(1).repeat(1, 2),
                    goals=-tag.repeat_interleave(2).unsqueeze(1).repeat(1, 2), is_safe=(torch.arange(B) + k) % 2 == 0)

    def check_resets(self):
        self.checks += 1


def _trainer(tmp_path, algo, B, **kw):
    from gcbf_b200.trainer import trainer as T

    class StubTrainer(T.Trainer):
        def _make_rollout(self):
            self.rollout = _Rollout(self.num_envs)
            return self.rollout

    return StubTrainer(_Env(), _Env(), algo, str(tmp_path / 'run'), num_envs=B, **kw)


def test_vectorised_trainer_cadence_and_env_major_staging(tmp_path):
    algo = _Algo(batch_size=12)
    tr = _trainer(tmp_path, algo, 4)
    assert algo.device_replay
    tr.train(steps=48, eval_interval=24, eval_epi=0)
    B, T = 4, 3
    assert np.allclose(tr.rollout.probs, [1 - k * B / 48 for k in range(12)])
    assert algo.updates == [12, 24, 36, 48] and algo.ring_at_update == [1, 2, 3, 4]       # every batch_size transitions
    assert algo.saved == ['step_24', 'step_48'] and algo._env is tr.env
    for j, (states, u_ref, is_safe, goals) in enumerate(algo.buffer.appended):
        assert states.shape == (B * T, 3, 4) and u_ref.shape == (B * T, 2, 2) and goals.shape == (B * T, 2, 2)
        for e in range(B):
            for t in range(T):
                k = j * T + t
                row = e * T + t                                   # ring entries e T .. e T + T - 1: env e's steps in order
                assert torch.all(states[row] == 1000 * k + e) and torch.all(u_ref[row] == 1000 * k + e)
                assert torch.all(goals[row] == -(1000 * k + e)) and bool(is_safe[row]) == ((e + k) % 2 == 0)
    assert tr.rollout.checks == 4


def test_vectorised_eval_restores_rng_states(tmp_path, monkeypatch):
    from gcbf_b200.trainer import trainer as T
    from gcbf_b200.trainer.utils import set_seed
    seen = {}

    def fake_eval(env, algo, seeds):
        seen['seeds'] = list(seeds)
        for s in seeds:
            set_seed(int(s))
        return {'mean': {'reward': 2.5, 'safe': 0.875, 'reach': 0.333}}

    monkeypatch.setattr(T, 'evaluate_episodes', fake_eval)
    algo = _Algo()
    tr = _trainer(tmp_path, algo, 4)
    set_seed(5)
    r0, n0, t0 = random.getstate(), np.random.get_state(), torch.get_rng_state()
    reward, info = tr.eval(7, 3)
    assert reward == 2.5 and info == {'safe': 0.88, 'reach': 0.33} and algo._env is tr.env_test
    np.random.set_state(n0)
    assert seen['seeds'] == np.random.randint(100000, size=3).tolist()      # the seeds come from the training stream ...
    n1 = np.random.get_state()
    set_seed(5)
    np.random.randint(100000, size=3)
    assert random.getstate() == r0 and torch.equal(torch.get_rng_state(), t0)       # ... which continues after eval
    assert np.array_equal(n1[1], np.random.get_state()[1])


def test_vectorised_eval_in_the_training_loop_keeps_the_stream(tmp_path, monkeypatch):
    from gcbf_b200.trainer import trainer as T
    monkeypatch.setattr(T, 'evaluate_episodes', lambda env, algo, seeds: {'mean': {'reward': 0.0, 'safe': 1.0, 'reach': 1.0}})
    algo = _Algo(batch_size=12)
    tr = _trainer(tmp_path, algo, 4)
    tr.train(steps=24, eval_interval=12, eval_epi=2)
    assert algo.saved == ['step_12', 'step_24'] and algo.updates == [12, 24]


def test_vectorised_trainer_refusals(tmp_path):
    from gcbf_b200.algo.macbf import MACBF
    with pytest.raises(ValueError, match='multiple of num_envs'):
        _trainer(tmp_path, _Algo(batch_size=12), 5)
    with pytest.raises(ValueError, match='at least 3'):
        _trainer(tmp_path, _Algo(batch_size=12), 6)
    algo = _Algo()
    algo.process_group = object()
    with pytest.raises(NotImplementedError, match='data-parallel'):
        _trainer(tmp_path, algo, 4)
    algo = _Algo()
    algo.buffer.size = 3
    with pytest.raises(ValueError, match='use_device_replay'):
        _trainer(tmp_path, algo, 4)
    macbf = MACBF.__new__(MACBF)
    macbf.batch_size = 12
    with pytest.raises(NotImplementedError, match='MACBF'):
        _trainer(tmp_path, macbf, 4)
    algo = _Algo()
    algo.device_replay = True                     # already on the device ring: kept as it is
    ring = algo.buffer
    _trainer(tmp_path, algo, 4)
    assert algo.buffer is ring
