"""GPU tests of the vectorised training loop: the batched episode reset (gcbf_env_reset_batch) against its numpy replica
(tests/reset_replica.py) bit for bit, its constraints and distribution, the device episode mode of VectorRollout, and
Trainer(num_envs=...)."""
import os

import numpy as np
import pytest
import torch

import reset_replica as RR
from gcbf_b200.algo.rollout import VectorRollout, evaluate_episodes
from gcbf_b200.env import make_env
from gcbf_b200.env.device_reset import raise_on_failure, reset_batch, reset_spec
from gcbf_b200.env.simple_car import SimpleCar
from gcbf_b200.trainer.utils import set_seed
from helpers import seeded_algo

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0') if torch.cuda.is_available() else None


def _env(name, n, **params):
    env = make_env(name, n, DEV)
    return make_env(name, n, DEV, params={**env.default_params, **params}) if params else env


def _device_reset(env, B, seed, first_env=0, max_tries=200000, episode=None):
    spec = reset_spec(env)
    states = torch.zeros(B * env.nodes_per_graph, env.state_dim, device=DEV)
    goals = torch.zeros(B * env.num_agents, spec['goal_dim'], device=DEV)
    t = torch.full((B,), env.max_episode_steps, device=DEV, dtype=torch.int32)
    ep = torch.full((B,), -1, device=DEV, dtype=torch.int32) if episode is None else episode
    failed = torch.full((B,), -7, device=DEV, dtype=torch.int32)
    reset_batch(env, states, goals, t, ep, failed, seed, max_tries=max_tries, first_env=first_env)
    torch.cuda.synchronize()
    return states, goals, t, ep, failed, spec


CASES = [('SimpleCar', 16, {}, 8, 0), ('SimpleCar', 64, {}, 4, 7), ('SimpleCar', 3, {}, 33, 2 ** 40 + 5), ('DubinsCar', 16, {'num_obs': 8}, 6, 3),
         ('DubinsCar', 40, {'num_obs': 4}, 3, 11), ('DubinsCar', 8, {}, 4, 1), ('SimpleDrone', 8, {}, 4, 5), ('SimpleDrone', 36, {}, 2, 9)]


@pytest.mark.parametrize('name,n,params,B,seed', CASES)
def test_kernel_equals_replica_bit_for_bit(name, n, params, B, seed):
    env = _env(name, n, **params)
    states, goals, t, ep, failed, spec = _device_reset(env, B, seed)
    N = env.nodes_per_graph
    assert failed.tolist() == [0] * B and t.tolist() == [0] * B and ep.tolist() == [0] * B
    for e in range(B):
        ws, wg, wf = RR.reset_env(name, spec, n, seed, e, 0)
        assert wf == 0
        assert np.array_equal(states[e * N:(e + 1) * N].cpu().numpy(), ws), e
        assert np.array_equal(goals[e * n:(e + 1) * n].cpu().numpy(), wg), e
    # second round: only the envs whose counter reached max_steps (or, given reach, whose agents all reached) are re-sampled
    t = torch.tensor([env.max_episode_steps if e % 2 else 1 for e in range(B)], device=DEV, dtype=torch.int32)
    reach = torch.zeros(B, n, dtype=torch.bool, device=DEV)
    reach[0] = True
    before_s, before_g = states.clone(), goals.clone()
    reset_batch(env, states, goals, t, ep, failed, seed, reach=reach)
    for e in range(B):
        sl, gl = slice(e * N, (e + 1) * N), slice(e * n, (e + 1) * n)
        if e % 2 or e == 0:
            ws, wg, _ = RR.reset_env(name, spec, n, seed, e, 1)
            assert np.array_equal(states[sl].cpu().numpy(), ws) and np.array_equal(goals[gl].cpu().numpy(), wg), e
            assert int(t[e]) == 0 and int(ep[e]) == 1
        else:
            assert torch.equal(states[sl], before_s[sl]) and torch.equal(goals[gl], before_g[gl]) and int(t[e]) == 1 and int(ep[e]) == 0


@pytest.mark.parametrize('name,params', [('SimpleCar', {}), ('DubinsCar', {'num_obs': 8})])
def test_reset_alone_equals_reset_in_a_batch(name, params):
    env = _env(name, 16, **params)
    states, goals, *_ = _device_reset(env, 256, 21)
    N, n = env.nodes_per_graph, 16
    for e in (0, 1, 77, 255):
        s1, g1, *_ = _device_reset(env, 1, 21, first_env=e)
        assert torch.equal(s1, states[e * N:(e + 1) * N]) and torch.equal(g1, goals[e * n:(e + 1) * n])


def _pair_d2(a, b):
    """[B, i, j] squared distances in the kernel's order (per-op rounding: separate eager launches)."""
    diff = a[:, :, None, :] - b[:, None, :, :]
    sq = diff * diff
    s = torch.zeros(sq.shape[:3], device=sq.device)
    for d in range(sq.shape[3]):
        s = s + sq[..., d]
    return s


@pytest.mark.parametrize('name,n,params,B', [('SimpleCar', 16, {}, 10000), ('DubinsCar', 16, {'num_obs': 8}, 10000), ('SimpleDrone', 8, {}, 10000)])
def test_constraints_hold_on_ten_thousand_resets(name, n, params, B):
    env = _env(name, n, **params)
    states, goals, t, ep, failed, spec = _device_reset(env, B, 5)
    assert int(failed.abs().sum()) == 0
    pd, N, o = env.POS_DIM, env.nodes_per_graph, spec['num_obs']
    S = states.view(B, N, -1)
    G = goals.view(B, n, -1)
    eye = torch.eye(n, dtype=torch.bool, device=DEV)
    for pts, md2 in ((S[:, :n, :pd], spec['agent_dist2']), (G[:, :, :pd], spec['goal_dist2'])):
        assert bool((pts >= 0).all()) and bool((pts < spec['area']).all())
        d2 = _pair_d2(pts, pts)
        assert bool((d2[:, ~eye] > np.float32(md2)).all())
        if o:
            assert bool((_pair_d2(pts, S[:, n:, :pd]) > np.float32(spec['clear2'])).all())
    if name == 'DubinsCar':
        for h in (S[:, :n, 2], G[:, :, 2]):
            assert bool((h >= -RR.PI).all()) and bool((h < RR.PI).all())
        assert bool((S[:, :n, 3] == 0).all()) and bool((S[:, n:, 3] < spec['obs_speed_limit']).all())
    else:
        assert bool((S[:, :, pd:] == 0).all()) and bool((G[:, :, pd:] == 0).all())


@pytest.mark.parametrize('name,params', [('SimpleCar', {}), ('DubinsCar', {'num_obs': 8})])
def test_distribution_matches_host_reset(name, params):
    from scipy.stats import ks_2samp
    n, R = 16, 400
    env = _env(name, n, **params)
    host_s, host_g = [], []
    for s in range(R):
        set_seed(10000 + s)
        data = env.reset()
        host_s.append(data.states[:n].cpu())
        host_g.append(env._goal.cpu())
    host_s, host_g = torch.stack(host_s), torch.stack(host_g)
    dev_s, dev_g, *_ = _device_reset(env, R, 99)
    dev_s, dev_g = dev_s.view(R, -1, env.state_dim)[:, :n].cpu(), dev_g.view(R, n, -1).cpu()

    def nn_dist(p):
        d = torch.cdist(p, p) + torch.eye(n) * 1e9
        return d.min(dim=2).values.reshape(-1).numpy()

    for what, a, b in (('agent x', host_s[..., 0], dev_s[..., 0]), ('agent y', host_s[..., 1], dev_s[..., 1]),
                       ('goal x', host_g[..., 0], dev_g[..., 0]), ('goal y', host_g[..., 1], dev_g[..., 1]),
                       ('agent nn', nn_dist(host_s[..., :2]), nn_dist(dev_s[..., :2])),
                       ('goal nn', nn_dist(host_g[..., :2]), nn_dist(dev_g[..., :2]))):
        a = a.reshape(-1).numpy() if torch.is_tensor(a) else a
        b = b.reshape(-1).numpy() if torch.is_tensor(b) else b
        p = ks_2samp(a, b).pvalue
        assert p > 1e-3, (what, p)


def test_unplaceable_configuration_fails_every_env_promptly():
    import time
    env = _env('SimpleCar', 400)
    t0 = time.perf_counter()
    states, goals, t, ep, failed, _ = _device_reset(env, 8, 0, max_tries=3000)
    assert time.perf_counter() - t0 < 10.0
    assert failed.tolist() == [1] * 8
    with pytest.raises(RuntimeError, match='env 0 .*400 agents with spacing 0.2'):
        raise_on_failure(env, failed.cpu().numpy())
    vr = VectorRollout(env, None, 2, reset_seed=0)                  # default budget: the next step's sync reports it
    with pytest.raises(RuntimeError, match='could not place 400 agents'):
        vr.step(store=False)


# ---- VectorRollout with device resets ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,params', [('SimpleCar', {}), ('DubinsCar', {'num_obs': 4}), ('SimpleDrone', {})])
def test_device_mode_step_equals_host_mode_step(name, params):
    n, B = 16 if name != 'SimpleDrone' else 8, 6
    env, algo = seeded_algo(name, n, DEV, 0, params)
    vd = VectorRollout(env, algo, B, reset_seed=4)
    s0, g0, *_ = _device_reset(env, B, 4)
    assert torch.equal(vd.states, s0) and torch.equal(vd.goals, g0)
    vh = VectorRollout(env, algo, B, states=vd.states.clone(), goals=vd.goals.clone())
    for k in range(3):
        a = vd.step(prob=0.0, store=False)
        b = vh.step(prob=0.0, store=False)
        for key in ('action', 'is_safe', 'u_ref', 'states', 'reach', 'collision'):
            assert torch.equal(a[key], b[key]), (k, key)
        assert torch.equal(vd.states, vh.states) and vd.t_dev.tolist() == [k + 1] * B and vd.episode.tolist() == [0] * B


class _ShortCar(SimpleCar):
    max_episode_steps = property(lambda self: 3)


def test_done_env_starts_its_next_episode_on_the_next_step():
    n, B, seed = 16, 4, 8
    _, algo = seeded_algo('SimpleCar', n, DEV, 0)
    env = _ShortCar(n, DEV)
    algo._env = env
    spec = reset_spec(env)
    N = env.nodes_per_graph
    vr = VectorRollout(env, algo, B, reset_seed=seed)
    # env 1 starts on its goals: all its agents reach at the first step
    vr.goals.view(B, n, -1)[1] = vr.states.view(B, N, -1)[1, :, :2]
    out = vr.step(prob=0.0, store=False)
    assert bool(out['reach'][1].all()) and not bool(out['reach'][0].all())
    assert vr.t_dev.tolist() == [1, 0, 1, 1] and vr.episode.tolist() == [0, 1, 0, 0]
    ws, wg, _ = RR.reset_env('SimpleCar', spec, n, seed, 1, 1)
    assert np.array_equal(vr.states[N:2 * N].cpu().numpy(), ws) and np.array_equal(vr.goals[n:2 * n].cpu().numpy(), wg)
    first = vr.states.clone()
    out = vr.step(prob=0.0, store=False)
    assert torch.equal(out['states'][N:2 * N], first[N:2 * N])         # env 1's next step starts from its episode-1 reset
    vr.step(prob=0.0, store=False)                                     # t = 3 for envs 0, 2, 3: timed out
    assert vr.t_dev.tolist() == [0, 2, 0, 0] and vr.episode.tolist() == [1, 1, 1, 1]
    for e in (0, 2, 3):
        ws, wg, _ = RR.reset_env('SimpleCar', spec, n, seed, e, 1)
        assert np.array_equal(vr.states[e * N:(e + 1) * N].cpu().numpy(), ws), e


def test_host_reset_rollout_is_unchanged():
    n, B = 16, 3
    env, algo = seeded_algo('SimpleCar', n, DEV, 0)
    set_seed(3)
    vr = VectorRollout(env, algo, B)
    set_seed(3)
    want = [env.reset().states.clone() for _ in range(B + 1)][1:]      # reset() draws one env first to size the batch
    assert torch.equal(vr.states, torch.cat(want)) and vr.reset_seed is None and not hasattr(vr, 't_dev')


# ---- Trainer(num_envs=...) --------------------------------------------------------------------------------------------------------
def _train(tmp_path, name='SimpleCar', n=16, params=None, B=8, batch_size=64, steps=256, eval_interval=128, eval_epi=2, seed=0, tag='run'):
    from gcbf_b200.trainer import Trainer
    set_seed(seed)
    env, algo = seeded_algo(name, n, DEV, 0, params)
    env_test = make_env(name, n, DEV, params=env._params)
    algo.batch_size = batch_size
    log = {'updates': [], 'ring': None, 'states': []}
    update = algo.update

    def counted(step, writer=None):
        log['updates'].append(step)
        if log['ring'] is None:
            log['ring'] = algo.buffer.states_of(range(algo.buffer.size)).clone()
        return update(step, writer)

    algo.update = counted

    class Recording(Trainer):
        def _make_rollout(self):
            vr = super()._make_rollout()
            step = vr.step

            def recorded(*a, **k):
                out = step(*a, **k)
                log['states'].append(out['states'].clone())
                return out

            vr.step = recorded
            return vr

    tr = Recording(env, env_test, algo, str(tmp_path / tag), num_envs=B, seed=seed)
    tr.train(steps, eval_interval, eval_epi)
    return tr, algo, log


def test_vectorised_trainer_runs_updates_and_checkpoints(tmp_path):
    from gcbf_b200.algo.gcbf import GCBF
    tr, algo, log = _train(tmp_path)
    B, T, n = 8, 8, 16
    assert log['updates'] == [64, 128, 192, 256]
    ring = log['ring']
    assert ring.shape[0] == B * T
    for e in range(B):
        for t in range(T):
            assert torch.equal(ring[e * T + t], log['states'][t].view(B, n, -1)[e]), (e, t)
    for k in (128, 256):
        path = os.path.join(tr.model_dir, f'step_{k}')
        fresh = GCBF(tr.env, n, tr.env.node_dim, tr.env.edge_dim, tr.env.action_dim, DEV)
        fresh.load(path)                                              # load_state_dict(strict=True)
        assert sorted(os.listdir(path)) == ['actor.pkl', 'cbf.pkl']


def test_vectorised_eval_equals_evaluate_episodes(tmp_path):
    from gcbf_b200.trainer import Trainer
    env, algo = seeded_algo('SimpleCar', 16, DEV, 0)
    env_test = make_env('SimpleCar', 16, DEV)
    tr = Trainer(env, env_test, algo, str(tmp_path / 'ev'), num_envs=8)
    cbf = {k: v.clone() for k, v in algo.cbf.state_dict().items()}
    np.random.seed(17)
    reward, info = tr.eval(0, 2)
    algo.cbf.load_state_dict(cbf)
    np.random.seed(17)
    res = evaluate_episodes(env_test, algo, np.random.randint(100000, size=2))
    assert reward == float(res['mean']['reward'])
    assert info == {'safe': round(float(res['mean']['safe']), 2), 'reach': round(float(res['mean']['reach']), 2)}


def test_vectorised_training_is_reproducible(tmp_path):
    a, _, _ = _train(tmp_path, steps=128, eval_interval=128, eval_epi=0, tag='a')
    b, _, _ = _train(tmp_path, steps=128, eval_interval=128, eval_epi=0, tag='b')
    for f in ('cbf.pkl', 'actor.pkl'):
        sa = torch.load(os.path.join(a.model_dir, 'step_128', f))
        sb = torch.load(os.path.join(b.model_dir, 'step_128', f))
        assert sa.keys() == sb.keys() and all(torch.equal(sa[k], sb[k]) for k in sa), f


@pytest.mark.parametrize('name,n,params', [('DubinsCar', 16, {'num_obs': 4}), ('SimpleDrone', 8, {})])
def test_one_interval_on_envs_with_obstacles(tmp_path, name, n, params):
    tr, algo, log = _train(tmp_path, name, n, params, steps=64, eval_interval=64, eval_epi=0)
    assert log['updates'] == [64] and os.path.isdir(os.path.join(tr.model_dir, 'step_64'))
    assert algo.memory.size == 64 and algo.memory.goals_of(range(64)).shape[1:] == (n, reset_spec(tr.env)['goal_dim'])
