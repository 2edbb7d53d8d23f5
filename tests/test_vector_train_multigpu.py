"""Data-parallel vectorised training: Trainer(num_envs=B) with algo.process_group set, two ranks.

Every GPU scenario runs twice: through NCCL with one GPU per rank (skipped below 2 devices), and through gloo with both ranks on
one GPU.  Workers are started with mp.spawn(join=True) and write what they saw under tmp_path; the test compares it against one
process.  Scenarios:
  1. rank r's device episode resets are envs r B .. r B + B - 1 of one rollout over 2 B envs, bit for bit, across episode ends;
  2. one update on two ranks equals one train step in one process on the union of the windows the ranks sampled;
  3. after a short run with updates and evaluations, the replicas (weights, Adam moments, spectral-norm u, v) are bitwise equal,
     the ranks drew different exploration coins and windows, each reproducible from the seed, only rank 0 wrote checkpoints and
     progress lines, and both ranks got the same eval() result;
  4. sharded evaluation equals evaluate_episodes over all seeds in one process, bit for bit, for even, odd and fewer-than-ranks
     episode counts;
  5. refusals come before any collective (no GPU needed)."""
import contextlib
import io
import os
import socket

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gcbf_b200.env.simple_car import SimpleCar
from gcbf_b200.synth import seeded_algo

B, N_AG, SEED = 8, 16, 5
BACKENDS = [pytest.param('nccl', marks=[pytest.mark.gpu, pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')]),
            pytest.param('gloo', marks=pytest.mark.gpu)]


class _ShortCar(SimpleCar):
    """SimpleCar whose episodes end after 4 steps: resets happen within a few vector steps."""
    max_episode_steps = property(lambda self: 4)


class _EvalCar(SimpleCar):
    """SimpleCar with 6-step evaluation episodes."""
    max_episode_steps = property(lambda self: 6)


def _port():
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        return s.getsockname()[1]


def _worker(rank, world, port, backend, scenario, out_dir):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dev = torch.device('cuda', rank if backend == 'nccl' else 0)
    torch.cuda.set_device(dev)
    if backend == 'nccl':
        dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    else:
        dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        out = scenario(rank, dev, out_dir)
        torch.save(out, os.path.join(out_dir, f'{scenario.__name__}_r{rank}.pt'))
    finally:
        dist.destroy_process_group()


def _spawn(backend, scenario, tmp_path):
    mp.spawn(_worker, args=(2, _port(), backend, scenario, str(tmp_path)), nprocs=2, join=True)
    return [torch.load(tmp_path / f'{scenario.__name__}_r{r}.pt', weights_only=False) for r in range(2)]


def _dp_algo(dev, env=None, batch_size=48):
    """SimpleCar n = 16 GCBF with the seeded initial weights, data-parallel over the default group."""
    train_env, algo = seeded_algo('SimpleCar', N_AG, dev, 0)
    if env is not None:
        algo._env = train_env = env
    algo.batch_size = batch_size
    algo.process_group = dist.group.WORLD if dist.is_initialized() else None
    return train_env, algo


def _nets(algo):
    return {f'{name}.{k}': v.detach().cpu().clone() for name, net in (('cbf', algo.cbf), ('actor', algo.actor))
            for k, v in net.state_dict().items()}


# ---- 1. global env ids ---------------------------------------------------------------------------------------------------------------
def _zero_policy(batch):
    return torch.zeros_like(batch.u_ref)


def _roll(vr, steps):
    """(states, goals, step counters, episode counters) before the first step and after every step, under zero actions."""
    rec = [(vr.states.cpu(), vr.goals.cpu(), vr.t_dev.cpu(), vr.episode.cpu())]
    for _ in range(steps):
        vr.step(store=False, policy=_zero_policy)
        rec.append((vr.states.cpu(), vr.goals.cpu(), vr.t_dev.cpu(), vr.episode.cpu()))
    return rec


def _envs_scenario(rank, dev, out_dir):
    from gcbf_b200.trainer import Trainer
    env, algo = _dp_algo(dev, _ShortCar(N_AG, dev))
    tr = Trainer(env, env, algo, os.path.join(out_dir, f'envs_{rank}'), num_envs=B, seed=SEED)
    return _roll(tr._make_rollout(), 10)


@pytest.mark.parametrize('backend', BACKENDS)
def test_rank_envs_are_rows_of_one_rollout(tmp_path, backend):
    from gcbf_b200.algo.rollout import VectorRollout
    ranks = _spawn(backend, _envs_scenario, tmp_path)
    dev = torch.device('cuda:0')
    env = _ShortCar(N_AG, dev)
    one = _roll(VectorRollout(env, None, 2 * B, reset_seed=SEED), 10)
    N, n = env.nodes_per_graph, env.num_agents
    assert int(one[-1][3].min()) >= 2                                  # every env has started at least two new episodes
    for r, rec in enumerate(ranks):
        for k, ((s, g, t, ep), (s1, g1, t1, ep1)) in enumerate(zip(rec, one)):
            assert torch.equal(s, s1[r * B * N:(r + 1) * B * N]), (r, k)
            assert torch.equal(g, g1[r * B * n:(r + 1) * B * n]), (r, k)
            assert torch.equal(t, t1[r * B:(r + 1) * B]) and torch.equal(ep, ep1[r * B:(r + 1) * B]), (r, k)


# ---- 2. one update across ranks = one process on the union ------------------------------------------------------------------------
def _update_scenario(rank, dev, out_dir):
    import gcbf_b200.algo.device_buffer as DB
    from gcbf_b200.trainer import Trainer
    from gcbf_b200.trainer.utils import set_seed
    set_seed(SEED)
    env, algo = _dp_algo(dev)
    algo.params['inner_iter'] = 1
    tr = Trainer(env, env, algo, os.path.join(out_dir, f'update_{rank}'), num_envs=B, seed=SEED)
    got = {}
    collate, train_step, update = DB.collate, algo.train_step, algo.update

    def recorded_collate(env_, parts):
        for key, of in (('states', 'states_of'), ('u_ref', 'u_ref_of'), ('goals', 'goals_of')):
            got[key] = torch.cat([getattr(ring, of)(idx) for ring, idx in parts if len(idx)]).cpu()
        return collate(env_, parts)

    def recorded_step(batch, apply_optim=True, compute_acc_h_dot=True):
        res = train_step(batch, apply_optim=False, compute_acc_h_dot=compute_acc_h_dot)
        got.update(scalars=res['scalars'].cpu().clone(), acc=float(res['acc_h_dot']), grad=algo._bucket.grad.cpu().clone())
        if apply_optim:
            algo.optim_step()
        return res

    def recorded_update(step, writer=None):
        got['before'] = _nets(algo)
        return update(step, writer)

    DB.collate, algo.train_step, algo.update = recorded_collate, recorded_step, recorded_update
    tr.train(steps=algo.batch_size, eval_interval=0, eval_epi=0)
    got['weights'] = algo._bucket.flat.cpu().clone()
    return got


@pytest.mark.parametrize('backend', BACKENDS)
def test_one_update_equals_one_process_on_the_union(tmp_path, backend):
    from gcbf_b200.algo.device_buffer import DeviceReplay, collate
    r0, r1 = _spawn(backend, _update_scenario, tmp_path)
    assert r0['before'].keys() == r1['before'].keys()
    assert all(torch.equal(r0['before'][k], r1['before'][k]) for k in r0['before'])     # same replicas going into the update
    dev = torch.device('cuda:0')
    env, algo = seeded_algo('SimpleCar', N_AG, dev, 0)
    algo.cbf.load_state_dict({k[4:]: v for k, v in r0['before'].items() if k.startswith('cbf.')})
    algo.actor.load_state_dict({k[6:]: v for k, v in r0['before'].items() if k.startswith('actor.')})
    ring = DeviceReplay(dev)
    states, u_ref, goals = (torch.cat([r0[k], r1[k]]).to(dev) for k in ('states', 'u_ref', 'goals'))
    ring.append_batch(states, u_ref, torch.ones(states.shape[0], dtype=torch.bool, device=dev), goals)
    env.set_goal(goals[-1])           # as after a rollout; the batch carries every graph's own goal set (batch.goal)
    res = algo.train_step(collate(env, [(ring, list(range(states.shape[0])))]), apply_optim=False)
    one = dict(scalars=res['scalars'].cpu(), acc=float(res['acc_h_dot']), grad=algo._bucket.grad.cpu())
    assert torch.equal(r0['grad'], r1['grad'])                                    # same reduced gradient on every rank
    for r in (r0, r1):
        assert torch.allclose(r['scalars'][:7], one['scalars'][:7], rtol=0, atol=2e-6)   # global masked means
        assert r['scalars'][7].item() == one['scalars'][7].item()                # global agent count
        assert abs(r['acc'] - one['acc']) < 1e-6
    rel = (r0['grad'].double() - one['grad'].double()).norm() / one['grad'].double().norm()
    assert rel < 2e-2, rel.item()     # (ReLU-flip noise, see test_parity_gpu.test_raw_gradients_against_live_oracle)
    assert torch.equal(r0['weights'], r1['weights'])                              # replicas stay bit-identical


# ---- 3. a short training run: lockstep, per-rank streams, rank-0 side effects --------------------------------------------------
def _recording(fn, log):
    def wrapped(*args, **kwargs):
        out = fn(*args, **kwargs)
        log.append(np.array(out, copy=True))
        return out
    return wrapped


def _one_run(rank, dev, log_dir):
    from gcbf_b200.trainer import Trainer
    from gcbf_b200.trainer.utils import set_seed
    set_seed(SEED)                                                     # every rank alike, as a training script does
    env, algo = _dp_algo(dev)
    tr = Trainer(env, _EvalCar(N_AG, dev), algo, log_dir, num_envs=B, seed=SEED)
    coins, windows, saved, evals = [], [], [], []
    for ring in (algo.buffer, algo.memory):
        ring.sample_windows = _recording(ring.sample_windows, windows)
    save, evaluate = algo.save, tr.eval
    algo.save = lambda path: (saved.append(os.path.basename(path)), save(path))
    tr.eval = lambda step, epi: evals.append(evaluate(step, epi)) or evals[-1]
    rand = np.random.rand
    np.random.rand = _recording(rand, coins)
    printed = io.StringIO()
    try:
        with contextlib.redirect_stdout(printed):
            tr.train(steps=2 * algo.batch_size, eval_interval=algo.batch_size, eval_epi=3)
    finally:
        np.random.rand = rand
    b = algo._bucket
    uv = {k: v for k, v in _nets(algo).items() if k.endswith(('_u', '_v'))}
    return dict(flat=b.flat.cpu().clone(), exp_avg=b.exp_avg.cpu().clone(), exp_avg_sq=b.exp_avg_sq.cpu().clone(), uv=uv,
                coins=coins, windows=windows, saved=saved, evals=evals, printed=printed.getvalue())


def _train_scenario(rank, dev, out_dir):
    return {tag: _one_run(rank, dev, os.path.join(out_dir, tag)) for tag in ('a', 'b')}


@pytest.mark.parametrize('backend', BACKENDS)
def test_training_run_stays_in_lockstep_with_rank_streams(tmp_path, backend):
    r0, r1 = _spawn(backend, _train_scenario, tmp_path)
    for tag in ('a', 'b'):
        a, b = r0[tag], r1[tag]
        for key in ('flat', 'exp_avg', 'exp_avg_sq'):
            assert torch.equal(a[key], b[key]), (tag, key)
        assert a['uv'].keys() == b['uv'].keys() and len(a['uv']) > 0
        assert all(torch.equal(a['uv'][k], b['uv'][k]) for k in a['uv']), tag
        # per-rank streams: 12 vector steps of coins; windows from the ring, then from ring and memory, for 10 inner iterations each
        assert len(a['coins']) == len(b['coins']) == 12 and len(a['windows']) == len(b['windows']) == 30
        assert not any(np.array_equal(x, y) for x, y in zip(a['coins'], b['coins']))
        assert not np.array_equal(np.concatenate(a['windows']), np.concatenate(b['windows']))
        # side effects on rank 0 only, the same evaluation on both ranks
        assert a['saved'] == ['step_48', 'step_96'] and b['saved'] == []
        assert sorted(os.listdir(tmp_path / tag / 'models')) == ['step_48', 'step_96']
        assert 'step: 96' in a['printed'] and b['printed'] == ''
        assert len(a['evals']) == 2 and a['evals'] == b['evals']
    for r in (r0, r1):                                                 # the same seed reproduces each rank's stream
        assert all(np.array_equal(x, y) for x, y in zip(r['a']['coins'], r['b']['coins']))
        assert all(np.array_equal(x, y) for x, y in zip(r['a']['windows'], r['b']['windows']))
        assert torch.equal(r['a']['flat'], r['b']['flat'])


# ---- 4. sharded evaluation = one process ------------------------------------------------------------------------------------------
EVAL_SEEDS = [[17], list(range(100, 104)), list(range(200, 205))]


def _same_start(algo):
    """Every controller call starts from the seeded spectral-norm u, v: sigma is not bit-stationary across passes, and the shards
    make different numbers of passes than one process does (test_apply_batch_gpu's evaluate_episodes test does the same)."""
    start = (algo.cbf.state_dict(), algo.actor.state_dict())
    start = tuple({k: v.clone() for k, v in sd.items()} for sd in start)
    apply_batch = algo.apply_batch

    def fresh(batch, **kwargs):
        algo.cbf.load_state_dict(start[0])
        algo.actor.load_state_dict(start[1])
        return apply_batch(batch, **kwargs)
    algo.apply_batch = fresh


def _eval_setup(dev):
    from gcbf_b200 import ops
    ops.GEMM_IMPL = 1                          # fp32 paths: a graph's controller result does not depend on its batch
    env, algo = seeded_algo('SimpleCar', N_AG, dev, 0)
    env_test = _EvalCar(N_AG, dev)
    algo._env = env_test
    _same_start(algo)
    return env_test, algo


def _eval_scenario(rank, dev, out_dir):
    from gcbf_b200.distributed import Reducer
    from gcbf_b200.trainer.trainer import evaluate_sharded
    env, algo = _eval_setup(dev)
    red = Reducer(dist.group.WORLD)
    return [evaluate_sharded(env, algo, seeds, red, rand=0) for seeds in EVAL_SEEDS]


@pytest.mark.parametrize('backend', BACKENDS)
def test_sharded_evaluation_equals_one_process(tmp_path, backend):
    from gcbf_b200 import ops
    from gcbf_b200.algo.rollout import EPISODE_ARRAYS, evaluate_episodes
    ranks = _spawn(backend, _eval_scenario, tmp_path)
    old = ops.GEMM_IMPL
    try:
        env, algo = _eval_setup(torch.device('cuda:0'))
        want = [evaluate_episodes(env, algo, seeds, rand=0) for seeds in EVAL_SEEDS]
    finally:
        ops.GEMM_IMPL = old
    for r, got in enumerate(ranks):
        for seeds, g, w in zip(EVAL_SEEDS, got, want):
            for k in EPISODE_ARRAYS:
                assert g[k].dtype == w[k].dtype and np.array_equal(g[k], w[k]), (r, len(seeds), k, g[k], w[k])
            assert g['mean'] == w['mean'] and g['std'] == w['std'], (r, len(seeds))
            assert torch.equal(g['final_states'], w['final_states']) and g['seeds'] == w['seeds'], (r, len(seeds))
    assert max(want[2]['length']) > 1                                  # episodes ran for more than one step


def _host_helpers_worker(rank, world, port):
    from gcbf_b200.distributed import Reducer
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        red = Reducer()
        seeds = red.broadcast_host(np.arange(5, dtype=np.int64) * (rank + 1))
        assert seeds.tolist() == [0, 1, 2, 3, 4]                      # rank 0's array everywhere
        for dtype in (np.float64, np.int64, np.float32):
            rows = (3, 0)[rank]                                          # unequal, one rank empty
            mine = np.arange(rows * 4, dtype=dtype).reshape(rows, 2, 2) + 100 * rank
            got = red.gather_rows(mine)
            assert got.dtype == dtype and got.shape == (3, 2, 2) and np.array_equal(got, np.arange(12, dtype=dtype).reshape(3, 2, 2))
            mine = np.full((rank + 1,), rank, dtype=dtype)
            assert red.gather_rows(mine, [1, 2]).tolist() == [0, 1, 1]
    finally:
        dist.destroy_process_group()


def test_host_broadcast_and_gather_of_unequal_rows():
    mp.spawn(_host_helpers_worker, args=(2, _port()), nprocs=2, join=True)


# ---- 5. refusals before any collective ---------------------------------------------------------------------------------------------
class _StubAlgo:
    device_replay = True

    def __init__(self, batch_size, group):
        self.batch_size, self.process_group = batch_size, group


def _refusal_worker(rank, world, port, log_dir):
    from gcbf_b200.algo.macbf import MACBF
    from gcbf_b200.trainer import Trainer
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    dist.init_process_group('gloo', rank=rank, world_size=world)
    try:
        calls = []
        for name in ('all_reduce', 'all_gather', 'all_gather_into_tensor', 'broadcast', 'barrier', 'new_group'):
            fn = getattr(dist, name)
            setattr(dist, name, lambda *a, _fn=fn, _name=name, **k: calls.append(_name) or _fn(*a, **k))
        macbf = MACBF.__new__(MACBF)
        macbf.batch_size, macbf.process_group = 12, dist.group.WORLD
        with pytest.raises(NotImplementedError, match='MACBF'):
            Trainer(None, None, macbf, log_dir, num_envs=4)
        with pytest.raises(ValueError, match='multiple of num_envs'):
            Trainer(None, None, _StubAlgo(12, dist.group.WORLD), log_dir, num_envs=5)
        with pytest.raises(ValueError, match='at least 3'):
            Trainer(None, None, _StubAlgo(12, dist.group.WORLD), log_dir, num_envs=6)
        assert calls == [] and not os.path.exists(log_dir)
    finally:
        dist.destroy_process_group()


def test_refusals_come_before_any_collective(tmp_path):
    mp.spawn(_refusal_worker, args=(2, _port(), str(tmp_path / 'run')), nprocs=2, join=True)


def test_group_without_initialised_distributed_is_refused(tmp_path):
    from gcbf_b200.trainer import Trainer
    assert not dist.is_initialized()
    with pytest.raises(NotImplementedError, match='torch.distributed to be initialised'):
        Trainer(None, None, _StubAlgo(12, object()), str(tmp_path / 'run'), num_envs=4)
    assert not os.path.exists(tmp_path / 'run')
