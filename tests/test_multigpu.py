"""2-GPU data-parallel equality (SURVEY section 4 tier 6): two NCCL ranks, each owning half of the graphs, must produce
the same losses and the same all-reduced gradient as one process on the concatenated batch.  Needs >= 2 visible GPUs
(`python -m pytest tests/test_multigpu.py -m gpu` on a machine with two GPUs)."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from gcbf_b200 import synth

pytestmark = pytest.mark.gpu
CASE = dict(env='DubinsCar', num_agents=32, num_obs=6, num_graphs=6, area_size=3.0, seed=71)


def _run(rank, world, port, out_dir):
    os.environ.update(MASTER_ADDR='127.0.0.1', MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device('cuda', rank)
    if world > 1:
        dist.init_process_group('nccl', rank=rank, world_size=world, device_id=dev)
    try:
        from gcbf_b200.distributed import shard_range
        sb = synth.make_states(**CASE)
        env, algo = synth.seeded_algo(sb.env, sb.num_agents, dev, 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
        env.set_goal(sb.goals)
        env._obs = sb.obs.to(dev)
        N = sb.nodes_per_graph
        lo, hi = shard_range(sb.num_graphs, world, rank)
        data = env.graph_from_states(sb.states[lo * N:hi * N].to(dev))
        res = algo.train_step(data, apply_optim=False)
        torch.save(dict(scalars=res['scalars'].cpu(), acc=float(res['acc_h_dot']), grad=algo._bucket.grad.cpu(),
                        h=res['h'].cpu()), os.path.join(out_dir, f'w{world}_r{rank}.pt'))
        algo.optim_step()
        torch.save(algo._bucket.flat.cpu(), os.path.join(out_dir, f'w{world}_r{rank}_weights.pt'))
    finally:
        if world > 1:
            dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason='needs 2 GPUs')
def test_two_ranks_equal_one_rank(tmp_path):
    with socket.socket() as s:
        s.bind(('127.0.0.1', 0))
        port = s.getsockname()[1]
    _run(0, 1, port, str(tmp_path))
    mp.spawn(_run, args=(2, port, str(tmp_path)), nprocs=2, join=True)
    one = torch.load(tmp_path / 'w1_r0.pt')
    r0, r1 = torch.load(tmp_path / 'w2_r0.pt'), torch.load(tmp_path / 'w2_r1.pt')
    assert torch.equal(r0['grad'], r1['grad'])                                    # same reduced gradient on every rank
    assert torch.allclose(r0['scalars'][:7], one['scalars'][:7], rtol=0, atol=2e-6)   # global masked means
    assert r0['scalars'][7].item() == one['scalars'][7].item()                    # global agent count
    assert abs(r0['acc'] - one['acc']) < 1e-6
    assert torch.allclose(torch.cat([r0['h'], r1['h']]), one['h'], rtol=0, atol=2e-6)
    rel = (r0['grad'].double() - one['grad'].double()).norm() / one['grad'].double().norm()
    assert rel < 2e-2, rel.item()     # (ReLU-flip noise, see test_parity_gpu.test_raw_gradients_against_live_oracle)
    w0, w1 = torch.load(tmp_path / 'w2_r0_weights.pt'), torch.load(tmp_path / 'w2_r1_weights.pt')
    assert torch.equal(w0, w1)                                                     # replicas stay bit-identical
