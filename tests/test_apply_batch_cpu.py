"""gcbf_apply_batch (the test-time controller over B graphs in one library call) without a GPU: the workspace query replays the call
without launching, and every argument check runs before any CUDA call."""
import ctypes

import torch

from gcbf_b200 import _C, native, synth
from gcbf_b200.synth import seeded_algo

OK = 0x7f0000000000          # aligned, never dereferenced: the calls below fail their checks first


def _desc(cfg='C1'):
    c = dict(synth.CONFIGS[cfg])
    sb = synth.make_states(c['env'], c['num_agents'], c['num_obs'], 1, c['area_size'], 1)
    env, algo = seeded_algo(sb.env, sb.num_agents, torch.device('cpu'), 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    env.set_goal(sb.goals)
    return sb, env, algo._step_desc()[0]


def _batch(env, sb, d, B, E):
    cfg_s = env._cfg(B)
    ctypes.memmove(ctypes.byref(d.env), ctypes.byref(cfg_s), ctypes.sizeof(_C.EnvCfg))
    b = native.StepBatch()
    fake = 1 << 20
    b.states, b.ld_state, b.x, b.edge_attr, b.edge_index, b.rowptr, b.u_ref = fake, env.state_dim, fake, fake, fake, fake, fake
    b.row_index = fake if sb.num_obs else None
    b.num_edges, b.num_nodes, b.num_agents_total = E, B * sb.nodes_per_graph, B * sb.num_agents
    return b


def _need(d, b):
    return native.fn('gcbf_apply_batch_workspace_bytes')(ctypes.byref(d), ctypes.byref(b))


def test_apply_batch_workspace_grows_with_graphs_and_edges_and_c3_fits():
    sb, env, d = _desc('C1')
    one = _need(d, _batch(env, sb, d, 1, 300))
    assert one > 0, _C.lib().gcbf_last_error()
    # the one-graph case is gcbf_apply's workspace
    assert native.fn('gcbf_apply_workspace_bytes')(ctypes.byref(d), ctypes.byref(_batch(env, sb, d, 1, 300))) == one
    many = _need(d, _batch(env, sb, d, 256, 300 * 256))
    more_edges = _need(d, _batch(env, sb, d, 256, 600 * 256))
    assert one < many < more_edges
    sb3, env3, d3 = _desc('C3')
    c3 = _need(d3, _batch(env3, sb3, d3, 64, 206139))
    assert 0 < c3 < 80e9, c3


def test_apply_batch_argument_checks_run_before_any_cuda_call():
    sb, env, d = _desc('C1')
    B = 4
    b = _batch(env, sb, d, B, 300 * B)
    need = _need(d, b)
    call = native.fn('gcbf_apply_batch')
    it = ctypes.c_int(0)
    err = lambda: _C.lib().gcbf_last_error().decode()      # noqa: E731

    def run(b_=b, rand=0.0, noise=None, rounds=OK, ws=OK, nbytes=None, ld=2):
        return call(ctypes.byref(d), ctypes.byref(b_), 0.1, rand, noise, 30, OK, ld, rounds, ctypes.byref(it), ws,
                    need if nbytes is None else nbytes, None)

    assert run(rand=30.0) == -1 and 'noise' in err()                       # rand without noise
    assert run(rounds=None) == -1 and 'rounds' in err()                   # no per-graph round counts
    assert run(ws=OK + 8) == -1 and 'bad arguments' in err()              # misaligned workspace
    assert run(ld=1) == -1                                                 # pitch < action_dim
    assert run(nbytes=1024) == native.E_WORKSPACE and 'too small' in err()
    bad = _batch(env, sb, d, B, 300 * B)
    bad.num_agents_total -= 1                                              # num_agents_total != num_graphs * num_agents
    assert run(b_=bad) == -1 and 'batch sizes' in err()
    bad = _batch(env, sb, d, B, 300 * B)
    bad.num_nodes += 1                                                     # num_nodes != num_graphs * nodes_per_graph
    assert run(b_=bad) == -1 and 'batch sizes' in err()
    # both goal modes are accepted: with per-graph goals the same checks pass up to the (too small) workspace
    for per_graph in (0, 1):
        d.goal_per_graph = per_graph
        assert _need(d, b) == need
        assert run(nbytes=1024) == native.E_WORKSPACE
    d.goal_per_graph = 0
    # gcbf_apply keeps refusing more than one graph
    assert native.fn('gcbf_apply')(ctypes.byref(d), ctypes.byref(b), 0.1, 0.0, None, 30, OK, 2, ctypes.byref(it), OK, need, None) == -1
    assert 'one graph' in err()
