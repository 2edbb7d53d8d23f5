"""GPU test of the analytic h_dot (SURVEY 8f-3; gcbf_b200/jvp.py + csrc/jvp.cu) against the CPU oracle (oracle/jvp_oracle.py: autograd
JVP through the GCBF port, itself pinned against a float64 finite difference in tests/test_jvp_cpu.py)."""
import pytest
import torch

import gcbf_oracle as O
import jvp_oracle as JO
from helpers import oracle_batch, product_batch, sd_clone, seeded_algo

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')

CASES = [('DubinsCar', 12, 3, 2, 2.0, 31, False), ('SimpleCar', 10, 0, 3, 1.5, 32, False), ('SimpleDrone', 6, 6, 2, 0.9, 33, False),
         ('DubinsCar', 12, 3, 1, 2.0, 34, True), ('DubinsCar', 64, 8, 4, 3.0, 7, False)]      # the last one engages the tensor-core layers


@pytest.mark.parametrize('env_name,n,obs,B,area,seed,on_goal', CASES)
def test_h_dot_analytic_matches_the_oracle(env_name, n, obs, B, area, seed, on_goal):
    from gcbf_b200 import synth
    sb = synth.make_states(env_name, n, obs, B, area, seed)
    if on_goal:
        pd = O.ENV_PARAMS[env_name]['pos_dim']
        sb.states[1, :pd] = sb.goals[1, :pd]                    # frozen agent of the single-graph branch
    env, algo = seeded_algo(env_name, n, DEV, 0, {'num_obs': sb.num_obs, 'area_size': sb.area_size})
    data = product_batch(env, sb, DEV)
    ob = oracle_batch(sb)
    assert torch.equal(data.edge_index.cpu(), ob['edge_index'])
    cbf = sd_clone(algo.cbf)
    g = torch.Generator().manual_seed(seed)
    action = torch.randn(B * n, O.ENV_PARAMS[env_name]['action_dim'], generator=g) * 0.3
    want_h, want_hd, want_sd = JO.h_and_h_dot(env_name, cbf, sb.states, sb.goals, ob['edge_index'], action, B, n, sb.num_obs, K=ob['K'])
    from gcbf_b200 import jvp
    sdot = jvp.state_dot(env, data, action.to(DEV))
    assert torch.allclose(sdot.cpu(), want_sd, rtol=1e-5, atol=1e-5)
    h, h_dot = algo.h_dot_analytic(data, action.to(DEV))
    torch.cuda.synchronize()
    assert float((h.cpu() - want_h).abs().max()) <= 1e-5
    scale = float(want_hd.abs().max())
    assert float((h_dot.cpu() - want_hd).abs().max()) <= 1e-4 * scale + 1e-6, (float((h_dot.cpu() - want_hd).abs().max()), scale)
