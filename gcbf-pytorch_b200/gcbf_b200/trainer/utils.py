"""Host-side helpers with the names the reference's scripts import from gcbf/trainer/utils.py."""
import os
import random
from typing import Optional

import numpy as np
import torch

# gcbf/trainer/hyperparams.yaml (gcbf rows)
_HYPERPARAMS = {
    'SimpleCar': dict(alpha=1.0, eps=0.02, inner_iter=10, loss_action_coef=0.05, loss_unsafe_coef=1.0,
                      loss_safe_coef=1.0, loss_h_dot_coef=0.5),
    'SimpleDrone': dict(alpha=1.0, eps=0.02, inner_iter=10, loss_action_coef=0.05, loss_unsafe_coef=1.0,
                        loss_safe_coef=1.0, loss_h_dot_coef=0.5),
    'DubinsCar': dict(alpha=1.0, eps=0.02, inner_iter=10, loss_action_coef=0.0001, loss_unsafe_coef=1.0,
                      loss_safe_coef=1.0, loss_h_dot_coef=0.2),
}


def set_seed(seed: int):
    """reference gcbf/trainer/utils.py:20-25"""
    random.seed(seed)
    np.random.seed(seed)
    torch.manual_seed(seed)
    torch.cuda.manual_seed_all(seed)


# gcbf/trainer/hyperparams.yaml (macbf rows): only the action and h_dot coefficients differ from the gcbf rows
_MACBF_COEFS = {'SimpleCar': (0.0001, 1.0), 'SimpleDrone': (0.01, 1.0), 'DubinsCar': (0.0005, 1.0)}


def read_params(env: str, algo: str) -> Optional[dict]:
    """reference gcbf/trainer/utils.py:317-340 (per-env hyper-parameter table)."""
    if algo not in ('gcbf', 'macbf') or env not in _HYPERPARAMS:
        return None
    hp = dict(_HYPERPARAMS[env])
    if algo == 'macbf':
        hp['loss_action_coef'], hp['loss_h_dot_coef'] = _MACBF_COEFS[env]
    return hp


def init_logger(log_path: str, env: str, algo: str, seed: int, args: dict = None, hyper_params: dict = None) -> str:
    """Creates <log_path>/<env>/<algo>/seed<seed>_<k>/ and writes settings.yaml (reference utils.py:28-105)."""
    import datetime
    import yaml
    base = os.path.join(log_path, env, algo)
    os.makedirs(base, exist_ok=True)
    stamp = datetime.datetime.now().strftime('%Y%m%d%H%M%S')
    run = os.path.join(base, f'seed{seed}_{stamp}')
    os.makedirs(run, exist_ok=True)
    with open(os.path.join(run, 'settings.yaml'), 'w') as f:
        yaml.safe_dump({**(args or {}), 'hyper_params': hyper_params or {}}, f)
    return run


def cbf_contour_data(cbf_algo, data, env, agent_id: int, x_dim: int, y_dim: int, attention: bool = True, n_mesh: int = 30,
                     condition: bool = False) -> dict:
    """What the reference's plot_cbf_contour (gcbf/trainer/utils.py:226-298) plots, without plotting: the meshgrids `x`, `y`
    [n_mesh, n_mesh] of env.state_lim along (x_dim, y_dim), the learned CBF `cbf` [n_mesh, n_mesh] of agent `agent_id` on them
    (cbf[i, j] at (x[i, j], y[i, j]); GCBF.cbf_field, one library call) and, with `attention`, the attention weights [E, 1] of
    `data` (cbf.attention, utils.py:292-293).  Its zero level set is the learned safe-set boundary.  With `condition`, also
    `h_dot` and `condition` = h_dot + alpha * cbf [n_mesh, n_mesh] under the learned controller (GCBF.cbf_condition_field; alpha =
    cbf_algo.params['alpha']): the certificate holds where condition >= 0."""
    if condition:
        xs, ys, h, h_dot = cbf_algo.cbf_condition_field(data, agents=int(agent_id), x_dim=x_dim, y_dim=y_dim, n_mesh=n_mesh,
                                                        lims=env.state_lim)
    else:
        xs, ys, h = cbf_algo.cbf_field(data, agents=int(agent_id), x_dim=x_dim, y_dim=y_dim, n_mesh=n_mesh, lims=env.state_lim)
    x, y = np.meshgrid(xs, ys)
    out = dict(x=x, y=y, cbf=h[0, 0].detach().cpu())
    if condition:
        out['h_dot'] = h_dot[0, 0].detach().cpu()
        out['condition'] = out['h_dot'] + float(cbf_algo.params['alpha']) * out['cbf']
    if attention:
        out['attention'] = cbf_algo.cbf.attention(data)
    return out
