"""TEST INFRASTRUCTURE ONLY -- CPU oracle of one analytic-h_dot train step (GCBF.params['h_dot'] = 'analytic'): gcbf_oracle.update_step
with h_dot = J_h(s) . f(s, clamp(actions + u_ref(s))) from an autograd JVP through the port (double backward, create_graph=True: the loss is
differentiated through it) and ONE spectral-norm power iteration, in place of the finite difference.

There is no reference implementation of this loss; what pins the oracle is tests/test_hdot_train_cpu.py: its gradient against a float64
central finite difference of its own total loss."""
from typing import Dict, Optional

import torch

import gcbf_oracle as O
import jvp_oracle as JO

Tensor = torch.Tensor


def analytic_losses(env: str, cbf_sd: Dict[str, Tensor], actor_sd: Dict[str, Tensor], states: Tensor, goal: Tensor, edge_index: Tensor,
                    u_ref_stored: Tensor, num_graphs: int, num_agents: int, num_obs: int, hp: dict, K: Optional[Tensor] = None,
                    freeze: Optional[bool] = None) -> dict:
    """Forward of the analytic step as a differentiable function of the two state dicts (advances the CBF's u, v once)."""
    N = num_agents + num_obs
    x, agent_mask = O.make_graph_inputs(env, states, num_graphs, num_agents, num_obs)
    x = x.to(states.dtype)
    eps, alpha = hp['eps'], hp['alpha']
    s = states.detach().clone().requires_grad_(True)
    h = O.cbf_forward(cbf_sd, x, O.edge_attr(env, s, edge_index), edge_index, agent_mask)             # the one power iteration
    actions = O.actor_forward(actor_sd, x, O.edge_attr(env, states, edge_index), edge_index, agent_mask, u_ref_stored.to(states.dtype))
    sdot = JO.closed_loop_state_dot(env, states, goal, actions, num_graphs, num_agents, num_obs, K, freeze)
    if edge_index.shape[1] == 0:
        h_dot = torch.zeros_like(h)                      # h depends on the states only through the edge features
    else:
        w = torch.zeros_like(h, requires_grad=True)
        (g,) = torch.autograd.grad(h, s, grad_outputs=w, create_graph=True)
        (h_dot,) = torch.autograd.grad(g, w, grad_outputs=sdot, create_graph=True)   # J_h(s) . sdot, differentiable in params and sdot
    um = O.unsafe_mask(env, states, num_graphs, N, num_agents)
    sm = O.safe_mask(env, states, num_graphs, N, num_agents)
    hu, hs = h[um], h[sm]
    zero, one = torch.zeros((), dtype=h.dtype), torch.ones((), dtype=h.dtype)
    loss_unsafe = torch.mean(torch.relu(hu + eps)) if hu.numel() else zero
    acc_unsafe = torch.mean(torch.less(hu, 0).type_as(hu)) if hu.numel() else one
    loss_safe = torch.mean(torch.relu(-hs + eps)) if hs.numel() else zero
    acc_safe = torch.mean(torch.greater_equal(hs, 0).type_as(hs)) if hs.numel() else one
    hf, hd = h.reshape(-1), h_dot.reshape(-1)
    loss_h_dot = torch.mean(torch.relu(-hd - alpha * hf + eps))
    loss_action = torch.mean(torch.square(actions).sum(dim=1))
    loss = (hp['loss_unsafe_coef'] * loss_unsafe + hp['loss_safe_coef'] * loss_safe + hp['loss_h_dot_coef'] * loss_h_dot +
            hp['loss_action_coef'] * loss_action)
    return dict(h=h, actions=actions, h_dot=h_dot, sdot=sdot, loss_unsafe=loss_unsafe, loss_safe=loss_safe, loss_h_dot=loss_h_dot,
                loss_action=loss_action, loss=loss, acc_unsafe=acc_unsafe, acc_safe=acc_safe, unsafe_mask=um, safe_mask=sm)


def analytic_update_step(env: str, cbf_sd: Dict[str, Tensor], actor_sd: Dict[str, Tensor], opt_cbf: dict, opt_actor: dict, states: Tensor,
                         goal: Tensor, edge_index: Tensor, u_ref_stored: Tensor, num_graphs: int, num_agents: int, num_obs: int,
                         hp: Optional[dict] = None, K: Optional[Tensor] = None, apply_optim: bool = True, freeze: Optional[bool] = None) -> dict:
    """gcbf_oracle.update_step with the analytic h_dot.  Mutates cbf_sd / actor_sd (weights, u / v) and the two Adam states in place;
    returns h, actions, h_dot, the four losses, the accuracies, the raw (pre-clip) gradients of both nets."""
    hp = O.HYPERPARAMS[env] if hp is None else hp
    cbf_p = {k: cbf_sd[k].requires_grad_(True) for k in O.trainable_keys(cbf_sd)}
    act_p = {k: actor_sd[k].requires_grad_(True) for k in O.trainable_keys(actor_sd)}
    r = analytic_losses(env, cbf_sd, actor_sd, states, goal, edge_index, u_ref_stored, num_graphs, num_agents, num_obs, hp, K, freeze)
    plist = list(cbf_p.values()) + list(act_p.values())
    glist = torch.autograd.grad(r['loss'], plist, allow_unused=True)
    gl = [g if g is not None else torch.zeros_like(p) for g, p in zip(glist, plist)]
    cbf_g = dict(zip(cbf_p.keys(), gl[:len(cbf_p)]))
    act_g = dict(zip(act_p.keys(), gl[len(cbf_p):]))
    for d in (cbf_sd, actor_sd):
        for k in d:
            d[k].requires_grad_(False)
    raw = dict(cbf={k: v.clone() for k, v in cbf_g.items()}, actor={k: v.clone() for k, v in act_g.items()})
    O.clip_grad_norm(cbf_g, 1e-3)
    O.clip_grad_norm(act_g, 1e-3)
    if apply_optim:
        with torch.no_grad():
            O.adam_step({k: cbf_sd[k] for k in cbf_g}, cbf_g, opt_cbf, lr=3e-4)
            O.adam_step({k: actor_sd[k] for k in act_g}, act_g, opt_actor, lr=1e-3)
    hd = r['h_dot'].detach()
    out = {k: (v.detach() if torch.is_tensor(v) else v) for k, v in r.items()}
    out['acc_h_dot'] = O.acc_h_dot_broadcast(hd.reshape(-1), r['h'].detach(), hp['alpha'])
    out['raw_grads'] = raw
    return out
