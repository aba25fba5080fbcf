"""CPU restatement of the Quantile Regression DQN learn step.  TEST INFRASTRUCTURE ONLY -- never imported by coach_b200.

  rl_coach/agents/qr_dqn_agent.py:66-137                              q values, target action, TD targets, midpoints
  rl_coach/architectures/tensorflow_components/heads/quantile_regression_q_head.py:33-71   quantile Huber loss

The numpy part (``qr_targets``) is pinned bit for bit against the unmodified reference agent (tests/golden/qr_dqn.npz,
written by oracle/make_golden_qr_dqn.py).  The TensorFlow part (the loss in the graph's op order and its gradient) is
restated in torch for any dtype -- parity unpinned, like oracle/nets.py.
"""
from collections import OrderedDict

import numpy as np
import torch

from oracle.nets import _t


def q_values(quantiles):
    """qr_dqn_agent.py:69-70: np.dot(quantiles, ones(N) / N), fp32 quantiles promoted to fp64"""
    n = quantiles.shape[-1]
    return np.dot(quantiles, np.ones(n) / float(n))


def quantile_midpoints(n):
    """qr_dqn_agent.py:123-124"""
    c = np.array(range(n + 1)) / float(n)
    return 0.5 * (c[1:] + c[:-1])


def qr_targets(next_quantiles, online_quantiles, actions, rewards, game_overs, discount):
    """What learn_from_batch computes between the predictions and the train op (qr_dqn_agent.py:108-129).
    *_quantiles: float32 [B, A, N]; rewards float64 [B]; game_overs [B].  Returns (TD targets float64 [B, N] -- the
    feed rounds them to fp32 --, target actions [B], midpoints float64 [B, N] in the reference's permutation
    tau_i = tau_hat[argsort(row)[i]]).  argsort with kind='stable': the device's tie-break; the reference's default
    kind leaves the order of equal quantiles to the numpy build."""
    B, _, n = next_quantiles.shape
    idx = np.arange(B)
    target_actions = np.argmax(q_values(next_quantiles), axis=1)
    r = np.asarray(rewards, dtype=np.float64)[:, None]
    d = np.asarray(game_overs, dtype=np.float64)[:, None]
    targets = r + (1.0 - d) * discount * next_quantiles[idx, target_actions]
    mid = quantile_midpoints(n)
    order = np.argsort(online_quantiles[idx, np.asarray(actions)], axis=1, kind="stable")
    taus = mid[order]
    return targets, target_actions, taus


def rank_midpoints(online_quantiles, actions):
    """what the paper intends: tau_i = tau_hat[rank(i)] (the inverse permutation) -- for the fixture coverage test"""
    B, _, n = online_quantiles.shape
    order = np.argsort(online_quantiles[np.arange(B), np.asarray(actions)], axis=1, kind="stable")
    return quantile_midpoints(n)[np.argsort(order, axis=1, kind="stable")]


def qr_loss_grad(theta, targets, taus, kappa):
    """quantile_regression_q_head.py:47-62 in the graph's op order, for torch tensors of one dtype.
    theta, targets, taus: [B, N] (the taken action's quantiles, T_j, tau_i).  Returns (loss, d loss / d theta).
    The gradient is TF's: tf.minimum passes it to its first argument on ties (torch.minimum would split it), tf.abs
    has derivative sign(e), so d loss / d theta_i = -(1/N) sum_j |tau_i - [e_ij < 0]| clamp(e_ij, -kappa, kappa)."""
    n = theta.shape[-1]
    k = torch.tensor(kappa, dtype=theta.dtype)
    theta_i = theta.unsqueeze(-1).expand(-1, n, n)
    t_j = targets.unsqueeze(-2).expand(-1, n, n)
    tau_i = taus.unsqueeze(-1).expand(-1, n, n)
    error = t_j - theta_i
    abs_error = error.abs()
    quadratic = torch.minimum(abs_error, k)
    huber = k * (abs_error - quadratic) + 0.5 * quadratic ** 2
    weight = (tau_i - (error < 0).to(theta.dtype)).abs()
    loss = (weight * huber).sum() / float(n)
    grad = -(weight * torch.clamp(error, -k, k)).sum(-1) / float(n)
    return loss, grad


def qr_learn_step(net, online, target, opt, batch, discount, n_actions, atoms, kappa=1.0, clip=None, kink=None,
                  sort_quantiles=None):
    """One learn_from_batch step of QuantileRegressionDQNAgent on a QNetOracle whose head has n_actions * atoms
    outputs.  The gradient of the network parameters is that of the surrogate sum(theta * stop_gradient(dtheta)).
    sort_quantiles (optional, [B, A, N]): the online quantiles whose taken rows decide the midpoints' permutation --
    those of the implementation under test, whose order may differ from this evaluation's where two quantiles lie
    within rounding of each other."""
    names = list(online.keys())
    params = [online[n].clone().requires_grad_(True) for n in names]
    pd = OrderedDict(zip(names, params))
    B = len(batch["actions"])
    with torch.no_grad():
        qn = net.forward(target, batch["next_states"]).reshape(B, n_actions, atoms)
        qo = net.forward(online, batch["states"]).reshape(B, n_actions, atoms)
    order_by = qo.float().numpy() if sort_quantiles is None else np.asarray(sort_quantiles, dtype=np.float32)
    targets, target_actions, taus = qr_targets(qn.float().numpy(), order_by, batch["actions"],
                                               batch["rewards"], batch["game_overs"], discount)
    t32, tau32 = targets.astype(np.float32), taus.astype(np.float32)          # the fp32 feeds
    out = net.forward(pd, batch["states"], kink=kink).reshape(B, n_actions, atoms)
    theta = out[torch.arange(B), torch.as_tensor(np.asarray(batch["actions"]))]
    loss, dtheta = qr_loss_grad(theta.detach(), _t(t32, net.dtype), _t(tau32, net.dtype), kappa)
    surrogate = (theta * dtheta).sum()
    grads = torch.autograd.grad(surrogate, params, allow_unused=True)
    grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, params)]
    gnorm = torch.sqrt(sum((g * g).sum() for g in grads))
    if clip:
        scale = clip / max(float(gnorm), clip)
        grads = [g * scale for g in grads]
    new_params = opt.step([p.detach() for p in params], grads)
    dq = torch.zeros((B, n_actions, atoms), dtype=net.dtype)
    dq[torch.arange(B), torch.as_tensor(np.asarray(batch["actions"]))] = dtheta
    return dict(loss=float(loss), targets=t32, taus=tau32, target_actions=target_actions, dq=dq.reshape(B, -1).numpy(),
                grads=OrderedDict(zip(names, [g.detach() for g in grads])), grad_norm=float(gnorm),
                new_params=OrderedDict(zip(names, new_params)), q_online=q_values(qo.float().numpy()))
