"""CPU restatement of the Actor-Critic (A3C) agent with continuous actions.  TEST INFRASTRUCTURE ONLY -- never imported
by coach_b200.

  rl_coach/agents/actor_critic_agent.py:127-186         targets and advantages (oracle/a3c.py), the action array fed
  heads/policy_head.py:102-152, heads/head.py:28-33     V | fc_mean | fc_std, tanh(z) * range, softplus(z) + eps,
                                                         MultivariateNormalDiag(mean, std) with its entropy
  exploration_policies/additive_noise.py:62-103         ContinuousEntropy: np.random.normal(mean, std) / the mean

The numpy part (``fed_actions``, ``normal_action``) and the targets are pinned bit for bit against the unmodified
reference (tests/golden/a3c_continuous.npz, written by oracle/make_golden_a3c_continuous.py).  ``learn_step`` restates
the TF part in torch for any dtype (parity unpinned: TensorFlow is not available to pin it).
"""
from collections import OrderedDict

import numpy as np
import torch

from oracle import a3c as oa
from oracle.nets import _t, huber

EPS32 = float(np.finfo(np.float32).eps)
LOG_2PI = float(np.log(2 * np.pi))
SOFTPLUS_THRESHOLD = float(np.log(np.float32(EPS32)) + np.float32(2))


def softplus_tf(x):
    """TF 1.x's softplus: x above -threshold, exp(x) below threshold, log(exp(x) + 1) between"""
    e = torch.exp(x)
    return torch.where(x > -SOFTPLUS_THRESHOLD, x, torch.where(x < SOFTPLUS_THRESHOLD, e, torch.log(e + 1)))


def gaussian_terms(z, actions, max_abs_range):
    """z [n, 1 + 2D] network outputs: (V [n], mean [n, D], std [n, D], log pi(x) [n], H [n])"""
    D = (z.shape[1] - 1) // 2
    rg = torch.as_tensor(np.asarray(max_abs_range, dtype=np.float32)).to(z.dtype)
    mean = torch.tanh(z[:, 1:1 + D]) * rg
    std = softplus_tf(z[:, 1 + D:]) + EPS32
    x = torch.as_tensor(fed_actions(actions, D)).to(z.dtype)
    logp = (-0.5 * ((x - mean) / std) ** 2 - torch.log(std) - 0.5 * LOG_2PI).sum(dim=1)
    ent = (0.5 * (1 + LOG_2PI) + torch.log(std)).sum(dim=1)
    return z[:, 0], mean, std, logp, ent


def fed_actions(actions, D):
    """the action array learn_from_batch feeds: [n, D] (1-D actions get a trailing axis), through the float32
    placeholder"""
    a = np.asarray(actions)
    if a.ndim < 2:
        a = a.reshape(len(a), 1) if D == 1 else a.reshape(-1, D)
    return a.astype(np.float32)


def normal_action(mean, std, n):
    """np.random.normal(mean, std) given its standard normals n: (double) mean + (double) std * n"""
    return np.asarray(mean, np.float32).astype(np.float64) + np.asarray(std, np.float32).astype(np.float64) * \
        np.asarray(n, np.float64)


def learn_step(net, online, opt, segments, discount, mode, max_abs_range, gae_lambda=0.96, beta=0.0, huber_loss=False,
               clip=40.0, v_weight=0.5, p_weight=1.0):
    """One learn step over segments [dict(states, next_states, actions, rewards, game_overs)], as oracle/a3c.py's
    learn_step with the Gaussian policy: loss = mean over the segments of v_weight mean l(V - target) - p_weight
    mean log pi(x) A - beta mean H, its gradient, the global-norm clip, TF Adam.  Returns dict(loss, grads, grad_norm,
    targets, advantages, new_params, z)."""
    names = list(online.keys())
    params = [online[n].clone().requires_grad_(True) for n in names]
    pd = OrderedDict(zip(names, params))
    states = np.concatenate([s["states"] for s in segments])
    with torch.no_grad():
        z0 = net.forward(online, states).numpy()
        boots = net.forward(online, np.stack([s["next_states"][-1] for s in segments])).numpy()[:, 0]
    tg, ad, off = [], [], 0
    for k, s in enumerate(segments):
        L = len(s["rewards"])
        t, a = oa.segment_targets(z0[off:off + L, 0].astype(np.float32), np.float32(boots[k]), s["rewards"],
                                  s["game_overs"], discount, mode, gae_lambda)
        tg.append(t)
        ad.append(a)
        off += L
    targets = np.concatenate(tg).astype(np.float32)
    advantages = np.concatenate(ad).astype(np.float32)
    z = net.forward(pd, states)
    D = (z.shape[1] - 1) // 2
    actions = np.concatenate([fed_actions(s["actions"], D) for s in segments])
    v, _, _, logp, ent = gaussian_terms(z, actions, max_abs_range)
    tt, aa = _t(targets, net.dtype), _t(advantages, net.dtype)
    lv = huber(v, tt) if huber_loss else (v - tt) ** 2
    losses, off = [], 0
    for s in segments:
        sl = slice(off, off + len(s["rewards"]))
        losses.append(v_weight * lv[sl].mean() - p_weight * (logp[sl] * aa[sl]).mean() - beta * ent[sl].mean())
        off += len(s["rewards"])
    loss = torch.stack(losses).mean()
    grads = torch.autograd.grad(loss, params, allow_unused=True)
    grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, params)]
    gnorm = torch.sqrt(sum((g * g).sum() for g in grads))
    if clip:
        scale = clip / max(float(gnorm), clip)
        grads = [g * scale for g in grads]
    new_params = opt.step([p.detach() for p in params], grads)
    return dict(loss=float(loss.detach()), grads=OrderedDict(zip(names, [g.detach() for g in grads])),
                grad_norm=float(gnorm), targets=targets, advantages=advantages,
                new_params=OrderedDict(zip(names, new_params)), z=z0)
