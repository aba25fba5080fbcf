"""CPU restatement of the Actor-Critic (A3C) agent, discrete actions.  TEST INFRASTRUCTURE ONLY -- never imported by
coach_b200.

  rl_coach/agents/actor_critic_agent.py:95-165           A_VALUE / GAE targets and advantages (numpy, scipy.signal.lfilter)
  rl_coach/exploration_policies/categorical.py:36-47     np.random.choice(A, p=p) / argmax
  heads/v_head.py, heads/policy_head.py, heads/head.py   VHead (loss weight 0.5) + PolicyHead (1.0, entropy beta)

The numpy part (``segment_targets``, ``categorical_choice``) is pinned bit for bit against the unmodified reference agent
(tests/golden/a3c.npz, written by oracle/make_golden_a3c.py).  ``learn_step`` restates the TF part in torch for any
dtype, like oracle/nets.py: the shared-trunk network, the three loss terms with tf Categorical(probs = p + eps)
semantics (parity unpinned: TensorFlow is not available to pin it), autograd, the global-norm clip and TF Adam.
"""
from collections import OrderedDict

import numpy as np
import torch

from oracle.nets import _t, huber

EPS32 = float(np.finfo(np.float32).eps)


def _lfilter_step(x, z, c):
    """one step of scipy.signal.lfilter([1], [1, -c]) as its C loop evaluates it: y = z + 1 * x; z' = x * 0 - y * (-c)"""
    y = np.float64(z) + np.float64(x)
    return y, np.float64(x) * 0.0 - y * np.float64(-c)


def segment_targets(values, boot, rewards, game_overs, discount, mode, gae_lambda=0.96):
    """learn_from_batch's targets of one segment (actor_critic_agent.py:111-150).  values float32 [L] = V(s_i); boot =
    V(last s') float32 (ignored when the last game_over is set); mode "A_VALUE", "GAE" or "GAE_VALUE"
    (estimate_state_value_using_gae).  Returns (V targets float64 [L], advantages float64 [L]), before TF's fp32 feed.
    Spelled out: A_VALUE's first step after a bootstrap and every GAE discount * value are numpy 2's python float *
    float32 = fp32 products; every other operation is fp64."""
    values = np.asarray(values, dtype=np.float32)
    L = len(values)
    terminal = bool(game_overs[-1])
    g32 = np.float32(discount)
    targets, adv = np.zeros(L), np.zeros(L)
    if mode == "A_VALUE":
        R, fp32_step = (np.float64(0.0), False) if terminal else (np.float32(boot), True)
        for i in reversed(range(L)):
            prod = np.float64(g32 * np.float32(R)) if fp32_step else np.float64(discount) * R
            R = np.float64(rewards[i]) + prod
            fp32_step = False
            targets[i] = R
            adv[i] = R - np.float64(values[i])
        return targets, adv
    vnext = np.float32(0.0) if terminal else np.float32(boot)
    gl = discount * gae_lambda
    _, zr = _lfilter_step(vnext, 0.0, discount)
    za = 0.0
    for i in reversed(range(L)):
        delta = (np.float64(rewards[i]) + np.float64(g32 * vnext)) - np.float64(values[i])
        adv[i], za = _lfilter_step(delta, za, gl)
        ret, zr = _lfilter_step(rewards[i], zr, discount)
        targets[i] = adv[i] + np.float64(values[i]) if mode == "GAE_VALUE" else ret
        vnext = values[i]
    return targets, adv


def categorical_choice(p, u):
    """np.random.choice(len(p), p=p) given its uniform u: cdf = cumsum(float64(p)), cdf /= cdf[-1], searchsorted right"""
    cdf = np.cumsum(np.asarray(p, dtype=np.float64))
    cdf /= cdf[-1]
    return int(np.searchsorted(cdf, u, side="right"))


def policy_terms(z, actions, dtype):
    """z [n, 1 + A] network outputs: (V [n], p [n, A], log pi(a) [n], H [n]) with Categorical(probs = p + eps)"""
    v, logits = z[:, 0], z[:, 1:]
    p = torch.softmax(logits, dim=1)
    u = p + EPS32
    ls = torch.log_softmax(torch.log(u), dim=1)
    a = torch.as_tensor(np.asarray(actions, dtype=np.int64))
    logp = ls.gather(1, a[:, None])[:, 0]
    return v, p, logp, -(u * ls).sum(dim=1)


def learn_step(net, online, opt, segments, discount, mode, gae_lambda=0.96, beta=0.0, huber_loss=False, clip=40.0,
               v_weight=0.5, p_weight=1.0, kink=None):
    """One learn step over segments [dict(states, next_states, actions, rewards, game_overs)], concatenated in order:
    targets and advantages of segment_targets on this network's own V values (fed as fp32), loss = mean over the
    segments of v_weight mean l(V - target) - p_weight mean log pi(a) A - beta mean H, its gradient, the global-norm
    clip, TF Adam.  Returns dict(loss, grads, grad_norm, targets, advantages, new_params, z)."""
    names = list(online.keys())
    params = [online[n].clone().requires_grad_(True) for n in names]
    pd = OrderedDict(zip(names, params))
    states = np.concatenate([s["states"] for s in segments])
    with torch.no_grad():
        z0 = net.forward(online, states).numpy()
        boots = net.forward(online, np.stack([s["next_states"][-1] for s in segments])).numpy()[:, 0]
    tg, ad, off = [], [], 0
    for k, s in enumerate(segments):
        L = len(s["actions"])
        t, a = segment_targets(z0[off:off + L, 0].astype(np.float32), np.float32(boots[k]), s["rewards"],
                               s["game_overs"], discount, mode, gae_lambda)
        tg.append(t)
        ad.append(a)
        off += L
    targets = np.concatenate(tg).astype(np.float32)
    advantages = np.concatenate(ad).astype(np.float32)
    z = net.forward(pd, states, kink=kink)
    v, _, logp, ent = policy_terms(z, np.concatenate([s["actions"] for s in segments]), net.dtype)
    tt, aa = _t(targets, net.dtype), _t(advantages, net.dtype)
    lv = huber(v, tt) if huber_loss else (v - tt) ** 2
    losses, off = [], 0
    for s in segments:
        sl = slice(off, off + len(s["actions"]))
        losses.append(v_weight * lv[sl].mean() - p_weight * (logp[sl] * aa[sl]).mean() - beta * ent[sl].mean())
        off += len(s["actions"])
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
