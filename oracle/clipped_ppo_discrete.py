"""Restates discrete ClippedPPO (agents/clipped_ppo_agent.py, heads/ppo_head.py:52-116) for the tests:

  numpy   Categorical.get_action's draw (np.random.choice on host uniforms, the first argmax in evaluation), the
          clipping schedule stepped once per choose_action, and what train_network feeds per minibatch
  torch   the categorical clipped-surrogate head and the whole minibatch step (value MSE + head, global norm, TF Adam),
          in fp32 or fp64

TEST INFRASTRUCTURE ONLY.
"""
from collections import OrderedDict

import numpy as np
import torch

from oracle.actor_critic import mlp


# ---- numpy ---------------------------------------------------------------------------------------------------------------
def choice(probs, u):
    """np.random.choice(len(p), p=p) with the uniform draw u: cdf = cumsum(float64 p), cdf /= cdf[-1], the number of
    entries <= u"""
    cdf = np.asarray(probs, dtype=np.float64).cumsum()
    cdf /= cdf[-1]
    return int(cdf.searchsorted(u, side='right'))


def act(probs, uniforms=None):
    """Categorical.get_action per row of probs [E, A]: the draw on uniforms [E] (training) or the first argmax
    (uniforms None, evaluation)"""
    if uniforms is None:
        return np.array([int(np.argmax(p)) for p in probs], dtype=np.int64)
    return np.array([choice(p, u) for p, u in zip(probs, uniforms)], dtype=np.int64)


def schedule_values(schedule, calls):
    """the schedule's value after each choose_action call (one step per call)"""
    out = []
    for _ in range(calls):
        schedule.step()
        out.append(float(schedule.current_value))
    return np.array(out, dtype=np.float64)


def shuffled_rows(N, B, epochs):
    """the rows of every minibatch of train_network: Batch.shuffle() once per epoch (python's random.shuffle of
    range(N), composed with the previous order), then floor(N / B) slices of B rows -> [epochs * (N // B), B]"""
    import random
    order = list(range(N))
    out = []
    for _ in range(epochs):
        o = list(range(N))
        random.shuffle(o)
        order = [order[i] for i in o]
        out += [order[i * B:(i + 1) * B] for i in range(N // B)]
    return np.array(out, dtype=np.int64)


def minibatch_feeds(rows, actions, old_probs, rescaler):
    """train_network's inputs for one discrete minibatch of the given rows: 1-D actions at output_1_0, the old policy's
    probabilities as the only old-policy input (output_1_1), and the clipping rescaler after it (output_1_2)"""
    return OrderedDict([("output_1_0", np.asarray(actions)[rows]), ("output_1_1", np.asarray(old_probs)[rows]),
                        ("output_1_2", rescaler)])


def clip_bounds(clip_eps, rescaler):
    """TF's 1 -+ eps * rescaler with the fp32 placeholder: every operation in fp32"""
    e = np.float32(np.float32(clip_eps) * np.float32(rescaler))
    return float(np.float32(1) - e), float(np.float32(1) + e)


# ---- torch ---------------------------------------------------------------------------------------------------------------
def head_terms(logits, actions, old_probs, advantages, lo, hi, beta):
    """Categorical(probs=p) with TF 1.x's logits = log p.  Returns (loss, [loss, KL, entropy, ratio, clipped ratio])"""
    B, A = logits.shape
    p = torch.softmax(logits, 1)
    lp = torch.log_softmax(torch.log(p), 1)
    lq = torch.log_softmax(torch.log(old_probs), 1)
    qn = torch.softmax(torch.log(old_probs), 1)
    a = torch.as_tensor(np.asarray(actions), dtype=torch.int64)
    valid = (a >= 0) & (a < A)
    idx = torch.where(valid, a, torch.zeros_like(a))[:, None]
    ratio = torch.exp(lp.gather(1, idx)[:, 0] - lq.gather(1, idx)[:, 0])
    clipped = torch.clamp(ratio, lo, hi)
    zero = torch.zeros_like(ratio)
    surr = torch.where(valid, torch.min(ratio * advantages, clipped * advantages), zero)
    entropy = -(p * lp).sum(1)
    kl = torch.where(qn > 0, qn * (lq - lp), torch.zeros_like(qn)).sum(1)
    loss = -surr.sum() / B - beta * entropy.mean()
    return loss, [loss, kl.mean(), entropy.mean(), torch.where(valid, ratio, zero).sum() / B,
                  torch.where(valid, clipped, zero).sum() / B]


def categorical_head(logits, actions, old_probs, advantages, clip_eps, rescaler, beta, dtype=torch.float64):
    """cb200_ppo_categorical_head: (d_logits [B, A], scalars [5]) as numpy arrays of dtype"""
    t = lambda x: torch.as_tensor(np.asarray(x)).to(dtype)      # noqa: E731
    z = t(logits).requires_grad_(True)
    lo, hi = clip_bounds(clip_eps, rescaler)
    loss, scalars = head_terms(z, actions, t(old_probs), t(advantages), lo, hi, beta)
    (dz,) = torch.autograd.grad(loss, [z])
    return dz.numpy(), np.array([float(s.detach()) for s in scalars])


def minibatch_step(named, opt, mb, clip_eps, rescaler, beta, dtype=torch.float32):
    """one discrete minibatch.  named: OrderedDict of ALL online parameters in creation order:
         v: W0 b0 W1 b1 Wv bv rescaler | p: W0 b0 W1 b1 Wfc bfc rescaler
    mb: dict(states [B, D], actions int64 [B], advantages [B], value_targets [B], old_probs [B, A]).  Returns the loss
    terms, the head's scalars, every gradient, the global norm and the parameters after TF's Adam step."""
    names = list(named.keys())
    params = [torch.as_tensor(named[n]).to(dtype).clone().requires_grad_(True) for n in names]
    v_params, p_params = params[0:6], params[7:13]
    t = lambda a: torch.as_tensor(np.asarray(a)).to(dtype)      # noqa: E731
    states = t(mb["states"])
    v = mlp(v_params, states, ["tanh", "tanh", None])
    value_loss = ((v[:, 0] - t(mb["value_targets"])) ** 2).mean()
    logits = mlp(p_params, states, ["tanh", "tanh", None])
    lo, hi = clip_bounds(clip_eps, rescaler)
    policy_loss, scalars = head_terms(logits, mb["actions"], t(mb["old_probs"]), t(mb["advantages"]), lo, hi, beta)
    grads = torch.autograd.grad(value_loss + policy_loss, params, allow_unused=True)
    grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, params)]
    gnorm = torch.sqrt(sum((g * g).sum() for g in grads))
    new_params = opt.step([p.detach() for p in params], grads)
    return dict(value_loss=float(value_loss.detach()), scalars=np.array([float(s.detach()) for s in scalars]),
                grad_norm=float(gnorm), grads=OrderedDict(zip(names, [g.detach() for g in grads])),
                new_params=OrderedDict(zip(names, new_params)))


def old_probs(named, states, dtype=torch.float32):
    """the frozen target network's softmax over the given states"""
    p = [torch.as_tensor(v).to(dtype) for v in list(named.values())[7:13]]
    with torch.no_grad():
        return torch.softmax(mlp(p, torch.as_tensor(np.asarray(states)).to(dtype), ["tanh", "tanh", None]), 1).numpy()
