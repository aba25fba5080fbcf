"""CPU restatement of the N-step Q-learning agent.  TEST INFRASTRUCTURE ONLY -- never imported by coach_b200.

  rl_coach/agents/n_step_q_agent.py:99-140              segment targets, both horizons (numpy)
  rl_coach/agents/policy_optimization_agent.py:85-135   segment cuts; n_step_q_agent.py:142-153 target copy first
  rl_coach/agents/agent.py:640-660, 820-834             target-copy cadence, one env step per act()

The numpy part (``segment_targets``, ``schedule``) is pinned bit for bit against the unmodified reference agent
(tests/golden/nstep_q.npz, written by oracle/make_golden_nstep_q.py).  ``learn_step`` restates the TF part (MSE / Huber
head loss of each segment, the mean over the segments' gradients, TF Adam) in torch for any dtype, like oracle/nets.py.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F

from oracle.nets import QNetOracle, _t, huber


def segment_targets(q_online, actions, rewards, game_overs, discount, horizon, q_next=None):
    """learn_from_batch's targets of one segment (n_step_q_agent.py:104-127).  q_online float32 [L, A]; q_next float32
    [L, A] = Q_target(s'_i) (N-Step reads its last row only); rewards float64 or int64 [L].  Returns (targets float32
    [L, A], bootstrap: N-Step the fp32 max of Q_target(last s') or 0.0 when the segment ends in a terminal state,
    1-Step [L] the row-wise maxima).  Spelled out: the first step after a bootstrap is numpy 2's python float *
    np.float32 = an fp32 product; every other operation is fp64."""
    targets = np.array(q_online, dtype=np.float32, copy=True)
    L = len(actions)
    if horizon == "1-Step":
        boot = np.max(np.asarray(q_next, dtype=np.float32), axis=1)
        for i in reversed(range(L)):
            not_done = 1.0 - float(bool(game_overs[i]))
            targets[i, actions[i]] = np.float64(rewards[i]) + not_done * discount * np.float64(boot[i])
        return targets, boot
    if horizon != "N-Step":
        return targets, None                                  # `assert True`: nothing is replaced
    if game_overs[-1]:
        R, boot, fp32_step = np.float64(0.0), np.float32(0.0), False
    else:
        boot = np.max(np.asarray(q_next, dtype=np.float32)[-1])
        R, fp32_step = boot, True
    for i in reversed(range(L)):
        prod = np.float64(np.float32(discount) * np.float32(R)) if fp32_step else np.float64(discount) * R
        R = np.float64(rewards[i]) + prod
        fp32_step = False
        targets[i, actions[i]] = R
    return targets, boot


def schedule(episode_lengths, t_max, copy_method, copy_steps):
    """One stream through NStepQAgent.train after every env step.  Returns (segments [(start, end, env step)] in
    episode coordinates, target-copy env steps, training_iteration)."""
    total = training_iteration = last_copy = 0
    segments, copies = [], []
    for n in episode_lengths:
        length = last = 0
        for k in range(n):
            total += 1
            length += 1
            complete = k == n - 1
            counter = training_iteration if copy_method == "TrainingSteps" else total
            if counter - last_copy >= copy_steps:
                last_copy = counter
                copies.append(total)
            passed = length - last
            if passed >= t_max or complete:
                if passed > 0:
                    segments.append((last, length, total))
                    training_iteration += 1
                last = 0 if complete else length
    return segments, copies, training_iteration


def lockstep_schedule(done, t_max):
    """E streams in lock step, done [steps, E] game_over flags: the segments each train() closes,
    [(step, [(stream, rows)])] -- the per-stream rule of ``schedule`` applied to every stream at each step"""
    steps, E = done.shape
    length = np.zeros(E, dtype=np.int64)
    last = np.zeros(E, dtype=np.int64)
    out = []
    for t in range(steps):
        length += 1
        closed = []
        for e in range(E):
            passed = length[e] - last[e]
            if passed >= t_max or done[t, e]:
                closed.append((e, int(passed)))
                last[e] = 0 if done[t, e] else length[e]
                if done[t, e]:
                    length[e] = 0
        out.append((t, closed))
    return out


class NStepQNetOracle(QNetOracle):
    """QNetOracle with an explicit embedder scheme: ``strides`` of the convolutions (images) or the number of dense
    embedder layers (vectors), and the middleware layer count (0 or 1)"""

    def __init__(self, observation_shape, num_actions, dtype=torch.float32, strides=(4, 2, 1), n_embed=1,
                 middleware=True):
        super().__init__(observation_shape, num_actions, False, dtype, middleware)
        self.strides, self.n_embed = tuple(strides), int(n_embed)

    def forward(self, params, x, kink=None):
        p = list(params.values())
        h = torch.as_tensor(x).to(self.dtype)
        masks = [] if kink is None else kink["masks"]
        n = [0]

        def relu(z):
            i = n[0]
            n[0] += 1
            if i >= len(masks) or masks[i] is None:
                return F.relu(z)
            own = z > 0
            other = masks[i].to(torch.bool).reshape(z.shape)
            near = z.detach().abs() <= kink["tol"] * z.detach().abs().max()
            m = torch.where(near, other, own)
            kink["flipped"] = kink.get("flipped", 0) + int((m != own).sum())
            kink["hard"] = kink.get("hard", 0) + int(((other != own) & ~near).sum())
            return z * m.to(z.dtype)

        k = 0
        if self.is_image:
            h = (h / 255.0).permute(0, 3, 1, 2)
            for stride in self.strides:
                h = relu(F.conv2d(h, p[k].permute(3, 2, 0, 1), p[k + 1], stride=stride))
                k += 2
            h = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)
        else:
            for _ in range(self.n_embed):
                h = relu(h @ p[k] + p[k + 1])
                k += 2
        if self.middleware:
            h = relu(h @ p[k] + p[k + 1])
            k += 2
        return h @ p[k] + p[k + 1]


def learn_step(net, online, target, opt, segments, discount, horizon, huber_loss=False, kink=None):
    """One learn step over segments [dict(states, next_states, actions, rewards, game_overs)], concatenated in order:
    the targets of segment_targets on this network's own Q values, loss = mean over segments of the segment's mean over
    rows of sum_a l, its gradient, TF Adam.  Returns dict(loss, grads, grad_norm, targets, new_params, q_online)."""
    names = list(online.keys())
    params = [online[n].clone().requires_grad_(True) for n in names]
    pd = OrderedDict(zip(names, params))
    states = np.concatenate([s["states"] for s in segments])
    with torch.no_grad():
        q_online = net.forward(online, states).numpy()
        q_next = net.forward(target, np.concatenate([s["next_states"] for s in segments])).numpy()
    tg, off = [], 0
    for s in segments:
        L = len(s["actions"])
        t, _ = segment_targets(np.asarray(q_online[off:off + L], dtype=np.float32), s["actions"], s["rewards"],
                               s["game_overs"], discount, horizon, np.asarray(q_next[off:off + L], dtype=np.float32))
        tg.append(t)
        off += L
    targets = np.concatenate(tg)
    q = net.forward(pd, states, kink=kink)
    tt = _t(targets, net.dtype)
    per_row = (huber(q, tt) if huber_loss else (q - tt) ** 2).sum(dim=1)
    losses, off = [], 0
    for s in segments:
        L = len(s["actions"])
        losses.append(per_row[off:off + L].mean())
        off += L
    loss = torch.stack(losses).mean()
    grads = torch.autograd.grad(loss, params, allow_unused=True)
    grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, params)]
    gnorm = torch.sqrt(sum((g * g).sum() for g in grads))
    new_params = opt.step([p.detach() for p in params], grads)
    return dict(loss=float(loss.detach()), grads=OrderedDict(zip(names, [g.detach() for g in grads])),
                grad_norm=float(gnorm), targets=targets, new_params=OrderedDict(zip(names, new_params)),
                q_online=q_online)
