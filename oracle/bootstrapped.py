"""CPU restatement of the Bootstrapped DQN learn step.  TEST INFRASTRUCTURE ONLY -- never imported by coach_b200.

  rl_coach/agents/bootstrapped_dqn_agent.py:57-86            per-head double-DQN targets where the bootstrap mask is set
  rl_coach/architectures/tensorflow_components/general_network.py:304-325
                                                             every head copy reads (1 - r) stop_gradient(x) + r x
  rl_coach/architectures/tensorflow_components/general_network.py:352-360   total loss = sum over the heads
  rl_coach/architectures/tensorflow_components/heads/head.py:170-181        head loss mean_b(sum_a l)

The numpy prologue (``bootstrapped_targets``) is pinned bit for bit against the unmodified reference agent
(tests/golden/bootstrapped.npz, written by oracle/make_golden_bootstrapped.py).  The network part is restated in torch
on oracle.nets.QNetOracle with K * A outputs -- parity unpinned, like oracle/nets.py.
"""
from collections import OrderedDict

import numpy as np
import torch

from oracle.nets import _t, q_head_loss


def bootstrapped_targets(q_next, q_select, q_online, actions, rewards, game_overs, masks, discount):
    """bootstrapped_dqn_agent.py:73-82, the loop verbatim: q_* are lists of K float32 [B, A] arrays (target(s'),
    online(s'), online(s)); masks [B, K].  Returns the K float32 [B, A] TD-target arrays handed to the train op."""
    K = len(q_online)
    targets = [np.array(q, dtype=np.float32, copy=True) for q in q_online]
    for i in range(len(actions)):
        for h in range(K):
            if masks[i][h] == 1:
                selected_action = np.argmax(q_select[h][i], 0)
                targets[h][i, actions[i]] = rewards[i] + (1.0 - game_overs[i]) * discount * q_next[h][i][selected_action]
    return targets


def split_heads(q, K):
    """[B, K A] network output -> list of K [B, A] arrays (head k = columns [k A, (k + 1) A))"""
    q = np.asarray(q)
    A = q.shape[1] // K
    return [np.ascontiguousarray(q[:, k * A:(k + 1) * A]) for k in range(K)]


def _head_names(params):
    kernels = [n for n in params if n.endswith("kernel")]
    w = kernels[-1]
    return w, w[:-len("kernel")] + "bias"


def features(net, params, x, kink=None):
    """the feature layer the heads read: the network evaluated with the head replaced by the identity (exact in any
    precision: every output is one product by 1 plus zeros)"""
    wname, bname = _head_names(params)
    F = params[wname].shape[0]
    p = OrderedDict(params)
    p[wname] = torch.eye(F, dtype=params[wname].dtype)
    p[bname] = torch.zeros(F, dtype=params[bname].dtype)
    return net.forward(p, x, kink=kink)


def bootstrapped_learn_step(net, online, target, opt, batch, discount, K, rescale, huber_loss=True, kink=None):
    """One learn_from_batch step of BootstrappedDQNAgent on a QNetOracle with K * A outputs.  batch: states,
    next_states, actions, rewards, game_overs, masks [B, K].  Returns dict(loss, losses [K], targets [K x [B, A]],
    grads, grad_norm, new_params, q_online / q_next / q_select [B, K A])."""
    names = list(online.keys())
    params = [online[n].clone().requires_grad_(True) for n in names]
    pd = OrderedDict(zip(names, params))
    with torch.no_grad():
        q_next = net.forward(target, batch["next_states"]).numpy()
        q_select = net.forward(online, batch["next_states"]).numpy()
        q_online = net.forward(online, batch["states"]).numpy()
    targets = bootstrapped_targets(split_heads(q_next, K), split_heads(q_select, K), split_heads(q_online, K),
                                   batch["actions"], batch["rewards"], batch["game_overs"], batch["masks"], discount)
    wname, bname = _head_names(pd)
    h = features(net, pd, batch["states"], kink=kink)
    x = (1.0 - rescale) * h.detach() + rescale * h              # general_network.py:321-324
    q = x @ pd[wname] + pd[bname]
    A = q.shape[1] // K
    losses = [q_head_loss(q[:, k * A:(k + 1) * A], _t(targets[k], net.dtype), None, huber_loss) for k in range(K)]
    total = losses[0]
    for l in losses[1:]:
        total = total + l
    grads = torch.autograd.grad(total, params, allow_unused=True)
    grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, params)]
    gnorm = torch.sqrt(sum((g * g).sum() for g in grads))
    new_params = opt.step([p.detach() for p in params], grads)
    return dict(loss=float(total.detach()), losses=[float(l.detach()) for l in losses], targets=targets,
                grads=OrderedDict(zip(names, [g.detach() for g in grads])), grad_norm=float(gnorm),
                new_params=OrderedDict(zip(names, new_params)), q_online=q_online, q_next=q_next, q_select=q_select)
