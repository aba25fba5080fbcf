"""torch-CPU fp32 / fp64 restatement of the NAF learn step.  TEST INFRASTRUCTURE ONLY.

The TD targets use oracle.rl_math.ac_td_targets, which tests/test_naf_host.py pins to the reference's own
NAFAgent.learn_from_batch (tests/golden/naf.npz).  The network arithmetic is **parity unpinned** (TensorFlow semantics
restated, see the oracle/nets.py header), in the TF graph's op order:

  network     rl_coach/agents/naf_agent.py:34-43: vector embedder Dense relu layers, FC middleware Dense relu layers
  head        architectures/tensorflow_components/heads/naf_head.py:45-86: V = Dense(1); mu = tanh(Dense(A)) * scale;
              l = Dense(A(A+1)/2) packed column by column into L with an exponentiated diagonal; P = L L^T;
              A = -0.5 d^T (P d), d = u - mu; Q = V + A
  loss        heads/head.py:165-177: mean_b sum l(y, Q), l = squared error or tf.losses.huber_loss (delta 1)
  gradients   architecture.py:193-245: the norm of the unclipped gradients; clip_by_value per tensor or
              clip_by_global_norm; then AdamTF (oracle/nets.py)
  learn step  agents/naf_agent.py:80-99: V of the TARGET network on s', r + (1 - done) * discount * V' in fp64
"""
from collections import OrderedDict

import numpy as np
import torch

from oracle.nets import huber
from oracle.rl_math import ac_td_targets


def unpack_l(lvec, A):
    """naf_head.py:63-73: l [B, A(A+1)/2] -> L [B, A, A]; column c is [0 .. 0, exp(l[i]), l[i+1 .. i+A-c-1]]"""
    columns, i = [], 0
    for col in range(A):
        n = A - col
        zeros = torch.zeros_like(lvec[:, 0:col])
        diag = torch.exp(lvec[:, i]).unsqueeze(1)
        rest = lvec[:, i + 1:i + n]
        columns.append(torch.cat([zeros, diag, rest], dim=1))
        i += n
    return torch.stack(columns, dim=1).transpose(1, 2)


def trunk(params, x, n_layers):
    h = x
    for k in range(n_layers):
        h = torch.relu(h @ params[2 * k] + params[2 * k + 1])
    return h


def naf_forward(params, s, u, scale, n_trunk, A):
    """params: the network's tensors in TF creation order (trunk kernels / biases, V, mu_unscaled, l_vector, rescaler).
    u None: no advantage.  Returns dict(v, mu, l, L, adv, q)."""
    h = trunk(params, s, n_trunk)
    k = 2 * n_trunk
    v = h @ params[k] + params[k + 1]
    mu = torch.tanh(h @ params[k + 2] + params[k + 3]) * scale
    lvec = h @ params[k + 4] + params[k + 5]
    out = dict(v=v, mu=mu, l=lvec)
    if u is not None:
        L = unpack_l(lvec, A)
        P = torch.matmul(L, L.transpose(1, 2))
        d = (u - mu).unsqueeze(-1)
        adv = (-0.5 * torch.matmul(d.transpose(1, 2), torch.matmul(P, d))).reshape(-1, 1)
        out.update(L=L, adv=adv, q=v + adv)
    return out


def target_v(named_target, s2, n_trunk, dtype=torch.float32):
    p = [torch.as_tensor(np.asarray(v)).to(dtype) for v in named_target.values()]
    with torch.no_grad():
        h = trunk(p, torch.as_tensor(np.asarray(s2)).to(dtype), n_trunk)
        return (h @ p[2 * n_trunk] + p[2 * n_trunk + 1]).numpy()


def naf_step(named, named_target, opt, batch, scale, n_trunk, discount=0.99, huber_loss=False, clip=None,
             dtype=torch.float32):
    """One NAFAgent.learn_from_batch.  named / named_target: OrderedDict name -> array (TF order).  batch: dict(states,
    next_states, actions, rewards, game_overs).  clip: None or (method, value).  Returns td_targets, loss, grads (named,
    clipped; raw_grads unclipped), grad_norm (unclipped), new_params (named), mu, q."""
    t = lambda a: torch.as_tensor(np.asarray(a)).to(dtype)      # noqa: E731
    names = list(named.keys())
    params = [t(named[n]).clone().requires_grad_(True) for n in names]
    A = np.asarray(batch["actions"]).shape[1]
    v_next = target_v(named_target, batch["next_states"], n_trunk, dtype)
    y = ac_td_targets(batch["rewards"], batch["game_overs"], v_next, discount)
    y = t(y.astype(np.float32) if dtype == torch.float32 else y)
    sc = t(np.asarray(scale, dtype=np.float32))
    f = naf_forward(params, t(batch["states"]), t(batch["actions"]), sc, n_trunk, A)
    per = huber(f["q"], y) if huber_loss else (y - f["q"]) ** 2
    loss = per.sum(dim=1).mean()
    grads = torch.autograd.grad(loss, params, allow_unused=True)
    grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, params)]
    gnorm = torch.sqrt(sum((g * g).sum() for g in grads))
    raw = OrderedDict(zip(names, [g.detach() for g in grads]))
    if clip is not None:
        method, c = clip
        if method == "ClipByValue":
            grads = [torch.clamp(g, -c, c) for g in grads]
        else:
            grads = [g * (c / max(float(gnorm), c)) for g in grads]
    new_params = opt.step([p.detach() for p in params], grads)
    return dict(td_targets=y.numpy(), v_next=v_next, loss=float(loss.detach()),
                grads=OrderedDict(zip(names, [g.detach() for g in grads])), raw_grads=raw, grad_norm=float(gnorm),
                new_params=OrderedDict(zip(names, new_params)), mu=f["mu"].detach().numpy(),
                q=f["q"].detach().numpy())


def naf_mu(named, states, scale, n_trunk, dtype=torch.float32):
    """mu of the online network (naf_agent.py:107-109)"""
    p = [torch.as_tensor(np.asarray(v)).to(dtype) for v in named.values()]
    with torch.no_grad():
        s = torch.as_tensor(np.asarray(states)).to(dtype)
        return naf_forward(p, s, None, torch.as_tensor(np.asarray(scale, np.float32)).to(dtype), n_trunk, 0)["mu"]\
            .numpy()
