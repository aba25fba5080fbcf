"""CPU restatement of the Policy Gradients (REINFORCE) agent.  TEST INFRASTRUCTURE ONLY -- never imported by coach_b200.

  rl_coach/core_types.py:771-801                       Episode.update_discounted_rewards (n_step = -1)
  rl_coach/agents/policy_gradients_agent.py:47-86      the four return rescalers, the targets fed to the PolicyHead
  rl_coach/agents/policy_optimization_agent.py:58-135  update_episode_statistics (the per-timestep running mean, np.mean
                                                       / np.std of the episode), accumulate, apply every x episodes
  rl_coach/exploration_policies/additive_noise.py      np.random.normal(mean, noise * (high - low)) / the mean
  heads/policy_head.py:54-150                          Categorical(probs = softmax + eps) / MultivariateNormalDiag(
                                                       tanh(z) * range, 1)

The numpy part (``episode_returns``, ``pairwise_sum``, ``mean_std``, ``episode_targets``, ``TimestepTable``,
``additive_noise``) is pinned bit for bit against the unmodified reference (tests/golden/pg.npz, written by
oracle/make_golden_pg.py).  ``episode_grads`` restates the TF part in torch for any dtype, like oracle/a3c.py;
``Learner`` adds the gradient accumulator and TF Adam on apply.
"""
from collections import OrderedDict

import numpy as np
import torch

RESCALERS = ("TOTAL_RETURN", "FUTURE_RETURN", "FUTURE_RETURN_NORMALIZED_BY_EPISODE",
             "FUTURE_RETURN_NORMALIZED_BY_TIMESTEP")
EPS32 = float(np.finfo(np.float32).eps)
LOG_2PI = float(np.log(2 * np.pi))


def episode_returns(rewards, discount):
    """update_discounted_rewards with n_step = -1: out[t] = sum_k discount^k r[t + k], accumulated as the reference
    does (k ascending, a running power of the discount, whole-array numpy adds)"""
    rewards = np.asarray(rewards).astype('float')
    out = rewards.copy()
    d = discount
    for i in range(1, len(rewards)):
        out += d * np.pad(rewards[i:], (0, i), 'constant', constant_values=0)
        d *= discount
    return out


def pairwise_sum(x):
    """numpy's pairwise summation of a contiguous float64 vector (np.add.reduce): below 8 terms a running sum from
    -0.0; up to 128 terms eight accumulators over blocks of 8, folded ((r0 + r1) + (r2 + r3)) + ((r4 + r5) + (r6 + r7)),
    then the tail; above, halves split at n / 2 rounded down to a multiple of 8"""
    x = np.asarray(x, dtype=np.float64)
    n = len(x)
    if n < 8:
        r = np.float64(-0.0)
        for v in x:
            r = r + v
        return r
    if n <= 128:
        acc = x[:8].copy()
        i = 8
        while i < n - n % 8:
            acc = acc + x[i:i + 8]
            i += 8
        r = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]))
        for v in x[i:]:
            r = r + v
        return r
    n2 = n // 2
    n2 -= n2 % 8
    return pairwise_sum(x[:n2]) + pairwise_sum(x[n2:])


def mean_std(R):
    """np.mean / np.std (population) of an episode's returns, spelled out with pairwise_sum"""
    R = np.asarray(R, dtype=np.float64)
    n = np.float64(len(R))
    mean = pairwise_sum(R) / n
    x = R - mean
    return mean, np.sqrt(pairwise_sum(x * x) / n)


class TimestepTable(object):
    """the per-timestep running mean of update_episode_statistics: n_i += 1; m_i -= m_i / n_i; m_i += R_i / n_i"""

    def __init__(self, size):
        self.mean = np.zeros(size)
        self.count = np.zeros(size)

    def fold(self, R):
        """folds one episode's returns; returns the baseline m[:L] right after the fold"""
        for i, r in enumerate(np.asarray(R, dtype=np.float64)):
            self.count[i] += 1
            self.mean[i] -= self.mean[i] / self.count[i]
            self.mean[i] += r / self.count[i]
        return self.mean[:len(R)].copy()


def episode_targets(R, rescaler, table=None):
    """learn_from_batch's rescaled returns (fp64) of one whole episode; the timestep rescaler folds it into ``table``
    first (update_episode_statistics runs before learn_from_batch)"""
    R = np.asarray(R, dtype=np.float64).copy()
    if rescaler == "TOTAL_RETURN":
        R[:] = R[0]
    elif rescaler == "FUTURE_RETURN_NORMALIZED_BY_EPISODE":
        mean, std = mean_std(R)
        R = (R - mean) / std if std != 0 else np.zeros_like(R)
    elif rescaler == "FUTURE_RETURN_NORMALIZED_BY_TIMESTEP":
        R = R - table.fold(R)
    return R


def additive_noise(mean, noise, low, high, z):
    """AdditiveNoise.get_action in training given the standard normals z np.random.normal draws: loc + scale * z in fp64
    with scale = noise * (high - low)"""
    scale = noise * (np.asarray(high) - np.asarray(low))
    return np.asarray(mean, dtype=np.float32).astype(np.float64) + scale * np.asarray(z, dtype=np.float64)


def policy_log_prob_entropy(z, actions, continuous, max_abs_range=None):
    """z [n, N] Dense outputs: (log pi(a) [n], H [n]) of Categorical(probs = softmax + eps) or of
    MultivariateNormalDiag(tanh(z) * range, 1) (its entropy a constant)"""
    if not continuous:
        u = torch.softmax(z, dim=1) + EPS32
        ls = torch.log_softmax(torch.log(u), dim=1)
        a = torch.as_tensor(np.asarray(actions, dtype=np.int64))
        return ls.gather(1, a[:, None])[:, 0], -(u * ls).sum(dim=1)
    D = z.shape[1]
    rg = torch.as_tensor(np.asarray(max_abs_range, dtype=np.float32)).to(z.dtype)
    mu = torch.tanh(z) * rg
    x = torch.as_tensor(np.asarray(actions, dtype=np.float32)).to(z.dtype).reshape(mu.shape)
    logp = -0.5 * ((x - mu) ** 2).sum(dim=1) - 0.5 * D * LOG_2PI
    return logp, torch.full_like(logp, 0.5 * D * (1 + LOG_2PI))


def episode_grads(net, params, episodes, continuous=False, max_abs_range=None, beta=0.0):
    """the summed gradient of the episodes' losses -mean_i(log pi(a_i) t_i) - beta mean_i H_i.  episodes: [dict(states,
    actions, targets)] with the fp32 targets.  Returns (sum of the losses, OrderedDict of gradients)."""
    names = list(params.keys())
    ps = [params[n].clone().requires_grad_(True) for n in names]
    pd = OrderedDict(zip(names, ps))
    loss = 0.0
    for ep in episodes:
        z = net.forward(pd, ep["states"])
        logp, ent = policy_log_prob_entropy(z, ep["actions"], continuous, max_abs_range)
        t = torch.as_tensor(np.asarray(ep["targets"], dtype=np.float32)).to(z.dtype)
        loss = loss - (logp * t).mean() - beta * ent.mean()
    grads = torch.autograd.grad(loss, ps, allow_unused=True)
    grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, ps)]
    return float(loss.detach()), OrderedDict(zip(names, [g.detach() for g in grads]))


class Learner(object):
    """one reference worker's PolicyGradientsAgent.train on whole episodes: returns, the rescaler (with its table),
    accumulate_gradients (a sum), and one TF-Adam step on the sum whenever the episode counter reaches a multiple of
    ``every``"""

    def __init__(self, net, params, opt, rescaler, discount, every, table_size, continuous=False, max_abs_range=None,
                 beta=0.0):
        self.net, self.opt = net, opt
        self.params = OrderedDict((k, v.clone()) for k, v in params.items())
        self.acc = OrderedDict((k, torch.zeros_like(v)) for k, v in params.items())
        self.rescaler, self.discount, self.every = rescaler, discount, every
        self.table = TimestepTable(table_size)
        self.continuous, self.range, self.beta = continuous, max_abs_range, beta
        self.episodes = 0

    def targets(self, rewards):
        return episode_targets(episode_returns(rewards, self.discount), self.rescaler, self.table).astype(np.float32)

    def learn(self, episodes):
        """one learn step of episodes [dict(states, actions, rewards)] that end a part: accumulate, then apply if the
        counter is at a multiple of ``every``.  Returns (loss, applied)."""
        eps = [dict(states=e["states"], actions=e["actions"], targets=self.targets(e["rewards"])) for e in episodes]
        loss, g = episode_grads(self.net, self.params, eps, self.continuous, self.range, self.beta)
        for k in self.acc:
            self.acc[k] = self.acc[k] + g[k]
        self.episodes += len(episodes)
        applied = self.episodes % self.every == 0
        if applied:
            new = self.opt.step(list(self.params.values()), list(self.acc.values()))
            self.params = OrderedDict(zip(self.params.keys(), new))
            self.acc = OrderedDict((k, torch.zeros_like(v)) for k, v in self.acc.items())
        return loss, applied


def split_parts(first_episode, n_closed, every):
    """the episodes that closed at one lock-step, numbered first_episode + 1 .. first_episode + n_closed, cut into
    learn steps: a part ends where the counter reaches a multiple of ``every`` (and at the last episode).  Returns the
    parts' sizes."""
    sizes, cur = [], 0
    for k in range(1, n_closed + 1):
        cur += 1
        if (first_episode + k) % every == 0 or k == n_closed:
            sizes.append(cur)
            cur = 0
    return sizes
