"""numpy / torch-CPU restatement of the PPO (KL-penalty) agent, fp32 and fp64.  TEST INFRASTRUCTURE ONLY.

The numpy parts (advantages, minibatch plan, KL coefficient rule, AdditiveNoise draw) are PINNED to the unmodified
reference by tests/golden/ppo.npz (oracle/make_golden_ppo.py); the network arithmetic (head, V loss, gradients, Adam)
restates TensorFlow's semantics, as oracle/actor_critic.py does for ClippedPPO.

Sources restated
  agents/ppo_agent.py:156-195  fill_advantages        agents/ppo_agent.py:197-242  train_value_network
  agents/ppo_agent.py:250-327  train_policy_network   agents/ppo_agent.py:329-353  update_kl_coefficient
  heads/ppo_head.py:52-144     PPOHead (KL penalty, no clipping)   heads/v_head.py: VHead MSE
  exploration_policies/additive_noise.py:84-103  np.random.normal(mean, std)
"""
import math
from collections import OrderedDict

import numpy as np
import torch

from oracle import rl_math as orm
from oracle.actor_critic import EPS, make_adam, mlp, ppo_logp  # noqa: F401  (make_adam re-exported for the tests)

ACTS = ["tanh", "tanh", None]


# ---- numpy prologue (pinned) ----------------------------------------------------------------------------------------
def fill_advantages(rewards, values, game_overs, returns, discount, lam, rescaler):
    """ppo_agent.py:156-195 on complete episodes: values fp32 V(s); GAE per episode with a zero bootstrap, or
    A_VALUE = returns - values in fp64; standardised with np.mean / np.std (population)"""
    if rescaler == "GAE":
        adv, _, n_valid = orm.ppo_fill_advantages(rewards, values, game_overs, discount, lam)
        assert n_valid == len(rewards)
        return adv
    adv = np.asarray(returns, np.float64) - np.asarray(values, np.float32)
    return (adv - np.mean(adv)) / np.std(adv)


def minibatches(n_rows, batch_size, playing_steps):
    """the in-order minibatches of train_value_network / train_policy_network on dataset[:playing_steps]: row ranges
    [i B, (i + 1) B) for i < floor(min(N, playing_steps) / B); the tail is dropped"""
    n = min(n_rows, playing_steps) // batch_size
    return [(i * batch_size, (i + 1) * batch_size) for i in range(n)]


def update_kl_coefficient(k, kl_mean, target):
    """ppo_agent.py:339-351 with the coefficient an fp32 variable"""
    new = np.float32(k)
    if kl_mean > 1.3 * target:
        new *= 1.5
    elif kl_mean < 0.7 * target:
        new /= 1.5
    return np.float32(new)


def normal_action(means, stds, n):
    """np.random.normal(mean, std) on the standard normals n: (double) mean + (double) std * n"""
    return np.asarray(means, np.float32).astype(np.float64) + np.asarray(stds, np.float32).astype(np.float64) * n


# ---- head and minibatch steps (torch) --------------------------------------------------------------------------------
def kl_head_loss(mu, logstd, actions, old_mu, old_logstd, advantages, kl_coef, kl_cutoff, high_kl_penalty, use_kl,
                 beta_entropy):
    """PPOHead without clipping: returns (loss, dict of the logged scalars)"""
    sigma, old_sigma = torch.exp(logstd) + EPS, torch.exp(old_logstd) + EPS
    logp = ppo_logp(mu, logstd, actions)
    logp_old = ppo_logp(old_mu, old_logstd, actions)
    ratio = torch.exp(logp - logp_old)
    surrogate = -(ratio * advantages).mean()
    # KL(old || new) of diagonal Gaussians, summed over the dimensions
    kl = (torch.log(sigma / old_sigma) + (old_sigma ** 2 + (old_mu - mu) ** 2) / (2 * sigma ** 2) - 0.5).sum(1)
    kl_mean = kl.mean()
    k = actions.shape[1]
    entropy = 0.5 * k * (1 + math.log(2 * math.pi)) + torch.log(sigma).sum()
    loss = surrogate - beta_entropy * entropy
    if use_kl:
        loss = loss + kl_coef * kl_mean + high_kl_penalty * torch.clamp(kl_mean - kl_cutoff, min=0) ** 2
    return loss, dict(kl=kl_mean, entropy=entropy, ratio=ratio.mean(), surrogate=surrogate)


def kl_head(mu, logstd, actions, old_mu, old_logstd, advantages, kl_coef, kl_cutoff, high_kl_penalty, use_kl,
            beta_entropy, dtype=torch.float64):
    """the head alone: (d_mu [B, A], d_logstd [A], scalars [loss, KL, entropy, mean ratio, surrogate]) as numpy"""
    t = lambda a: torch.as_tensor(np.asarray(a)).to(dtype)      # noqa: E731
    mu_t, ls_t = t(mu).requires_grad_(True), t(logstd).requires_grad_(True)
    loss, ex = kl_head_loss(mu_t, ls_t, t(actions), t(old_mu), t(old_logstd), t(advantages), float(kl_coef),
                            float(kl_cutoff), float(high_kl_penalty), use_kl, float(beta_entropy))
    g_mu, g_ls = torch.autograd.grad(loss, [mu_t, ls_t])
    scalars = np.array([float(v.detach()) for v in (loss, ex["kl"], ex["entropy"], ex["ratio"], ex["surrogate"])])
    return g_mu.numpy(), g_ls.numpy(), scalars


def _step(named, opt, loss_fn, dtype):
    names = list(named.keys())
    params = [torch.as_tensor(np.asarray(named[n])).to(dtype).clone().requires_grad_(True) for n in names]
    loss, extra = loss_fn(params)
    grads = torch.autograd.grad(loss, params)
    new = opt.step([p.detach() for p in params], grads)
    return dict(loss=float(loss.detach()), grads=OrderedDict(zip(names, [g.detach().numpy() for g in grads])),
                new_params=OrderedDict(zip(names, [p.numpy() for p in new])), **extra)


def critic_step(named, opt, states, targets, dtype=torch.float32):
    """one train_value_network minibatch: V = critic(s), MSE against the fp32-fed returns, Adam"""
    t = lambda a: torch.as_tensor(np.asarray(a)).to(dtype)      # noqa: E731

    def loss_fn(p):
        v = mlp(p[0:6], t(states), ACTS)[:, 0]
        return ((v - t(targets).reshape(-1)) ** 2).mean(), {}
    return _step(named, opt, loss_fn, dtype)


def actor_step(named, old_named, opt, states, actions, advantages, kl_coef, kl_cutoff, high_kl_penalty, use_kl,
               beta_entropy, dtype=torch.float32):
    """one train_policy_network minibatch: the old policy from the target parameters ``old_named``, the KL-penalty
    head, Adam.  named: the actor's parameters in creation order (6 dense tensors, then policy_log_std)."""
    t = lambda a: torch.as_tensor(np.asarray(a)).to(dtype)      # noqa: E731
    old = [t(v) for v in old_named.values()]
    s = t(states)
    with torch.no_grad():
        old_mu = mlp(old[0:6], s, ACTS)

    def loss_fn(p):
        mu = mlp(p[0:6], s, ACTS)
        loss, ex = kl_head_loss(mu, p[6].reshape(-1), t(actions), old_mu, old[6].reshape(-1), t(advantages),
                                float(kl_coef), float(kl_cutoff), float(high_kl_penalty), use_kl, float(beta_entropy))
        return loss, dict(kl=float(ex["kl"].detach()), ratio=float(ex["ratio"].detach()), old_mu=old_mu.numpy())
    return _step(named, opt, loss_fn, dtype)


def values(named, states, dtype=torch.float32):
    t = lambda a: torch.as_tensor(np.asarray(a)).to(dtype)      # noqa: E731
    with torch.no_grad():
        return mlp([t(v) for v in list(named.values())[0:6]], t(states), ACTS)[:, 0].numpy()
