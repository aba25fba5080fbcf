"""CPU restatement of the PAL and Mixed Monte Carlo target prologues.  TEST INFRASTRUCTURE ONLY -- never imported by
coach_b200.

  rl_coach/agents/mmc_agent.py:56-78     double-DQN target mixed with the Monte Carlo return
  rl_coach/agents/pal_agent.py:70-106    (persistent) advantage learning, then the same mixing

The loops follow the reference statement by statement on the same dtypes (float32 Q arrays, float64 rewards and
returns), so numpy's scalar promotion rounds them exactly as the reference does; tests/test_pal_mmc_host.py pins them
bit for bit against tests/golden/pal_mmc.npz (written from the unmodified reference by oracle/make_golden_pal_mmc.py).
"""
import numpy as np


def mmc_targets(q_next, q_select, q_online, actions, rewards, game_overs, returns, discount, mixing_rate):
    """mmc_agent.py:63-78.  q_next = Q_target(s'), q_select = Q_online(s'), q_online = Q_online(s): float32 [B, A].
    Returns the float32 [B, A] TD targets handed to the train op."""
    selected_actions = np.argmax(q_select, 1)
    targets = np.array(q_online, dtype=np.float32, copy=True)
    for i in range(len(actions)):
        one_step_target = rewards[i] + (1.0 - game_overs[i]) * discount * q_next[i][selected_actions[i]]
        targets[i, actions[i]] = (1 - mixing_rate) * one_step_target + mixing_rate * returns[i]
    return targets


def pal_targets(q_next, q_select, q_target_s, q_online, actions, rewards, game_overs, returns, discount, alpha,
                persistent, mixing_rate):
    """pal_agent.py:70-106.  q_target_s = Q_target(s); the rest as mmc_targets."""
    selected_actions = np.argmax(q_select, 1)
    v_next = np.max(q_next, 1)
    v_s = np.max(q_target_s, 1)
    targets = np.array(q_online, dtype=np.float32, copy=True)
    for i in range(len(actions)):
        a = actions[i]
        targets[i, a] = rewards[i] + (1.0 - game_overs[i]) * discount * q_next[i][selected_actions[i]]
        adv = v_s[i] - q_target_s[i, a]
        next_adv = v_next[i] - q_next[i, selected_actions[i]]
        if persistent:
            targets[i, a] -= alpha * min(adv, next_adv)
        else:
            targets[i, a] -= alpha * adv
        targets[i, a] = (1 - mixing_rate) * targets[i, a] + mixing_rate * returns[i]
    return targets


def learn_step(net, online, target, opt, batch, discount, rule, alpha=0.9, mixing_rate=0.1, huber_loss=True,
               kink=None):
    """One learn_from_batch step of MixedMonteCarloAgent (rule "mmc") or PALAgent ("pal" / "pal_persistent") on an
    oracle.nets.QNetOracle.  batch: states, next_states, actions, rewards, game_overs, returns.  Returns dict(loss,
    targets, grads, grad_norm, new_params, q_online, q_next, q_select, q_target_s)."""
    from collections import OrderedDict

    import torch

    from oracle.nets import _t, q_head_loss
    names = list(online.keys())
    params = [online[n].clone().requires_grad_(True) for n in names]
    with torch.no_grad():
        q_next = net.forward(target, batch["next_states"]).numpy()
        q_select = net.forward(online, batch["next_states"]).numpy()
        q_target_s = net.forward(target, batch["states"]).numpy()
        q_online = net.forward(online, batch["states"]).numpy()
    common = dict(actions=batch["actions"], rewards=batch["rewards"], game_overs=batch["game_overs"],
                  returns=batch["returns"], discount=discount, mixing_rate=mixing_rate)
    f32 = lambda q: np.asarray(q, dtype=np.float32)                     # noqa: E731 (fp64 oracle: same promotion)
    if rule == "mmc":
        targets = mmc_targets(f32(q_next), f32(q_select), f32(q_online), **common)
    else:
        targets = pal_targets(f32(q_next), f32(q_select), f32(q_target_s), f32(q_online), alpha=alpha,
                              persistent=rule == "pal_persistent", **common)
    q = net.forward(OrderedDict(zip(names, params)), batch["states"], kink=kink)
    loss = q_head_loss(q, _t(targets, net.dtype), None, huber_loss)
    grads = torch.autograd.grad(loss, params, allow_unused=True)
    grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, params)]
    gnorm = torch.sqrt(sum((g * g).sum() for g in grads))
    new_params = opt.step([p.detach() for p in params], grads)
    return dict(loss=float(loss.detach()), targets=targets, grads=OrderedDict(zip(names, [g.detach() for g in grads])),
                grad_norm=float(gnorm), new_params=OrderedDict(zip(names, new_params)), q_online=q_online,
                q_next=q_next, q_select=q_select, q_target_s=q_target_s)
