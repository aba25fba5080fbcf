"""Pins the Actor-Critic (A3C) agent to the unmodified reference: tests/golden/a3c.npz.

  ActorCriticAgent.learn_from_batch   rl_coach/agents/actor_critic_agent.py:111-165, stand-in networks (as in
      oracle/make_golden_nstep_q.py): the state_value_head_targets and action_advantages handed to accumulate_gradients
      for A_VALUE, GAE and GAE with estimate_state_value_using_gae on crafted segments: lengths 1, 2, 5, 7, 20, 23,
      terminal and bootstrapped last rows, lambda in {1, 0.96}, discount 0.99 / 0.9, mixed, integer and r / 200 rewards
  Categorical.get_action              exploration_policies/categorical.py:36-47 under np.random.seed: crafted
      probability vectors (zeros, near-ties at cdf boundaries, 18 actions, fp32 sums != 1), training and evaluation
  parameter defaults                  ActorCritic agent / algorithm / network parameters and the two presets' values

Run in the build container only:   python -m oracle.make_golden_a3c          TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
from types import SimpleNamespace
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# (length, discount, gae_lambda, terminal, reward kind)
CASES = [(1, 0.99, 0.96, False, "mix"), (1, 0.99, 1, True, "mix"), (2, 0.9, 0.96, False, "mix"),
         (5, 0.99, 1, False, "scaled"), (5, 0.99, 0.96, True, "mix"), (7, 0.9, 1, False, "mix"),
         (7, 0.99, 0.96, False, "int"), (20, 0.99, 0.96, False, "mix"), (20, 0.99, 1, True, "scaled"),
         (23, 0.99, 1, False, "mix"), (23, 0.9, 0.96, True, "int"), (5, 0.99, 0.96, False, "big")]
MODES = ("A_VALUE", "GAE", "GAE_VALUE")


def _case(rng, L, terminal, kind):
    values = (rng.randn(L, 1) * 3).astype(np.float32)
    boot = (rng.randn(1, 1) * 3).astype(np.float32)
    if kind == "big":
        values *= np.float32(300.0)
        boot *= np.float32(300.0)
    if kind == "int":
        rewards = rng.randint(-3, 4, L).astype(np.int64)
    elif kind == "scaled":
        rewards = rng.choice([-1.0, 0.0, 1.0], L) * (1 / 200.)
    else:
        rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0, 1 / 200.], L).astype(np.float64)
    game_overs = np.zeros(L, dtype=bool)
    game_overs[-1] = terminal
    return values, boot, rewards, game_overs


def golden_targets(out, rng):
    from rl_coach.agents.actor_critic_agent import ActorCriticAgent
    from rl_coach.agents.policy_optimization_agent import PolicyGradientRescaler
    from rl_coach.core_types import Batch, Transition
    from rl_coach.spaces import DiscreteActionSpace
    sig = SimpleNamespace(add_sample=lambda x: None)
    for c, (L, discount, lam, terminal, kind) in enumerate(CASES):
        values, boot, rewards, game_overs = _case(rng, L, terminal, kind)
        actions = rng.randint(0, 4, L)
        batch = Batch([Transition(state={'observation': np.zeros(4, dtype=np.float32)}, action=int(actions[i]),
                                  reward=rewards[i].item(),
                                  next_state={'observation': np.full(4, i, dtype=np.float32)},
                                  game_over=bool(game_overs[i])) for i in range(L)])
        assert batch.rewards().dtype == (np.int64 if kind == "int" else np.float64)
        out.update({"c%d_values" % c: values[:, 0], "c%d_boot" % c: boot[0, 0], "c%d_rewards" % c: rewards,
                    "c%d_game_overs" % c: game_overs.astype(np.uint8), "c%d_discount" % c: np.float64(discount),
                    "c%d_lambda" % c: np.float64(lam)})
        for mode in MODES:
            rec, calls = {}, []

            def predict(s):
                calls.append(1)
                v = values.copy() if len(calls) == 1 else boot.copy()
                return [v, np.full((len(v), 4), 0.25, dtype=np.float32)]
            net = SimpleNamespace(online_network=SimpleNamespace(
                predict=predict,
                accumulate_gradients=lambda s, t: rec.update(t=np.array(t[0]), a=np.array(t[1])) or (0.0, [0.0, 0.0],
                                                                                                      0.0)))
            alg = SimpleNamespace(discount=discount, gae_lambda=lam,
                                  estimate_state_value_using_gae=mode == "GAE_VALUE")
            fake = SimpleNamespace(
                ap=SimpleNamespace(network_wrappers={'main': SimpleNamespace(
                    input_embedders_parameters={'observation': None})}, algorithm=alg),
                networks={'main': net}, spaces=SimpleNamespace(action=DiscreteActionSpace(4)),
                policy_gradient_rescaler=PolicyGradientRescaler.A_VALUE if mode == "A_VALUE" else
                PolicyGradientRescaler.GAE,
                state_values=sig, action_advantages=sig, unclipped_grads=sig, value_loss=sig, policy_loss=sig)
            fake.discount = lambda x, g: ActorCriticAgent.discount(fake, x, g)
            fake.get_general_advantage_estimation_values = \
                lambda r, v: ActorCriticAgent.get_general_advantage_estimation_values(fake, r, v)
            ActorCriticAgent.learn_from_batch(fake, batch)
            assert rec["t"].dtype == np.float64 and rec["a"].dtype == np.float64, (rec["t"].dtype, rec["a"].dtype)
            out["c%d_%s_targets" % (c, mode.lower())] = rec["t"].reshape(L)
            out["c%d_%s_advantages" % (c, mode.lower())] = rec["a"].reshape(L)
    out["n_cases"] = np.int64(len(CASES))


def _probability_vectors(rng):
    ps = []
    ps.append(np.array([0.0, 1.0, 0.0], np.float32))                                  # zeros
    ps.append(np.array([0.5, 0.5], np.float32))
    ps.append(np.array([0.25, 0.0, 0.25, 0.0, 0.5], np.float32))
    x = rng.randn(18).astype(np.float32)
    e = np.exp(x - x.max()).astype(np.float32)
    ps.append((e / e.sum()).astype(np.float32))                                        # 18 actions, fp32 sum != 1
    ps.append(np.full(18, np.float32(1 / 18.), np.float32))
    ps.append(np.array([1 / 3., 1 / 3., 1 / 3.], np.float32))                           # fp32 sum != 1
    ps.append(np.array([0.1, 0.2, 0.3, 0.4], np.float32))
    ps.append(np.array([0.5, 0.5 - 2 ** -24, 2 ** -24], np.float32))                   # near-ties at a cdf boundary
    for _ in range(4):
        x = (rng.randn(6) * 2).astype(np.float32)
        e = np.exp(x - x.max()).astype(np.float32)
        ps.append((e / e.sum()).astype(np.float32))
    return ps


def golden_categorical(out, rng):
    from rl_coach.core_types import RunPhase
    from rl_coach.exploration_policies.categorical import Categorical
    from rl_coach.spaces import DiscreteActionSpace
    ps = _probability_vectors(rng)
    for k, p in enumerate(ps):
        pol = Categorical(DiscreteActionSpace(len(p)))
        pol.change_phase(RunPhase.TRAIN)
        np.random.seed(100 + k)
        draws = [pol.get_action(p)[0] for _ in range(64)]
        pol.change_phase(RunPhase.TEST)
        out["cat%d_p" % k] = p
        out["cat%d_seed" % k] = np.int64(100 + k)
        out["cat%d_train" % k] = np.array(draws, dtype=np.int64)
        out["cat%d_eval" % k] = np.int64(pol.get_action(p)[0])
    out["n_cat"] = np.int64(len(ps))


def golden_parameters(out):
    from rl_coach.agents.actor_critic_agent import ActorCriticAgentParameters
    ap = ActorCriticAgentParameters()
    alg, net = ap.algorithm, ap.network_wrappers['main']
    out["par_algorithm"] = np.array([alg.num_steps_between_gradient_updates, alg.apply_gradients_every_x_episodes,
                                     alg.beta_entropy, alg.gae_lambda, float(alg.estimate_state_value_using_gae),
                                     alg.discount])
    out["par_rescaler"] = np.array(alg.policy_gradient_rescaler.name)
    out["par_network"] = np.array([net.learning_rate, net.adam_optimizer_beta1, net.adam_optimizer_beta2,
                                   net.optimizer_epsilon, float(net.replace_mse_with_huber_loss),
                                   float(net.create_target_network), float(net.async_training), net.clip_gradients,
                                   net.heads_parameters[0].loss_weight, net.heads_parameters[1].loss_weight])
    out["par_heads"] = np.array([type(h).__name__ for h in net.heads_parameters])
    for name in ("rl_coach.environments.gym_environment", "rl_coach.graph_managers.graph_manager",
                 "rl_coach.graph_managers.basic_rl_graph_manager"):
        sys.modules.setdefault(name, mock.MagicMock())
    import importlib
    for tag, preset in (("cartpole", "CartPole_A3C"), ("atari", "Atari_A3C")):
        mod = importlib.import_module("rl_coach.presets." + preset)
        ap = mod.agent_params
        net, alg = ap.network_wrappers['main'], ap.algorithm
        out["pre_%s" % tag] = np.array([net.learning_rate, alg.discount, alg.num_steps_between_gradient_updates,
                                        alg.apply_gradients_every_x_episodes, alg.beta_entropy, alg.gae_lambda])
        out["pre_%s_rescaler" % tag] = np.array(alg.policy_gradient_rescaler.name)
        rf = getattr(ap.input_filter, "reward_filters", {}) if ap.input_filter is not None else {}
        out["pre_%s_reward_rescale" % tag] = np.array([f.rescale_factor for f in rf.values()], dtype=np.float64)
        out["pre_%s_workers" % tag] = np.int64(getattr(mod.preset_validation_params, "num_workers", 1))


def main():
    from oracle import ref_loader
    ref_loader.load()
    rng = np.random.RandomState(2025)
    out = {}
    golden_targets(out, rng)
    golden_categorical(out, rng)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "a3c.npz"), **out)
    print("a3c", len(out), "arrays")


if __name__ == "__main__":
    main()
