"""Pins the Policy Gradients (REINFORCE) agent to the unmodified reference: tests/golden/pg.npz.

  Episode.update_discounted_rewards     core_types.py:771-801 with n_step -1: the returns of crafted episodes of lengths
                                        1, 7, 8, 9, 127, 128, 129, 200 and 1000 (mixed, integer and r / 20 rewards)
                                        and a zero-std episode
  PolicyGradientsAgent.learn_from_batch policy_gradients_agent.py:47-86 with a stand-in network (as in
                                        oracle/make_golden_a3c.py): the targets handed to accumulate_gradients for the
                                        four return rescalers, each episode on fresh statistics after
                                        update_episode_statistics (so its timestep targets are all zero: the
                                        sequence below pins that rescaler)
  update_episode_statistics             policy_optimization_agent.py:58-71 over a sequence of 12 episodes: the
                                        per-timestep table, mean and std after each, and the targets learn_from_batch
                                        hands over with FUTURE_RETURN_NORMALIZED_BY_TIMESTEP on that running table
  AdditiveNoise.get_action              exploration_policies/additive_noise.py under np.random.seed: a range-3 action
                                        in training (LinearSchedule(0.1, 0.1, 50000)) and evaluation
  parameter defaults                    PolicyGradients agent / algorithm / network parameters and the two presets

Run in the build container only:   python -m oracle.make_golden_pg          TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
from types import SimpleNamespace
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# (length, discount, reward kind)
CASES = [(1, 0.99, "mix"), (7, 0.99, "mix"), (8, 0.9, "int"), (9, 0.99, "scaled"), (127, 0.99, "mix"),
         (128, 0.99, "scaled"), (129, 0.9, "mix"), (200, 0.99, "ones"), (1000, 0.99, "mix"), (5, 0.99, "zero_std")]
RESCALERS = ("TOTAL_RETURN", "FUTURE_RETURN", "FUTURE_RETURN_NORMALIZED_BY_EPISODE",
             "FUTURE_RETURN_NORMALIZED_BY_TIMESTEP")
TABLE = 1000


def _rewards(rng, L, kind):
    if kind == "int":
        return rng.randint(-3, 4, L).astype(np.int64)
    if kind == "scaled":
        return rng.choice([-1.0, 0.0, 1.0], L) * (1 / 20.)
    if kind == "ones":
        return np.full(L, 1 / 200.)
    if kind == "zero_std":
        return np.zeros(L)
    return rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0, 1 / 200.], L).astype(np.float64)


def _episode(rewards, discount):
    from rl_coach.core_types import Episode, Transition
    ep = Episode(discount=discount, n_step=-1)
    for i, r in enumerate(rewards):
        ep.insert(Transition(state={'observation': np.zeros(4, dtype=np.float32)}, action=0, reward=r.item(),
                             next_state={'observation': np.zeros(4, dtype=np.float32)},
                             game_over=i == len(rewards) - 1))
    ep.update_transitions_rewards_and_bootstrap_data()
    return ep


def _fake_agent(rescaler):
    from rl_coach.agents.policy_optimization_agent import PolicyGradientRescaler
    from rl_coach.spaces import DiscreteActionSpace
    rec = {}
    sig = SimpleNamespace(add_sample=lambda x: None)
    net = SimpleNamespace(online_network=SimpleNamespace(
        accumulate_gradients=lambda s, t: rec.update(t=np.array(t)) or (0.0, [0.0], 0.0)))
    fake = SimpleNamespace(
        ap=SimpleNamespace(network_wrappers={'main': SimpleNamespace(input_embedders_parameters={'observation': None})}),
        networks={'main': net}, spaces=SimpleNamespace(action=DiscreteActionSpace(2)),
        policy_gradient_rescaler=PolicyGradientRescaler[rescaler], returns_mean=sig, returns_variance=sig,
        mean_return_over_multiple_episodes=np.zeros(TABLE), num_episodes_where_step_has_been_seen=np.zeros(TABLE))
    return fake, rec


def golden_targets(out, rng):
    from rl_coach.agents.policy_gradients_agent import PolicyGradientsAgent
    from rl_coach.agents.policy_optimization_agent import PolicyOptimizationAgent
    from rl_coach.core_types import Batch
    for c, (L, discount, kind) in enumerate(CASES):
        rewards = _rewards(rng, L, kind)
        ep = _episode(rewards, discount)
        R = np.array([t.n_step_discounted_rewards for t in ep.transitions])
        assert R.dtype == np.float64
        out.update({"c%d_rewards" % c: rewards, "c%d_discount" % c: np.float64(discount), "c%d_returns" % c: R})
        for name in RESCALERS:
            fake, rec = _fake_agent(name)
            if "NORMALIZED" in name:
                PolicyOptimizationAgent.update_episode_statistics(fake, ep)
            PolicyGradientsAgent.learn_from_batch(fake, Batch(ep.transitions))
            assert rec["t"].dtype == np.float64
            out["c%d_%s" % (c, name.lower())] = rec["t"].reshape(L)
    out["n_cases"] = np.int64(len(CASES))


def golden_table_sequence(out, rng):
    from rl_coach.agents.policy_gradients_agent import PolicyGradientsAgent
    from rl_coach.agents.policy_optimization_agent import PolicyOptimizationAgent
    from rl_coach.core_types import Batch
    fake, rec = _fake_agent("FUTURE_RETURN_NORMALIZED_BY_TIMESTEP")
    lengths = [9, 3, 17, 9, 1, 130, 40, 9, 200, 2, 64, 129]
    for k, L in enumerate(lengths):
        rewards = _rewards(rng, L, "mix" if k % 3 else "scaled")
        ep = _episode(rewards, 0.99)
        PolicyOptimizationAgent.update_episode_statistics(fake, ep)
        PolicyGradientsAgent.learn_from_batch(fake, Batch(ep.transitions))
        assert rec["t"].dtype == np.float64
        out["seq%d_rewards" % k] = rewards
        out["seq%d_targets" % k] = rec["t"].reshape(L)
        out["seq%d_mean_table" % k] = fake.mean_return_over_multiple_episodes[:max(lengths)].copy()
        out["seq%d_count_table" % k] = fake.num_episodes_where_step_has_been_seen[:max(lengths)].copy()
        out["seq%d_mean_std" % k] = np.array([fake.mean_discounted_return, fake.std_discounted_return])
    out["n_seq"] = np.int64(len(lengths))


def golden_additive_noise(out, rng):
    from rl_coach.core_types import RunPhase
    from rl_coach.exploration_policies.additive_noise import AdditiveNoise, AdditiveNoiseParameters
    from rl_coach.spaces import BoxActionSpace
    low, high = np.full(1, -3, np.float32), np.full(1, 3, np.float32)      # gym's float32 Box bounds
    par = AdditiveNoiseParameters()
    pol = AdditiveNoise(BoxActionSpace(1, low, high), par.noise_schedule, par.evaluation_noise,
                        par.noise_as_percentage_from_action_space)
    means = (np.tanh(rng.randn(32, 1)) * 3).astype(np.float32)
    pol.change_phase(RunPhase.TRAIN)
    np.random.seed(7)
    train = np.array([pol.get_action(m[None, :]) for m in means])
    pol.change_phase(RunPhase.TEST)
    evals = np.array([pol.get_action(m[None, :]) for m in means])
    out.update({"noise_means": means, "noise_seed": np.int64(7), "noise_train": train, "noise_eval": evals,
                "noise_low": low, "noise_high": high, "noise_value": np.float64(pol.noise_schedule.current_value)})


def golden_parameters(out):
    from rl_coach.agents.policy_gradients_agent import PolicyGradientsAgentParameters
    ap = PolicyGradientsAgentParameters()
    alg, net = ap.algorithm, ap.network_wrappers['main']
    out["par_algorithm"] = np.array([alg.num_steps_between_gradient_updates, alg.apply_gradients_every_x_episodes,
                                     alg.beta_entropy, alg.discount, alg.n_step])
    out["par_rescaler"] = np.array(alg.policy_gradient_rescaler.name)
    out["par_network"] = np.array([net.learning_rate, net.adam_optimizer_beta1, net.adam_optimizer_beta2,
                                   net.optimizer_epsilon, float(net.async_training),
                                   -1.0 if net.clip_gradients is None else net.clip_gradients,
                                   net.heads_parameters[0].loss_weight])
    out["par_heads"] = np.array([type(h).__name__ for h in net.heads_parameters])
    out["par_exploration"] = np.array(sorted(type(v).__name__ for v in ap.exploration.values()))
    for name in ("rl_coach.environments.gym_environment", "rl_coach.graph_managers.graph_manager",
                 "rl_coach.graph_managers.basic_rl_graph_manager"):
        sys.modules.setdefault(name, mock.MagicMock())
    import importlib
    for tag, preset in (("cartpole", "CartPole_PG"), ("pendulum", "InvertedPendulum_PG")):
        mod = importlib.import_module("rl_coach.presets." + preset)
        ap = mod.agent_params
        net, alg = ap.network_wrappers['main'], ap.algorithm
        out["pre_%s" % tag] = np.array([net.learning_rate, alg.discount, alg.num_steps_between_gradient_updates,
                                        alg.apply_gradients_every_x_episodes, alg.beta_entropy])
        out["pre_%s_rescaler" % tag] = np.array(alg.policy_gradient_rescaler.name)
        rf = ap.input_filter.reward_filters
        out["pre_%s_reward_rescale" % tag] = np.array([f.rescale_factor for f in rf.values()], dtype=np.float64)
        out["pre_%s_observation_filters" % tag] = np.array(
            [type(f).__name__ for f in ap.input_filter.observation_filters.get('observation', {}).values()] or [""])


def main():
    from oracle import ref_loader
    ref_loader.load()
    rng = np.random.RandomState(2026)
    out = {}
    golden_targets(out, rng)
    golden_table_sequence(out, rng)
    golden_additive_noise(out, rng)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "pg.npz"), **out)
    print("pg", len(out), "arrays")


if __name__ == "__main__":
    main()
