"""Pins the continuous Actor-Critic (A3C) agent to the unmodified reference: tests/golden/a3c_continuous.npz.

  ActorCriticAgent.learn_from_batch   rl_coach/agents/actor_critic_agent.py:127-186 with a BoxActionSpace, stand-in
      networks (as in oracle/make_golden_a3c.py): the state_value_head_targets, the action_advantages and the action
      array handed to accumulate_gradients for A_VALUE, GAE and GAE with estimate_state_value_using_gae on crafted
      segments of 1 to 1000 rows (whole Mujoco episodes), terminal and bootstrapped, scalar (D = 1) and vector actions
  ContinuousEntropy.get_action        exploration_policies/additive_noise.py:62-103 on [mean, std] under
      np.random.seed: E successive calls in training (and the noise schedule after them), the mean in evaluation
  parameter defaults                  the exploration per action space and the Mujoco_A3C preset

Run in the build container only:   python -m oracle.make_golden_a3c_continuous          TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
from types import SimpleNamespace
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# (length, action dimensions, discount, gae_lambda, terminal)
CASES = [(1, 1, 0.99, 0.96, False), (1, 3, 0.99, 1, True), (2, 6, 0.9, 0.96, False), (37, 1, 0.99, 1, False),
         (64, 17, 0.99, 0.96, True), (200, 3, 0.99, 0.96, False), (999, 1, 0.99, 1, False),
         (1000, 6, 0.99, 0.96, True), (1000, 1, 0.9, 0.96, False)]
MODES = ("A_VALUE", "GAE", "GAE_VALUE")
# (environments, action dimensions, seed)
ACTING = [(1, 1, 300), (8, 1, 301), (16, 3, 302), (5, 17, 303)]


def golden_targets(out, rng):
    from rl_coach.agents.actor_critic_agent import ActorCriticAgent
    from rl_coach.agents.policy_optimization_agent import PolicyGradientRescaler
    from rl_coach.core_types import Batch, Transition
    from rl_coach.spaces import BoxActionSpace
    sig = SimpleNamespace(add_sample=lambda x: None)
    for c, (L, D, discount, lam, terminal) in enumerate(CASES):
        values = (rng.randn(L, 1) * 3).astype(np.float32)
        boot = (rng.randn(1, 1) * 3).astype(np.float32)
        rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0, 1 / 20.], L).astype(np.float64)
        game_overs = np.zeros(L, dtype=bool)
        game_overs[-1] = terminal
        # what ContinuousEntropy.get_action returns: np.random.normal of a 0-d mean (a float) or of a [D] mean
        acts = rng.randn(L, D) * 2
        actions = [float(acts[i, 0]) if D == 1 else acts[i].copy() for i in range(L)]
        batch = Batch([Transition(state={'observation': np.zeros(4, dtype=np.float32)}, action=actions[i],
                                  reward=rewards[i].item(),
                                  next_state={'observation': np.full(4, i, dtype=np.float32)},
                                  game_over=bool(game_overs[i])) for i in range(L)])
        out.update({"c%d_values" % c: values[:, 0], "c%d_boot" % c: boot[0, 0], "c%d_rewards" % c: rewards,
                    "c%d_game_overs" % c: game_overs.astype(np.uint8), "c%d_discount" % c: np.float64(discount),
                    "c%d_lambda" % c: np.float64(lam), "c%d_actions" % c: acts, "c%d_dim" % c: np.int64(D)})
        for mode in MODES:
            rec, calls = {}, []

            def predict(s):
                calls.append(1)
                v = values.copy() if len(calls) == 1 else boot.copy()
                return [v, np.zeros((len(v), D), np.float32), np.ones((len(v), D), np.float32)]

            def accumulate(inputs, targets):
                rec.update(t=np.array(targets[0]), a=np.array(targets[1]), x=np.array(inputs['output_1_0']))
                return 0.0, [0.0, 0.0], 0.0
            net = SimpleNamespace(online_network=SimpleNamespace(predict=predict, accumulate_gradients=accumulate))
            alg = SimpleNamespace(discount=discount, gae_lambda=lam,
                                  estimate_state_value_using_gae=mode == "GAE_VALUE")
            fake = SimpleNamespace(
                ap=SimpleNamespace(network_wrappers={'main': SimpleNamespace(
                    input_embedders_parameters={'observation': None})}, algorithm=alg),
                networks={'main': net},
                spaces=SimpleNamespace(action=BoxActionSpace(D, -np.ones(D), np.ones(D))),
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
            if mode == "A_VALUE":
                out["c%d_fed_actions" % c] = rec["x"]
    out["n_cases"] = np.int64(len(CASES))


def golden_acting(out, rng):
    from rl_coach.core_types import RunPhase
    from rl_coach.exploration_policies.continuous_entropy import ContinuousEntropy
    from rl_coach.schedules import LinearSchedule
    from rl_coach.spaces import BoxActionSpace
    for k, (E, D, seed) in enumerate(ACTING):
        high = (rng.rand(D) * 3 + 0.5).astype(np.float32)
        means = (rng.randn(E, D) * high).astype(np.float32)
        stds = (np.abs(rng.randn(E, D)) + 1e-3).astype(np.float32)
        schedule = LinearSchedule(0.5, 0.1, 7)
        pol = ContinuousEntropy(BoxActionSpace(D, -high, high), schedule, 0.05)
        pol.change_phase(RunPhase.TRAIN)
        np.random.seed(seed)
        train = np.array([np.asarray(pol.get_action([means[e][None], stds[e][None]]), np.float64).reshape(D)
                          for e in range(E)])
        out["act%d_noise_after" % k] = np.float64(schedule.current_value)
        pol.change_phase(RunPhase.TEST)
        ev = np.array([np.asarray(pol.get_action([means[e][None], stds[e][None]])).reshape(D) for e in range(E)])
        out["act%d_noise_after_eval" % k] = np.float64(schedule.current_value)
        out.update({"act%d_means" % k: means, "act%d_stds" % k: stds, "act%d_high" % k: high,
                    "act%d_seed" % k: np.int64(seed), "act%d_train" % k: train, "act%d_eval" % k: ev})
    out["n_acting"] = np.int64(len(ACTING))


def golden_parameters(out):
    from rl_coach.agents.actor_critic_agent import ActorCriticAgentParameters
    ap = ActorCriticAgentParameters()
    ex = {k.__name__: v for k, v in ap.exploration.items()}
    out["par_exploration"] = np.array(sorted("%s:%s" % (k, type(v).__name__) for k, v in ex.items()))
    box = ex["BoxActionSpace"]
    out["par_box_path"] = np.array(box.path)
    out["par_box_noise"] = np.array([box.noise_schedule.initial_value, box.noise_schedule.final_value,
                                     box.noise_schedule.decay_steps, box.evaluation_noise,
                                     float(box.noise_as_percentage_from_action_space)])
    for name in ("rl_coach.environments.gym_environment", "rl_coach.graph_managers.graph_manager",
                 "rl_coach.graph_managers.basic_rl_graph_manager"):
        sys.modules.setdefault(name, mock.MagicMock())
    import importlib
    mod = importlib.import_module("rl_coach.presets.Mujoco_A3C")
    ap = mod.agent_params
    net, alg = ap.network_wrappers['main'], ap.algorithm
    out["pre_mujoco"] = np.array([net.learning_rate, alg.discount, alg.num_steps_between_gradient_updates,
                                  alg.apply_gradients_every_x_episodes, alg.beta_entropy, alg.gae_lambda])
    out["pre_mujoco_rescaler"] = np.array(alg.policy_gradient_rescaler.name)
    rf = ap.input_filter.reward_filters
    out["pre_mujoco_reward_rescale"] = np.array([f.rescale_factor for f in rf.values()], dtype=np.float64)
    out["pre_mujoco_observation_filters"] = np.array(
        [type(f).__name__ for flt in ap.input_filter.observation_filters.values() for f in flt.values()])
    v = mod.preset_validation_params
    out["pre_mujoco_workers"] = np.int64(v.num_workers)
    out["pre_mujoco_reward_test_level"] = np.array(v.reward_test_level)


def main():
    from oracle import ref_loader
    ref_loader.load()
    rng = np.random.RandomState(2026)
    out = {}
    golden_targets(out, rng)
    golden_acting(out, rng)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "a3c_continuous.npz"), **out)
    print("a3c_continuous", len(out), "arrays")


if __name__ == "__main__":
    main()
