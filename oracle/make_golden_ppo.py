"""Pins the PPO (KL-penalty) agent to the unmodified reference: tests/golden/ppo.npz.

  PPOAgent.fill_advantages          rl_coach/agents/ppo_agent.py:156-195 with a stand-in critic (its V(s) per row):
      GAE (lambda 0.96 and 1) and A_VALUE over back-to-back episodes of 1 to 1000 transitions
  PPOAgent.train                    ppo_agent.py:362-391 with stand-in networks (mocked TF): what train_value_network
      and train_policy_network feed per minibatch (rows, Monte Carlo return targets, actions, advantages, the old
      policy's mean and std) on rollouts longer than num_consecutive_playing_steps and not a multiple of 128, and the
      KL coefficient after post_training_commands
  PPOAgent.update_kl_coefficient    ppo_agent.py:329-353: coefficient trajectories over KL means
  AdditiveNoise.get_action          exploration_policies/additive_noise.py:62-103 on [mean, std] under np.random.seed
  parameter defaults                PPOAgentParameters and the Mujoco_PPO preset

Run in the build container only:   python -m oracle.make_golden_ppo          TEST INFRASTRUCTURE ONLY.
"""
import importlib
import os
import sys
from types import SimpleNamespace
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# fill_advantages: (episode lengths, discount, rescaler, gae_lambda)
ADV_CASES = [([1, 2], 0.99, "GAE", 0.96), ([1, 1, 3], 0.99, "A_VALUE", 1.0), ([1000, 1, 37], 0.99, "GAE", 1.0),
             ([200, 1000, 5], 0.9, "GAE", 0.96), ([999, 2, 1, 64], 0.99, "A_VALUE", 1.0), ([1000], 0.99, "GAE", 0.96)]
# train: (episode lengths, action dimensions, rescaler, gae_lambda, per-minibatch KL of the stand-in head)
TRAIN_CASES = [([1000, 1, 999, 300, 1000, 1000, 1000], 3, "GAE", 0.96, 0.002),
               ([1000] * 6 + [1], 1, "A_VALUE", 1.0, 0.05)]
# update_kl_coefficient: (initial coefficient, target, KL means)
KL_CASES = [(1.0, 0.01, [0.02, 0.02, 0.005, 0.0131, 0.0069, 0.01, 0.1, 0.0]),
            (0.2, 0.01, [0.001] * 20 + [1.0] * 20),
            (0.2, 0.003, [0.004, 0.002, 0.0039, 0.0021, 0.003])]
# acting: (environments, action dimensions, seed)
ACTING = [(1, 1, 400), (8, 1, 401), (16, 3, 402), (5, 6, 403), (3, 17, 404)]


def _dataset(rng, lengths, A):
    from rl_coach.core_types import Transition
    N = int(sum(lengths))
    rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0, 1 / 20.], N).astype(np.float64)
    returns = rng.randn(N) * 5
    values = (rng.randn(N) * 3).astype(np.float32)
    actions = rng.randn(N, A) * 2
    game_overs = np.zeros(N, dtype=bool)
    game_overs[np.cumsum(lengths) - 1] = True
    ts = []
    for i in range(N):
        t = Transition(state={'observation': np.array([i, 0.5], dtype=np.float32)},
                       action=float(actions[i, 0]) if A == 1 else actions[i].copy(), reward=rewards[i].item(),
                       next_state={'observation': np.zeros(2, dtype=np.float32)}, game_over=bool(game_overs[i]))
        t.n_step_discounted_rewards = returns[i]
        ts.append(t)
    return ts, dict(rewards=rewards, returns=returns, values=values, actions=actions,
                    game_overs=game_overs.astype(np.uint8))


def _fake(alg, values, A, kl_value, rec):
    """a PPOAgent stand-in: numpy plumbing of the reference, networks replaced by recorders"""
    from rl_coach.agents.actor_critic_agent import ActorCriticAgent
    from rl_coach.agents.ppo_agent import PPOAgent
    from rl_coach.spaces import BoxActionSpace
    sig = SimpleNamespace(add_sample=lambda x: None)
    rows = lambda s: s['observation'][:, 0].astype(np.int64)         # noqa: E731
    old_mean = lambda r: np.stack([np.sin(r + j).astype(np.float32) for j in range(A)], 1)    # noqa: E731
    old_std = lambda r: np.tile(np.exp(np.float32(-0.5) + np.arange(A, dtype=np.float32) / 8), (len(r), 1))  # noqa

    def critic_accumulate(inputs, targets):
        rec["critic"].append((rows(inputs), np.array(targets)))
        return [0.0]

    def actor_accumulate(inputs, targets, additional_fetches=None):
        rec["actor"].append((rows(inputs), np.array(inputs['output_0_0']), np.array(targets[0]),
                             np.array(inputs['output_0_1']), np.array(inputs['output_0_2'])))
        return 0.0, [0.0], 0.0, [np.float32(kl_value), np.float32(0.0)]

    variables = {"kl": np.float32(alg.initial_kl_coefficient)}

    def set_variable_value(assign, value, ph):
        variables["kl"] = np.float32(value)
    critic_online = SimpleNamespace(predict=lambda s: values[rows(s)][:, None].copy(), optimizer_type='Adam',
                                    inputs={}, accumulate_gradients=critic_accumulate,
                                    reset_accumulated_gradients=lambda: None)
    head = SimpleNamespace(kl_divergence=None, entropy=None, kl_coefficient="kl", assign_kl_coefficient=None,
                           kl_coefficient_ph=None)
    actor_online = SimpleNamespace(accumulate_gradients=actor_accumulate, output_heads=[head],
                                   reset_accumulated_gradients=lambda: None,
                                   get_variable_value=lambda name: variables[name],
                                   set_variable_value=set_variable_value)
    nop = lambda *a: None        # noqa: E731
    critic = SimpleNamespace(online_network=critic_online, sync=nop, set_is_training=nop,
                             apply_gradients_to_online_network=nop,
                             target_network=SimpleNamespace(predict=lambda s: values[rows(s)][:, None].copy()))
    actor = SimpleNamespace(online_network=actor_online, sync=nop, set_is_training=nop,
                            apply_gradients_to_online_network=nop,
                            target_network=SimpleNamespace(predict=lambda s: [old_mean(rows(s)), old_std(rows(s))]))
    net = lambda: SimpleNamespace(input_embedders_parameters={'observation': None}, batch_size=128,   # noqa: E731
                                  learning_rate_decay_rate=0, learning_rate=5e-5)
    fake = SimpleNamespace(
        ap=SimpleNamespace(algorithm=alg, network_wrappers={'critic': net(), 'actor': net()}, task_parameters=None),
        networks={'critic': critic, 'actor': actor}, spaces=SimpleNamespace(action=BoxActionSpace(A)),
        policy_gradient_rescaler=alg.policy_gradient_rescaler, action_advantages=sig, value_loss=sig,
        policy_loss=sig, unclipped_grads=sig, entropy=sig, kl_divergence=sig, training_iteration=0,
        total_kl_divergence_during_training_process=0.0, _should_train=lambda: True,
        call_memory=lambda name: rec["memory_calls"].append(name), update_log=nop)
    fake.discount = lambda x, g: ActorCriticAgent.discount(fake, x, g)
    fake.get_general_advantage_estimation_values = \
        lambda r, v: ActorCriticAgent.get_general_advantage_estimation_values(fake, r, v)
    for m in ("fill_advantages", "train_value_network", "train_policy_network", "update_kl_coefficient",
              "post_training_commands"):
        setattr(fake, m, (lambda f: lambda *a: f(fake, *a))(getattr(PPOAgent, m)))
    return fake, variables


def _algorithm(rescaler, lam, discount=0.99):
    from rl_coach.agents.policy_optimization_agent import PolicyGradientRescaler
    from rl_coach.agents.ppo_agent import PPOAlgorithmParameters
    alg = PPOAlgorithmParameters()
    alg.policy_gradient_rescaler = getattr(PolicyGradientRescaler, rescaler)
    alg.gae_lambda, alg.discount = lam, discount
    return alg


def golden_advantages(out, rng):
    for c, (lengths, discount, rescaler, lam) in enumerate(ADV_CASES):
        ts, d = _dataset(rng, lengths, 1)
        rec = dict(critic=[], actor=[], memory_calls=[])
        fake, _ = _fake(_algorithm(rescaler, lam, discount), d["values"], 1, 0.0, rec)
        fake.memory = SimpleNamespace(transitions=ts)
        fake.fill_advantages(ts)
        adv = np.array([t.info['advantage'] for t in ts], dtype=np.float64)
        out.update({"adv%d_%s" % (c, k): d[k] for k in ("rewards", "returns", "values", "game_overs")})
        out.update({"adv%d_discount" % c: np.float64(discount), "adv%d_lambda" % c: np.float64(lam),
                    "adv%d_rescaler" % c: np.array(rescaler), "adv%d_advantages" % c: adv})
    out["n_adv"] = np.int64(len(ADV_CASES))


def golden_train(out, rng):
    for c, (lengths, A, rescaler, lam, kl_value) in enumerate(TRAIN_CASES):
        ts, d = _dataset(rng, lengths, A)
        rec = dict(critic=[], actor=[], memory_calls=[])
        alg = _algorithm(rescaler, lam)
        fake, variables = _fake(alg, d["values"], A, kl_value, rec)
        fake.memory = SimpleNamespace(transitions=ts)
        k0 = variables["kl"]
        fake_train = __import__("rl_coach.agents.ppo_agent", fromlist=["PPOAgent"]).PPOAgent.train
        fake_train(fake)
        n_mb = min(len(ts), alg.num_consecutive_playing_steps.num_steps) // 128
        assert len(rec["critic"]) == n_mb and len(rec["actor"]) == 10 * n_mb, (len(rec["critic"]), len(rec["actor"]))
        first = rec["actor"][:n_mb]
        for e in range(1, 10):                          # every epoch feeds the same minibatches in the same order
            for a, b in zip(first, rec["actor"][e * n_mb:(e + 1) * n_mb]):
                assert all(np.array_equal(x, y) for x, y in zip(a, b))
        cat = lambda xs: np.concatenate(xs, 0)          # noqa: E731
        out.update({"train%d_%s" % (c, k): d[k] for k in ("rewards", "returns", "values", "game_overs", "actions")})
        out.update({"train%d_rescaler" % c: np.array(rescaler), "train%d_lambda" % c: np.float64(lam),
                    "train%d_kl_value" % c: np.float64(kl_value), "train%d_dim" % c: np.int64(A),
                    "train%d_critic_rows" % c: cat([r for r, _ in rec["critic"]]),
                    "train%d_critic_targets" % c: cat([t for _, t in rec["critic"]]),
                    "train%d_actor_rows" % c: cat([f[0] for f in first]),
                    "train%d_actor_actions" % c: cat([f[1] for f in first]),
                    "train%d_actor_advantages" % c: cat([f[2] for f in first]),
                    "train%d_actor_old_mean" % c: cat([f[3] for f in first]),
                    "train%d_actor_old_std" % c: cat([f[4] for f in first]),
                    "train%d_kl_before" % c: k0, "train%d_kl_after" % c: variables["kl"],
                    "train%d_memory_calls" % c: np.array(rec["memory_calls"])})
    out["n_train"] = np.int64(len(TRAIN_CASES))


def golden_kl(out):
    for c, (k0, target, kls) in enumerate(KL_CASES):
        alg = _algorithm("GAE", 0.96)
        alg.initial_kl_coefficient, alg.target_kl_divergence = k0, target
        fake, variables = _fake(alg, np.zeros(1, np.float32), 1, 0.0, dict(critic=[], actor=[], memory_calls=[]))
        traj = []
        for kl in kls:
            fake.total_kl_divergence_during_training_process = np.float32(kl)
            fake.update_kl_coefficient()
            traj.append(variables["kl"])
        out.update({"kl%d_initial" % c: np.float32(k0), "kl%d_target" % c: np.float64(target),
                    "kl%d_means" % c: np.array(kls, np.float32), "kl%d_coefficients" % c: np.array(traj, np.float32)})
    out["n_kl"] = np.int64(len(KL_CASES))


def golden_acting(out, rng):
    from rl_coach.core_types import RunPhase
    from rl_coach.exploration_policies.additive_noise import AdditiveNoise
    from rl_coach.schedules import LinearSchedule
    from rl_coach.spaces import BoxActionSpace
    for k, (E, A, seed) in enumerate(ACTING):
        high = (rng.rand(A) * 3 + 0.5).astype(np.float32)
        means = (rng.randn(E, A) * high).astype(np.float32)
        stds = np.exp(rng.randn(A) * 0.5).astype(np.float32)[None].repeat(E, 0)
        schedule = LinearSchedule(0.5, 0.1, 7)
        pol = AdditiveNoise(BoxActionSpace(A, -high, high), schedule, 0.05)
        pol.change_phase(RunPhase.TRAIN)
        np.random.seed(seed)
        train = np.array([np.asarray(pol.get_action([means[e][None], stds[e][None]]), np.float64).reshape(A)
                          for e in range(E)])
        out["act%d_noise_after" % k] = np.float64(schedule.current_value)
        pol.change_phase(RunPhase.TEST)
        ev = np.array([np.asarray(pol.get_action([means[e][None], stds[e][None]])).reshape(A) for e in range(E)])
        out.update({"act%d_means" % k: means, "act%d_stds" % k: stds, "act%d_seed" % k: np.int64(seed),
                    "act%d_train" % k: train, "act%d_eval" % k: ev})
    out["n_acting"] = np.int64(len(ACTING))


def golden_parameters(out):
    from rl_coach.agents.ppo_agent import PPOAgentParameters
    ap = PPOAgentParameters()
    alg = ap.algorithm
    out["par_algorithm"] = np.array([alg.gae_lambda, alg.target_kl_divergence, alg.initial_kl_coefficient,
                                     alg.high_kl_penalty_coefficient, alg.value_targets_mix_fraction,
                                     alg.beta_entropy, alg.num_consecutive_playing_steps.num_steps, alg.discount,
                                     alg.num_consecutive_training_steps], dtype=np.float64)
    out["par_flags"] = np.array([alg.clip_likelihood_ratio_using_epsilon is None, alg.estimate_state_value_using_gae,
                                 alg.use_kl_regularization, alg.act_for_full_episodes])
    out["par_rescaler"] = np.array(alg.policy_gradient_rescaler.name)
    nets = []
    for name in ("critic", "actor"):
        n = ap.network_wrappers[name]
        nets.append([n.batch_size, n.learning_rate, n.optimizer_epsilon, n.adam_optimizer_beta1,
                     n.adam_optimizer_beta2, float(n.create_target_network), n.l2_regularization])
        out["par_%s_optimizer" % name] = np.array(n.optimizer_type)
        out["par_%s_schemes" % name] = np.array([str(n.input_embedders_parameters['observation'].scheme.value),
                                                 str(n.middleware_parameters.scheme.value)])
    out["par_networks"] = np.array(nets, dtype=np.float64)
    ex = {k.__name__: v for k, v in ap.exploration.items()}
    box = ex["BoxActionSpace"]
    out["par_box_exploration"] = np.array(type(box).__name__)
    out["par_box_noise"] = np.array([box.noise_schedule.initial_value, box.noise_schedule.final_value,
                                     box.noise_schedule.decay_steps, box.evaluation_noise,
                                     float(box.noise_as_percentage_from_action_space)])
    for name in ("rl_coach.environments.gym_environment", "rl_coach.graph_managers.graph_manager",
                 "rl_coach.graph_managers.basic_rl_graph_manager"):
        sys.modules.setdefault(name, mock.MagicMock())
    mod = importlib.import_module("rl_coach.presets.Mujoco_PPO")
    ap = mod.agent_params
    out["pre_mujoco"] = np.array([ap.network_wrappers['actor'].learning_rate,
                                  ap.network_wrappers['critic'].learning_rate, ap.algorithm.initial_kl_coefficient,
                                  ap.algorithm.gae_lambda])
    out["pre_mujoco_widths"] = np.array([[d.units for d in ap.network_wrappers[n].input_embedders_parameters[
        'observation'].scheme] + [d.units for d in ap.network_wrappers[n].middleware_parameters.scheme]
        for n in ("actor", "critic")], dtype=np.int64)
    out["pre_mujoco_observation_filters"] = np.array(
        [type(f).__name__ for flt in ap.input_filter.observation_filters.values() for f in flt.values()])
    out["pre_mujoco_reward_test_level"] = np.array(mod.preset_validation_params.reward_test_level)


def main():
    from oracle import ref_loader
    ref_loader.load()
    import rl_coach.agents.ppo_agent as ref_ppo
    ref_ppo.screen = mock.MagicMock()              # the agent's console logging
    rng = np.random.RandomState(2027)
    out = {}
    golden_advantages(out, rng)
    golden_train(out, rng)
    golden_kl(out)
    golden_acting(out, rng)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "ppo.npz"), **out)
    print("ppo", len(out), "arrays")


if __name__ == "__main__":
    main()
