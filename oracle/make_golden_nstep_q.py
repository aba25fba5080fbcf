"""Pins the N-step Q-learning agent to the unmodified reference: tests/golden/nstep_q.npz.

  NStepQAgent.learn_from_batch   rl_coach/agents/n_step_q_agent.py:99-140, stand-in networks (as in
      oracle/make_golden_pal_mmc.py): the fp32 targets handed to accumulate_gradients for both horizons (and an unknown
      one) on crafted segments: lengths 1, 2, 5, 7, 23, terminal and bootstrapped last rows, rewards
      {-1, 0, 1, 0.37, 11, r / 200} and one segment of integer rewards, discount 0.99 / 0.9, A in {2, 6, 18}, Q values
      up to 1e3
  NStepQAgent.train              n_step_q_agent.py:142-153 + policy_optimization_agent.py:85-135 after every env step
      of a scripted episode stream (lengths 1, 3, 5, 6, 10, 11, 23) at t_max 5 and 3: the learned segments, the
      target copies under EnvironmentSteps(7) and TrainingSteps(3), training_iteration
  parameter defaults             NStepQ agent / algorithm / network parameters and the two presets' agent values

Run in the build container only:   python -m oracle.make_golden_nstep_q          TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
from types import SimpleNamespace
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# (length, actions, discount, terminal, reward kind)
CASES = [(1, 2, 0.99, False, "mix"), (1, 6, 0.99, True, "mix"), (2, 2, 0.9, False, "mix"), (5, 6, 0.99, False, "mix"),
         (5, 18, 0.99, True, "mix"), (7, 18, 0.9, False, "mix"), (23, 6, 0.99, False, "mix"),
         (23, 2, 0.99, True, "mix"), (5, 6, 0.99, False, "int"), (3, 6, 0.99, True, "int"),
         (7, 2, 0.99, False, "scaled"), (5, 18, 0.9, False, "big")]
HORIZONS = ("N-Step", "1-Step", "none")
EPISODES = [1, 3, 5, 6, 10, 11, 23]


def _case(rng, L, A, terminal, kind):
    q_online = (rng.randn(L, A) * 3).astype(np.float32)
    q_next = (rng.randn(L, A) * 3).astype(np.float32)
    if kind == "big":
        q_online *= np.float32(300.0)
        q_next *= np.float32(300.0)
    actions = rng.randint(0, A, L).astype(np.int64)
    if kind == "int":
        rewards = rng.randint(-3, 4, L).astype(np.int64)
    elif kind == "scaled":
        rewards = rng.choice([-1.0, 0.0, 1.0], L) * (1 / 200.)
    else:
        rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0, 1 / 200.], L).astype(np.float64)
    game_overs = np.zeros(L, dtype=bool)
    game_overs[-1] = terminal
    return q_online, q_next, actions, rewards, game_overs


def _batch(actions, rewards, game_overs):
    from rl_coach.core_types import Batch, Transition
    ts = [Transition(state={'observation': np.zeros(4, dtype=np.float32)}, action=int(actions[i]),
                     reward=rewards[i].item(), next_state={'observation': np.full(4, i, dtype=np.float32)},
                     game_over=bool(game_overs[i])) for i in range(len(actions))]
    return Batch(ts)


def golden_targets(out, rng):
    from rl_coach.agents.n_step_q_agent import NStepQAgent
    for c, (L, A, discount, terminal, kind) in enumerate(CASES):
        q_online, q_next, actions, rewards, game_overs = _case(rng, L, A, terminal, kind)
        batch = _batch(actions, rewards, game_overs)
        assert batch.rewards().dtype == (np.int64 if kind == "int" else np.float64)
        out.update({"c%d_q_online" % c: q_online, "c%d_q_next" % c: q_next, "c%d_actions" % c: actions,
                    "c%d_rewards" % c: rewards, "c%d_game_overs" % c: game_overs.astype(np.uint8),
                    "c%d_discount" % c: np.float64(discount)})
        for horizon in HORIZONS:
            rec = {}

            def predict_target(s):
                n = len(s['observation'])
                return q_next.copy() if n == L else q_next[-1:].copy()       # last_sample(): one row
            net = SimpleNamespace(online_network=SimpleNamespace(
                predict=lambda s: q_online.copy(),
                accumulate_gradients=lambda s, t: rec.update(t=np.array(t[0])) or (0.0, [0.0], 0.0)),
                target_network=SimpleNamespace(predict=predict_target))
            fake = SimpleNamespace(ap=SimpleNamespace(
                network_wrappers={'main': SimpleNamespace(input_embedders_parameters={'observation': None})},
                algorithm=SimpleNamespace(targets_horizon=horizon, discount=discount)),
                networks={'main': net}, q_values=SimpleNamespace(add_sample=lambda x: None),
                value_loss=SimpleNamespace(add_sample=lambda x: None))
            NStepQAgent.learn_from_batch(fake, batch)
            assert rec["t"].dtype == np.float32
            out["c%d_%s_targets" % (c, horizon.lower().replace("-", ""))] = rec["t"]
    out["n_cases"] = np.int64(len(CASES))


def golden_schedule(out):
    from rl_coach.agents.agent import Agent
    from rl_coach.agents.n_step_q_agent import NStepQAgent
    from rl_coach.core_types import Episode, EnvironmentSteps, TrainingSteps, Transition
    for t_max in (5, 3):
        for tag, method in (("env7", EnvironmentSteps(7)), ("train3", TrainingSteps(3))):
            learned, copies = [], []
            fake = SimpleNamespace(
                ap=SimpleNamespace(algorithm=SimpleNamespace(num_steps_between_gradient_updates=t_max,
                                                             num_steps_between_copying_online_weights_to_target=method,
                                                             rate_for_copying_weights_to_target=1.0,
                                                             apply_gradients_every_x_episodes=1)),
                total_steps_counter=0, training_iteration=0, last_target_network_update_step=0,
                last_gradient_update_step_idx=0, current_episode=0, policy_gradient_rescaler=None,
                agent_logger=SimpleNamespace(create_signal_value=lambda *a, **k: None),
                post_training_commands=lambda: None)
            fake._should_update_online_weights_to_target = lambda: Agent._should_update_online_weights_to_target(fake)
            net = SimpleNamespace(has_target=True, set_is_training=lambda x: None,
                                  apply_gradients_and_sync_networks=lambda: None,
                                  update_target_network=lambda rate: copies.append(fake.total_steps_counter))
            fake.networks = {'main': net}
            for n in EPISODES:
                fake.current_episode_buffer = Episode(discount=0.99)
                for k in range(n):
                    fake.total_steps_counter += 1                                  # act()
                    fake.current_episode_buffer.insert(Transition(
                        state={'observation': np.zeros(1)}, action=0, reward=0.0,
                        next_state={'observation': np.zeros(1)}, game_over=k == n - 1))
                    if k == n - 1:
                        fake.current_episode += 1                                  # handle_episode_ended
                    first = fake.last_gradient_update_step_idx

                    def lfb(batch, first=first):
                        learned.append((first, first + batch.size, fake.total_steps_counter))
                        return 0.0, [0.0], 0.0
                    fake.learn_from_batch = lfb
                    NStepQAgent.train(fake)
            key = "sch_t%d_%s" % (t_max, tag)
            out[key + "_segments"] = np.array(learned, dtype=np.int64)
            out[key + "_copies"] = np.array(copies, dtype=np.int64)
            out[key + "_training_iteration"] = np.int64(fake.training_iteration)
    out["sch_episodes"] = np.array(EPISODES, dtype=np.int64)


def golden_parameters(out):
    from rl_coach.agents.n_step_q_agent import NStepQAgentParameters
    ap = NStepQAgentParameters()
    alg, net = ap.algorithm, ap.network_wrappers['main']
    out["par_algorithm"] = np.array([alg.num_steps_between_gradient_updates, alg.apply_gradients_every_x_episodes,
                                     alg.num_steps_between_copying_online_weights_to_target.num_steps, alg.discount,
                                     alg.rate_for_copying_weights_to_target])
    out["par_copy_method"] = np.array(type(alg.num_steps_between_copying_online_weights_to_target).__name__)
    out["par_horizon"] = np.array(alg.targets_horizon)
    out["par_network"] = np.array([net.learning_rate, net.adam_optimizer_beta1, net.adam_optimizer_beta2,
                                   net.optimizer_epsilon, float(net.replace_mse_with_huber_loss),
                                   float(net.create_target_network), float(net.async_training),
                                   float(net.shared_optimizer)])
    sch = ap.exploration.epsilon_schedule
    out["par_epsilon"] = np.array([sch.initial_value, sch.final_value, sch.decay_steps, ap.exploration.evaluation_epsilon])
    for name in ("rl_coach.environments.gym_environment", "rl_coach.graph_managers.graph_manager",
                 "rl_coach.graph_managers.basic_rl_graph_manager"):
        sys.modules.setdefault(name, mock.MagicMock())
    import importlib
    for tag, preset in (("cartpole", "CartPole_NStepQ"), ("atari", "Atari_NStepQ")):
        mod = importlib.import_module("rl_coach.presets." + preset)
        ap = mod.agent_params
        net, alg = ap.network_wrappers['main'], ap.algorithm
        out["pre_%s" % tag] = np.array([net.learning_rate, alg.discount,
                                        alg.num_steps_between_copying_online_weights_to_target.num_steps,
                                        alg.num_steps_between_gradient_updates])
        emb = net.input_embedders_parameters['observation'].scheme
        mid = net.middleware_parameters.scheme
        out["pre_%s_embedder" % tag] = np.array(
            [[c.num_filters, c.kernel_size, c.strides] for c in emb] if isinstance(emb, list) else [], dtype=np.int64)
        out["pre_%s_middleware" % tag] = np.array([d.units for d in mid] if isinstance(mid, list) else [],
                                                  dtype=np.int64)
        rf = getattr(ap.input_filter, "reward_filters", {}) if ap.input_filter is not None else {}
        out["pre_%s_reward_rescale" % tag] = np.array([f.rescale_factor for f in rf.values()], dtype=np.float64)
        out["pre_%s_workers" % tag] = np.int64(getattr(mod.preset_validation_params, "num_workers", 1))


def main():
    from oracle import ref_loader
    ref_loader.load()
    rng = np.random.RandomState(2024)
    out = {}
    golden_targets(out, rng)
    golden_schedule(out)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "nstep_q.npz"), **out)
    print("nstep_q", len(out), "arrays")


if __name__ == "__main__":
    main()
