"""Pins PAL and Mixed Monte Carlo to the unmodified reference: tests/golden/pal_mmc.npz.

  PALAgent.learn_from_batch               rl_coach/agents/pal_agent.py:70-112 (regular and persistent)
  MixedMonteCarloAgent.learn_from_batch   rl_coach/agents/mmc_agent.py:56-84
      stand-in networks, as in oracle/make_golden_agents.py: the fp32 TD targets handed to the train op, on crafted
      rows (argmax ties on Q_online(s'), terminal rows, adv == nadv, adv < nadv, adv > nadv, large returns)
  EpisodicExperienceReplay((Episodes, k)) rl_coach/memories/episodic/episodic_experience_replay.py: variable-length
      episodes stored one transition at a time, the counters after every store, seeded sample() draws with their
      n_step_discounted_rewards (0.99-discounted: Episode's default discount, core_types.py:700)
  parameter defaults                      PAL / MMC algorithm and agent parameters and the two presets' agent values

Run in the build container only:   python -m oracle.make_golden_pal_mmc          TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
from types import SimpleNamespace
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

B, A = 64, 6


def _inputs(rng):
    """Q arrays, transitions and returns with crafted rows"""
    q_next = rng.randn(B, A).astype(np.float32)
    q_select = rng.randn(B, A).astype(np.float32)
    q_target_s = rng.randn(B, A).astype(np.float32)
    q_online = rng.randn(B, A).astype(np.float32)
    actions = rng.randint(0, A, B).astype(np.int64)
    rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], B).astype(np.float64)
    dones = (rng.rand(B) < 0.2).astype(np.uint8)
    returns = rng.randn(B) * 20.0
    for i in range(0, 4):                                     # ties on Q_online(s'): np.argmax takes the first
        q_select[i, 1] = q_select[i, 4] = q_select[i].max() + 1.0
    dones[4:8] = 1                                            # terminal rows
    for i in range(8, 16):                                    # adv == nadv: Q_target(s) = Q_target(s'), a = a*
        q_target_s[i] = q_next[i]
        actions[i] = int(np.argmax(q_select[i]))
    for i in range(16, 20):                                   # adv = 0 < nadv: the taken action is Q_target(s)'s max
        actions[i] = int(np.argmax(q_target_s[i]))
    for i in range(20, 24):                                   # nadv = 0 < adv: a* is Q_target(s')'s max
        q_select[i] = q_next[i]
        actions[i] = (int(np.argmax(q_target_s[i])) + 1) % A
    returns[24:28] = [1.0e6 + 0.1, -3.0e5 - 0.7, 1.0e9 / 3.0, 123456.789]        # large returns
    q_online[28:30] *= np.float32(1000.0)
    return q_next, q_select, q_target_s, q_online, actions, rewards, dones, returns


def _batch(actions, rewards, dones, returns):
    from rl_coach.core_types import Batch, Transition
    ts = []
    for i in range(B):
        t = Transition(state={'observation': np.zeros(4, dtype=np.float32)}, action=int(actions[i]),
                       reward=float(rewards[i]), next_state={'observation': np.zeros(4, dtype=np.float32)},
                       game_over=bool(dones[i]))
        t.n_step_discounted_rewards = float(returns[i])
        ts.append(t)
    return Batch(ts)


def golden_prologues(out, rng):
    from rl_coach.agents.mmc_agent import MixedMonteCarloAgent
    from rl_coach.agents.pal_agent import PALAgent
    q_next, q_select, q_target_s, q_online, actions, rewards, dones, returns = _inputs(rng)
    out.update(q_next=q_next, q_select=q_select, q_target_s=q_target_s, q_online=q_online, actions=actions,
               rewards=rewards, game_overs=dones, returns=returns, discount=np.float64(0.99))
    batch = _batch(actions, rewards, dones, returns)
    ap = SimpleNamespace(network_wrappers={'main': SimpleNamespace(input_embedders_parameters={'observation': None})},
                         algorithm=SimpleNamespace(discount=0.99))
    for tag, alpha, rate in (("", 0.9, 0.1), ("_b", 0.35, 0.6)):
        for persistent in (False, True):
            rec, calls = {}, []

            def pp(pairs):
                calls.append(len(calls))
                return [q_next.copy(), q_select.copy()] if len(calls) == 1 else [q_target_s.copy(), q_online.copy()]
            net = SimpleNamespace(target_network="T", online_network="O", parallel_prediction=pp,
                                  train_and_sync_networks=lambda s, t: rec.update(t=np.array(t)) or (0.0, [0.0], 0.0))
            fake = SimpleNamespace(ap=ap, networks={'main': net}, alpha=alpha, persistent=persistent,
                                   monte_carlo_mixing_rate=rate)
            PALAgent.learn_from_batch(fake, batch)
            assert rec["t"].dtype == np.float32
            out["pal%s%s_targets" % ("_persistent" if persistent else "", tag)] = rec["t"]
        rec = {}
        net = SimpleNamespace(target_network="T", online_network=SimpleNamespace(predict=lambda s: q_select.copy()),
                              parallel_prediction=lambda pairs: [q_next.copy(), q_online.copy()],
                              train_and_sync_networks=lambda s, t: rec.update(t=np.array(t)) or (0.0, [0.0], 0.0))
        fake = SimpleNamespace(ap=ap, networks={'main': net}, mixing_rate=rate)
        MixedMonteCarloAgent.learn_from_batch(fake, batch)
        assert rec["t"].dtype == np.float32
        out["mmc%s_targets" % tag] = rec["t"]
        out["alpha_rate%s" % tag] = np.array([alpha, rate])


def golden_episodic(out, rng, k=3):
    """an Episodes-sized replay fed transition by transition; counters after every store, samples at checkpoints"""
    from rl_coach.core_types import Transition
    from rl_coach.memories.episodic.episodic_experience_replay import EpisodicExperienceReplay
    from rl_coach.memories.memory import MemoryGranularity
    mem = EpisodicExperienceReplay((MemoryGranularity.Episodes, k))
    lengths = [3, 1, 5, 2, 4, 6, 1, 3, 2]
    rewards = np.round(rng.randn(sum(lengths)) * 4.0, 3)
    counters, samples, sample_at = [], [], []
    sid = 0
    for L in lengths:
        for j in range(L):
            mem.store(Transition(state={'observation': np.array([sid], dtype=np.float32)}, action=0,
                                 reward=float(rewards[sid]),
                                 next_state={'observation': np.array([sid + 1], dtype=np.float32)},
                                 game_over=j == L - 1))
            counters.append([mem.num_transitions(), mem.num_transitions_in_complete_episodes(),
                             mem.num_complete_episodes(), mem.length()])
            sid += 1
            if j == 0 and mem.num_complete_episodes() >= 1 or j == L - 1:
                np.random.seed(1000 + sid)
                ts = mem.sample(7)
                samples.append([[float(t.state['observation'][0]), float(t.n_step_discounted_rewards)] for t in ts])
                sample_at.append(sid)
    out["ep_k"] = np.int64(k)
    out["ep_lengths"] = np.array(lengths, dtype=np.int64)
    out["ep_rewards"] = rewards
    out["ep_counters"] = np.array(counters, dtype=np.int64)          # [stores, 4]: transitions, in complete, complete, length
    out["ep_samples"] = np.array(samples, dtype=np.float64)          # [checks, 7, 2]: state id, return
    out["ep_sample_at"] = np.array(sample_at, dtype=np.int64)        # the number of stores before each check


def golden_parameters(out):
    from rl_coach.agents.mmc_agent import MixedMonteCarloAgentParameters
    from rl_coach.agents.pal_agent import PALAgentParameters
    pal, mmc = PALAgentParameters(), MixedMonteCarloAgentParameters()
    out["par_pal"] = np.array([pal.algorithm.pal_alpha, float(pal.algorithm.persistent_advantage_learning),
                               pal.algorithm.monte_carlo_mixing_rate, pal.algorithm.discount])
    out["par_mmc"] = np.array([mmc.algorithm.monte_carlo_mixing_rate, mmc.algorithm.discount])
    for tag, ap in (("pal", pal), ("mmc", mmc)):
        out["par_%s_memory" % tag] = np.array(type(ap.memory).__name__)
        out["par_%s_max_size" % tag] = np.array([ap.memory.max_size[0].value, ap.memory.max_size[1]], dtype=np.int64)
        out["par_%s_copy_steps" % tag] = np.int64(ap.algorithm.num_steps_between_copying_online_weights_to_target
                                                  .num_steps)
    # the presets' agent parameters (the environment modules are stubbed: only agent_params is read)
    for name in ("rl_coach.environments.gym_environment", "rl_coach.environments.doom_environment",
                 "rl_coach.graph_managers.graph_manager", "rl_coach.graph_managers.basic_rl_graph_manager"):
        sys.modules.setdefault(name, mock.MagicMock())
    import importlib
    for tag, preset in (("cartpole_pal", "CartPole_PAL"), ("doom_mmc", "Doom_Health_MMC")):
        ap = importlib.import_module("rl_coach.presets." + preset).agent_params
        net, alg = ap.network_wrappers['main'], ap.algorithm
        out["pre_%s" % tag] = np.array([net.learning_rate, float(net.replace_mse_with_huber_loss), alg.discount,
                                        alg.num_steps_between_copying_online_weights_to_target.num_steps,
                                        alg.num_consecutive_playing_steps.num_steps, ap.memory.max_size[0].value,
                                        ap.memory.max_size[1], net.batch_size])
        out["pre_%s_path" % tag] = np.array(ap.path.split(":")[-1])


def main():
    from oracle import ref_loader
    ref_loader.load()
    rng = np.random.RandomState(4242)
    out = {}
    golden_prologues(out, rng)
    golden_episodic(out, rng)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "pal_mmc.npz"), **out)
    print("pal_mmc", len(out), "arrays")


if __name__ == "__main__":
    main()
