"""Pins Quantile Regression DQN to the unmodified reference: tests/golden/qr_dqn.npz.

  QuantileRegressionDQNAgent.learn_from_batch   rl_coach/agents/qr_dqn_agent.py:97-137 on a stand-in network whose
      parallel_prediction returns planted fp32 quantiles of target(s') and online(s) and whose train_and_sync_networks
      records what it is handed: the TD targets, `output_0_0` (the [b, a] pairs) and `output_0_1` (the midpoints).
      Cases: A in {2, 6, 18}, N in {1, 7, 50, 200}, B = 32 and 64, discount 0.99 and 0.9, terminal rows, large /
      negative / fractional rewards.  Every taken row is free of ties (np.argsort's default kind leaves their order to
      the numpy build) and the best action's Q' beats the runner-up by a margin (np.dot's summation order is
      unspecified, so a near tie could flip the argmax).
  parameter defaults   the QR-DQN parameter classes and the Atari_QR_DQN / CartPole_QR_DQN presets' agent values

Run in the build container only:   python -m oracle.make_golden_qr_dqn          TEST INFRASTRUCTURE ONLY.
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

# (tag, A, N, B, discount)
CASES = [("a2_n50", 2, 50, 64, 0.99), ("a6_n200", 6, 200, 32, 0.99), ("a18_n7", 18, 7, 64, 0.9),
         ("a2_n1", 2, 1, 32, 0.9), ("a6_n7", 6, 7, 32, 0.9)]
MARGIN = 1e-6


def _planted(rng, A, N, B):
    """fp32 quantiles [B, A, N] of target(s') with a clear best action, and of online(s) with tie-free rows"""
    nxt = (rng.randn(B, A, N) * 3.0).astype(np.float32)
    for b in range(B):
        q = np.sort(nxt[b].astype(np.float64).mean(axis=1))
        if A > 1 and q[-1] - q[-2] < MARGIN * max(1.0, abs(q[-1])):
            nxt[b, int(np.argmax(nxt[b].astype(np.float64).mean(axis=1)))] += np.float32(0.5)
    onl = (rng.randn(B, A, N) * 3.0).astype(np.float32)
    return nxt, onl


def golden_cases(out, rng):
    from rl_coach.agents.qr_dqn_agent import QuantileRegressionDQNAgent
    from rl_coach.core_types import Batch, Transition
    for tag, A, N, B, discount in CASES:
        nxt, onl = _planted(rng, A, N, B)
        actions = rng.randint(0, A, B).astype(np.int64)
        rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, -2.5e3, 1.0e6 + 0.1, 1.0 / 3.0], B)
        dones = (rng.rand(B) < 0.25).astype(np.uint8)
        dones[:3], dones[3:6] = 1, 0
        for b in range(B):                                        # the generator's own guards
            row = onl[b, actions[b]]
            assert len(np.unique(row)) == N, "tied quantiles in a taken row"
            q = np.sort(nxt[b].astype(np.float64).mean(axis=1))
            assert A == 1 or q[-1] - q[-2] >= MARGIN * max(1.0, abs(q[-1])), "near tie of the best actions"
        ts = [Transition(state={'observation': np.zeros(4, dtype=np.float32)}, action=int(actions[i]),
                         reward=float(rewards[i]), next_state={'observation': np.zeros(4, dtype=np.float32)},
                         game_over=bool(dones[i])) for i in range(B)]
        rec = {}

        def train(inputs, targets):
            rec.update(t=np.array(targets), a=np.array(inputs['output_0_0']), tau=np.array(inputs['output_0_1']))
            return 0.0, [0.0], 0.0
        net = SimpleNamespace(target_network="T", online_network="O", train_and_sync_networks=train,
                              parallel_prediction=lambda pairs: [nxt.copy(), onl.copy()])
        ap = SimpleNamespace(network_wrappers={'main': SimpleNamespace(input_embedders_parameters={'observation': 0})},
                             algorithm=SimpleNamespace(discount=discount, atoms=N))
        fake = SimpleNamespace(ap=ap, networks={'main': net}, q_values=SimpleNamespace(add_sample=lambda x: None),
                               quantile_probabilities=np.ones(N) / float(N))
        fake.get_q_values = lambda qv: QuantileRegressionDQNAgent.get_q_values(fake, qv)
        QuantileRegressionDQNAgent.learn_from_batch(fake, Batch(ts))
        p = "c_%s_" % tag
        out[p + "next"], out[p + "online"], out[p + "actions"] = nxt, onl, actions
        out[p + "rewards"], out[p + "dones"], out[p + "discount"] = rewards, dones, np.float64(discount)
        out[p + "targets"] = rec["t"]                             # float64 [B, N]: the feed rounds it to fp32
        out[p + "output_0_0"] = rec["a"]
        out[p + "output_0_1"] = rec["tau"]                        # float64 [B, N], fed as fp32
        out[p + "target_actions"] = np.argmax(fake.get_q_values(nxt), axis=1)


def golden_parameters(out):
    from rl_coach.agents.qr_dqn_agent import QuantileRegressionDQNAgentParameters
    for name in ("rl_coach.environments.gym_environment", "rl_coach.graph_managers.graph_manager",
                 "rl_coach.graph_managers.basic_rl_graph_manager"):
        sys.modules.setdefault(name, mock.MagicMock())

    def values(ap):
        net, alg, ex = ap.network_wrappers['main'], ap.algorithm, ap.exploration
        return np.array([net.learning_rate, net.optimizer_epsilon, net.adam_optimizer_beta1, net.adam_optimizer_beta2,
                         net.batch_size, float(net.replace_mse_with_huber_loss), float(net.create_target_network),
                         alg.atoms, alg.huber_loss_interval, alg.discount,
                         alg.num_steps_between_copying_online_weights_to_target.num_steps,
                         alg.num_consecutive_playing_steps.num_steps, alg.num_consecutive_training_steps,
                         ap.memory.max_size[0].value, ap.memory.max_size[1],
                         ex.epsilon_schedule.initial_value, ex.epsilon_schedule.final_value,
                         ex.epsilon_schedule.decay_steps, ex.evaluation_epsilon], dtype=np.float64)
    ap = QuantileRegressionDQNAgentParameters()
    out["par_defaults"] = values(ap)
    out["par_memory"] = np.array(type(ap.memory).__name__)
    out["par_copy_unit"] = np.array(type(ap.algorithm.num_steps_between_copying_online_weights_to_target).__name__)
    for tag, preset in (("atari", "Atari_QR_DQN"), ("cartpole", "CartPole_QR_DQN")):
        pap = importlib.import_module("rl_coach.presets." + preset).agent_params
        out["pre_%s" % tag] = values(pap)
        out["pre_%s_path" % tag] = np.array(pap.path.split(":")[-1])


def main():
    from oracle import ref_loader
    ref_loader.load()
    rng = np.random.RandomState(2024)
    out = {}
    golden_cases(out, rng)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "qr_dqn.npz"), **out)
    print("qr_dqn", len(out), "arrays")


if __name__ == "__main__":
    main()
