"""Pins discrete ClippedPPO to the unmodified reference: tests/golden/clipped_ppo_discrete.npz.

  ClippedPPOAgent.choose_action     rl_coach/agents/clipped_ppo_agent.py:352-354 -> policy_optimization_agent.py:144-162
      with a stand-in network (its softmax per environment) and the real Categorical policy, under np.random.seed:
      actions in training and evaluation, and the clipping schedule's value after every call
  ClippedPPOAgent.train_network     clipped_ppo_agent.py:209-308 on a discrete rollout with a stand-in network: what each
      minibatch feeds (the fed rows, the 1-D actions, the old policy's probabilities, the rescaler's input and value)
  parameter defaults                ClippedPPOAgentParameters' exploration classes and the CartPole_ClippedPPO preset

Run in the build container only:   python -m oracle.make_golden_clipped_ppo_discrete     TEST INFRASTRUCTURE ONLY.
"""
import importlib
import os
import random
import sys
from types import SimpleNamespace
from unittest import mock

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

# acting: (environments, actions, seed, LinearSchedule(initial, final, decay steps) of the clipping rescaler)
ACTING = [(1, 2, 500, (1.0, 0.0, 1000000)), (8, 2, 501, (1.0, 0.0, 5)), (16, 3, 502, (0.5, 0.1, 7)),
          (5, 18, 503, (1.0, 0.0, 1000000)), (3, 4, 504, (1.0, 0.2, 2))]
# train_network: (rows, actions, batch size, epochs, rescaler value, seed)
TRAIN = [(256, 2, 64, 2, 1.0, 600), (192, 18, 64, 3, 0.75, 601)]


def _softmax(z):
    e = np.exp(z - z.max(1, keepdims=True))
    return (e / e.sum(1, keepdims=True)).astype(np.float32)


def golden_acting(out, rng):
    from rl_coach.agents.clipped_ppo_agent import ClippedPPOAgent, ClippedPPOAlgorithmParameters
    from rl_coach.core_types import RunPhase
    from rl_coach.exploration_policies.categorical import Categorical
    from rl_coach.schedules import LinearSchedule
    from rl_coach.spaces import DiscreteActionSpace
    for k, (E, A, seed, sched) in enumerate(ACTING):
        probs = _softmax(rng.randn(E, A) * 1.5)
        alg = ClippedPPOAlgorithmParameters()
        alg.clipping_decay_schedule = LinearSchedule(*sched)
        agent = ClippedPPOAgent.__new__(ClippedPPOAgent)          # no network: a stand-in prediction per state
        agent.ap = SimpleNamespace(algorithm=alg)
        agent.spaces = SimpleNamespace(action=DiscreteActionSpace(A))
        agent.exploration_policy = Categorical(DiscreteActionSpace(A))
        agent.entropy = SimpleNamespace(add_sample=lambda x: None)
        agent.get_prediction = lambda state: probs[state][None]
        agent.exploration_policy.change_phase(RunPhase.TRAIN)
        np.random.seed(seed)
        train, values = [], []
        for e in range(E):
            train.append(agent.choose_action(e).action)
            values.append(alg.clipping_decay_schedule.current_value)
        agent.exploration_policy.change_phase(RunPhase.TEST)
        ev = []
        for e in range(E):
            ev.append(agent.choose_action(e).action)
            values.append(alg.clipping_decay_schedule.current_value)
        out.update({"act%d_probs" % k: probs, "act%d_seed" % k: np.int64(seed),
                    "act%d_schedule" % k: np.array(sched, dtype=np.float64),
                    "act%d_train" % k: np.array(train, dtype=np.int64), "act%d_eval" % k: np.array(ev, dtype=np.int64),
                    "act%d_clipping" % k: np.array(values, dtype=np.float64)})
    out["n_acting"] = np.int64(len(ACTING))


def golden_train(out, rng):
    from rl_coach.agents.clipped_ppo_agent import ClippedPPOAgent, ClippedPPOAlgorithmParameters
    from rl_coach.core_types import Batch, Transition
    from rl_coach.schedules import ConstantSchedule
    from rl_coach.spaces import DiscreteActionSpace
    for c, (N, A, B, epochs, rescaler, seed) in enumerate(TRAIN):
        actions = rng.randint(0, A, N).astype(np.int64)
        probs = _softmax(rng.randn(N, A))
        ts = []
        for i in range(N):
            t = Transition(state={'observation': np.array([i, 0.5], dtype=np.float32)}, action=int(actions[i]),
                           reward=0.0, next_state={'observation': np.zeros(2, dtype=np.float32)}, game_over=False)
            t.info['advantage'] = float(rng.randn())
            t.info['gae_based_value_target'] = float(rng.randn())
            t.n_step_discounted_rewards = 0.0
            ts.append(t)
        alg = ClippedPPOAlgorithmParameters()
        alg.clipping_decay_schedule = ConstantSchedule(rescaler)
        fed = []
        rows = lambda s: s['observation'][:, 0].astype(np.int64)         # noqa: E731

        def train_and_sync_networks(inputs, targets, additional_fetches=None):
            fed.append(dict(inputs))
            return 0.0, [0.0, 0.0], 0.0, [np.float32(0)] * 4
        head = SimpleNamespace(kl_divergence=None, entropy=None, likelihood_ratio=None, clipped_likelihood_ratio=None)
        net = SimpleNamespace(
            online_network=SimpleNamespace(output_heads=[None, head]), train_and_sync_networks=train_and_sync_networks,
            target_network=SimpleNamespace(predict=lambda s: [np.zeros((len(rows(s)), 1), np.float32),
                                                              probs[rows(s)]]))
        sig = SimpleNamespace(add_sample=lambda x: None)
        fake = SimpleNamespace(
            ap=SimpleNamespace(algorithm=alg, network_wrappers={'main': SimpleNamespace(
                batch_size=B, input_embedders_parameters={'observation': None}, learning_rate_decay_rate=0,
                learning_rate=3e-4)}),
            networks={'main': net}, spaces=SimpleNamespace(action=DiscreteActionSpace(A)), unclipped_grads=sig,
            value_targets=sig, likelihood_ratio=sig, clipped_likelihood_ratio=sig, value_loss=sig, policy_loss=sig,
            loss=sig, entropy=sig, kl_divergence=sig, total_kl_divergence_during_training_process=0.0)
        random.seed(seed)
        ClippedPPOAgent.train_network(fake, Batch(ts), epochs)
        assert len(fed) == epochs * (N // B), len(fed)
        keys = sorted(fed[0])
        assert all(sorted(f) == keys for f in fed)
        out.update({"train%d_shape" % c: np.array([N, A, B, epochs], dtype=np.int64),
                    "train%d_rescaler" % c: np.float64(rescaler), "train%d_actions" % c: actions,
                    "train%d_probs" % c: probs, "train%d_keys" % c: np.array(keys),
                    "train%d_rows" % c: np.stack([rows(f) for f in fed]),
                    "train%d_fed_actions" % c: np.stack([np.asarray(f['output_1_0']) for f in fed]),
                    "train%d_fed_actions_ndim" % c: np.array([np.asarray(f['output_1_0']).ndim for f in fed]),
                    "train%d_fed_old" % c: np.stack([np.asarray(f['output_1_1']) for f in fed]),
                    "train%d_fed_rescaler" % c: np.array([f['output_1_2'] for f in fed], dtype=np.float64)})
    out["n_train"] = np.int64(len(TRAIN))


def golden_parameters(out):
    from rl_coach.agents.clipped_ppo_agent import ClippedPPOAgentParameters
    ap = ClippedPPOAgentParameters()
    out["par_exploration"] = np.array(sorted("%s:%s" % (k.__name__, type(v).__name__) for k, v in ap.exploration.items()))
    for name in ("rl_coach.environments.gym_environment", "rl_coach.graph_managers.graph_manager",
                 "rl_coach.graph_managers.basic_rl_graph_manager"):
        sys.modules.setdefault(name, mock.MagicMock())
    mod = importlib.import_module("rl_coach.presets.CartPole_ClippedPPO")
    ap = mod.agent_params
    net, alg = ap.network_wrappers['main'], ap.algorithm
    sched = alg.clipping_decay_schedule
    out["pre_cartpole_network"] = np.array([net.learning_rate, net.batch_size, net.optimizer_epsilon,
                                            net.adam_optimizer_beta2], dtype=np.float64)
    out["pre_cartpole_widths"] = np.array([d.units for d in net.input_embedders_parameters['observation'].scheme] +
                                          [d.units for d in net.middleware_parameters.scheme], dtype=np.int64)
    out["pre_cartpole_activations"] = np.array([net.input_embedders_parameters['observation'].activation_function,
                                                net.middleware_parameters.activation_function])
    out["pre_cartpole_algorithm"] = np.array([alg.clip_likelihood_ratio_using_epsilon, alg.beta_entropy,
                                              alg.gae_lambda, alg.discount, alg.optimization_epochs,
                                              float(alg.estimate_state_value_using_gae),
                                              alg.num_steps_between_copying_online_weights_to_target.num_steps],
                                             dtype=np.float64)
    out["pre_cartpole_schedule"] = np.array([type(sched).__name__])
    out["pre_cartpole_schedule_values"] = np.array([sched.initial_value, sched.final_value, sched.decay_steps],
                                                   dtype=np.float64)
    out["pre_cartpole_observation_filters"] = np.array(
        [type(f).__name__ for flt in ap.pre_network_filter.observation_filters.values() for f in flt.values()])


def main():
    from oracle import ref_loader
    ref_loader.load()
    import rl_coach.agents.clipped_ppo_agent as ref_cppo
    ref_cppo.screen = mock.MagicMock()              # the agent's console logging
    rng = np.random.RandomState(2028)
    out = {}
    golden_acting(out, rng)
    golden_train(out, rng)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "clipped_ppo_discrete.npz"), **out)
    print("clipped_ppo_discrete", len(out), "arrays")


if __name__ == "__main__":
    main()
