"""Pins NAF to the unmodified reference: tests/golden/naf.npz.

  NAFAgent.learn_from_batch     rl_coach/agents/naf_agent.py:80-99 on a stand-in network whose target `predict` returns
                                planted fp32 V(s') values and whose train_and_sync_networks records what it is handed:
                                the fp32 TD targets and the `output_0_0` action array (A in {1, 6}, B = 64,
                                discount 0.99 and 0.9, terminal rows, large / negative / fractional rewards)
  OUProcess                     rl_coach/exploration_policies/ou_process.py:43-84: E = 4 policies stepped in turn from
                                numpy's global generator (A in {1, 3, 6}, 60 steps), with resets and a TEST stretch
  parameter defaults            NAFAgentParameters, OUProcessParameters, NAFHeadParameters.activation_function

Run in the build container only:   python -m oracle.make_golden_naf          TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

B = 64
E, STEPS = 4, 60
RESETS = {17: (0, 2), 33: (1,), 34: (3,)}        # step -> environments reset before that step
TEST_STEPS = range(40, 48)                       # the TEST phase: no noise, nothing drawn


def golden_targets(out, rng):
    from rl_coach.agents.naf_agent import NAFAgent
    from rl_coach.core_types import Batch, Transition
    for A in (1, 6):
        for tag, discount in (("", 0.99), ("_g09", 0.9)):
            v = (rng.randn(B, 1) * 30.0).astype(np.float32)
            rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, -2.5e3, 1.0e6 + 0.1, 1.0 / 3.0], B)
            dones = (rng.rand(B) < 0.25).astype(np.uint8)
            dones[:3] = 1
            dones[3:6] = 0
            actions = np.tanh(rng.randn(B, A)).astype(np.float32)
            ts = [Transition(state={'observation': np.zeros(3, dtype=np.float32)}, action=actions[i].copy(),
                             reward=float(rewards[i]), next_state={'observation': np.zeros(3, dtype=np.float32)},
                             game_over=bool(dones[i])) for i in range(B)]
            rec = {}

            def train(inputs, targets):
                rec.update(t=np.array(targets), u=np.array(inputs['output_0_0']))
                return 0.0, [0.0], 0.0
            target_net = SimpleNamespace(output_heads=[SimpleNamespace(V="V")],
                                         predict=lambda inputs, outputs, squeeze_output: v.copy())
            net = SimpleNamespace(target_network=target_net, train_and_sync_networks=train)
            ap = SimpleNamespace(network_wrappers={'main': SimpleNamespace(input_embedders_parameters={'observation': 0})},
                                 algorithm=SimpleNamespace(discount=discount))
            fake = SimpleNamespace(ap=ap, networks={'main': net}, TD_targets=SimpleNamespace(add_sample=lambda x: None))
            NAFAgent.learn_from_batch(fake, Batch(ts))
            k = "a%d%s" % (A, tag)
            out["td_%s_v" % k], out["td_%s_rewards" % k], out["td_%s_dones" % k] = v, rewards, dones
            out["td_%s_discount" % k] = np.float64(discount)
            out["td_%s_targets" % k] = rec["t"]               # as handed to the train op (fp64: the feed casts)
            out["td_%s_actions" % k] = actions
            out["td_%s_output_0_0" % k] = rec["u"]


def golden_ou(out, rng):
    from rl_coach.core_types import RunPhase
    from rl_coach.exploration_policies.ou_process import OUProcess
    from rl_coach.spaces import BoxActionSpace
    for A in (1, 3, 6):
        pols = [OUProcess(BoxActionSpace(A, -2.0, 2.0)) for _ in range(E)]
        for p in pols:
            p.change_phase(RunPhase.TRAIN)
        mus = np.tanh(rng.randn(STEPS, E, A)).astype(np.float32)
        acts = np.zeros((STEPS, E, A))
        np.random.seed(100 + A)
        for step in range(STEPS):
            for e in RESETS.get(step, ()):
                pols[e].reset()
            phase = RunPhase.TEST if step in TEST_STEPS else RunPhase.TRAIN
            for e in range(E):
                pols[e].change_phase(phase)
                acts[step, e] = pols[e].get_action(mus[step, e][None, :])      # predict()'s [1, A] output
        out["ou_a%d_mu" % A], out["ou_a%d_actions" % A] = mus, acts
    out["ou_seed_base"] = np.int64(100)
    out["ou_resets"] = np.array([[s, e] for s, es in sorted(RESETS.items()) for e in es], dtype=np.int64)
    out["ou_test_steps"] = np.array(list(TEST_STEPS), dtype=np.int64)


def golden_parameters(out):
    from rl_coach.agents.naf_agent import NAFAgentParameters
    from rl_coach.architectures.head_parameters import NAFHeadParameters
    from rl_coach.exploration_policies.ou_process import OUProcessParameters
    ap = NAFAgentParameters()
    net, alg = ap.network_wrappers['main'], ap.algorithm
    out["par_network"] = np.array([net.learning_rate, net.adam_optimizer_beta1, net.adam_optimizer_beta2,
                                   net.optimizer_epsilon, net.batch_size, float(net.replace_mse_with_huber_loss),
                                   float(net.create_target_network)])
    out["par_algorithm"] = np.array([alg.num_consecutive_training_steps,
                                     alg.num_steps_between_copying_online_weights_to_target.num_steps,
                                     alg.rate_for_copying_weights_to_target, alg.discount])
    out["par_copy_unit"] = np.array(type(alg.num_steps_between_copying_online_weights_to_target).__name__)
    out["par_memory"] = np.array(type(ap.memory).__name__)
    out["par_max_size"] = np.array([ap.memory.max_size[0].value, ap.memory.max_size[1]], dtype=np.int64)
    out["par_schemes"] = np.array([net.input_embedders_parameters['observation'].scheme.value,
                                   net.middleware_parameters.scheme.value])
    ou = OUProcessParameters()
    out["par_ou"] = np.array([ou.mu, ou.theta, ou.sigma, ou.dt], dtype=np.float64)
    out["par_head_activation"] = np.array(NAFHeadParameters().activation_function)


def main():
    from oracle import ref_loader
    ref_loader.load()
    rng = np.random.RandomState(777)
    out = {}
    golden_targets(out, rng)
    golden_ou(out, rng)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "naf.npz"), **out)
    print("naf", len(out), "arrays")


if __name__ == "__main__":
    main()
