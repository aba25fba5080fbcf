"""Actor-Critic (A3C) without a GPU: the oracle (oracle/a3c.py) against the reference fixture (tests/golden/a3c.npz,
written by oracle/make_golden_a3c.py from the unmodified agent), a hand-worked GAE segment, the categorical sampler, the
lock-step schedule, the defaults and presets, the network layout and the agent's refusals."""
import os

import numpy as np
import pytest

from oracle import a3c as oa

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "a3c.npz")))
MODES = ("A_VALUE", "GAE", "GAE_VALUE")


def _case(c):
    return (G["c%d_values" % c], G["c%d_boot" % c], G["c%d_rewards" % c], G["c%d_game_overs" % c],
            float(G["c%d_discount" % c]), float(G["c%d_lambda" % c]))


@pytest.mark.parametrize("c", range(int(G["n_cases"])))
@pytest.mark.parametrize("mode", MODES)
def test_oracle_targets_and_advantages_equal_the_reference_bit_for_bit(c, mode):
    v, b, r, d, disc, lam = _case(c)
    t, a = oa.segment_targets(v, b, r, d, disc, mode, lam)
    for got, key in ((t, "targets"), (a, "advantages")):
        want = G["c%d_%s_%s" % (c, mode.lower(), key)]
        assert got.dtype == np.float64
        np.testing.assert_array_equal(got.view(np.uint64), want.view(np.uint64), err_msg=key)


def test_fp32_value_products_are_what_the_fixture_pins():
    """fp64 discount * value products differ from the reference on some bootstrapped A_VALUE and some GAE segment"""
    differs = {"A_VALUE": False, "GAE": False}
    for c in range(int(G["n_cases"])):
        v, b, r, d, disc, lam = _case(c)
        if d[-1]:
            continue
        R = np.float64(b)
        t = np.zeros(len(r))
        for i in reversed(range(len(r))):
            R = np.float64(r[i]) + disc * R
            t[i] = R
        differs["A_VALUE"] |= not np.array_equal(t, G["c%d_a_value_targets" % c])
        vals = np.append(v.astype(np.float64), np.float64(b))
        delta = r + disc * vals[1:] - vals[:-1]
        differs["GAE"] |= not np.array_equal(delta[-1:] + 0.0, G["c%d_gae_advantages" % c][-1:])
    assert differs["A_VALUE"] and differs["GAE"]


def test_hand_worked_gae_segment():
    v = np.array([1.0, 2.0, 0.5], np.float32)
    r = np.array([1.0, 0.0, -1.0])
    # discount 0.5, lambda 0.5: deltas = r + 0.5 V_{i+1} - V_i with V_3 = 4 (bootstrapped)
    #   d2 = -1 + 2 - 0.5 = 0.5; d1 = 0 + 0.25 - 2 = -1.75; d0 = 1 + 1 - 1 = 1
    #   A2 = 0.5; A1 = -1.75 + 0.25 * 0.5 = -1.625; A0 = 1 + 0.25 * -1.625 = 0.59375
    #   returns of [1, 0, -1, 4]: R2 = -1 + 2 = 1; R1 = 0.5; R0 = 1.25
    t, a = oa.segment_targets(v, np.float32(4.0), r, np.zeros(3, bool), 0.5, "GAE", 0.5)
    np.testing.assert_array_equal(a, [0.59375, -1.625, 0.5])
    np.testing.assert_array_equal(t, [1.25, 0.5, 1.0])
    t, _ = oa.segment_targets(v, np.float32(4.0), r, np.zeros(3, bool), 0.5, "GAE_VALUE", 0.5)
    np.testing.assert_array_equal(t, [1.59375, 0.375, 1.0])
    # terminal: V_3 = 0; d2 = -1.5, A2 = -1.5; d1 = -1.75, A1 = -2.125; d0 = 1, A0 = 1 - 0.53125 = 0.46875
    t, a = oa.segment_targets(v, np.float32(4.0), r, np.array([0, 0, 1], bool), 0.5, "GAE", 0.5)
    np.testing.assert_array_equal(a, [0.46875, -2.125, -1.5])
    np.testing.assert_array_equal(t, [0.75, -0.5, -1.0])
    t, a = oa.segment_targets(v, np.float32(4.0), r, np.zeros(3, bool), 0.5, "A_VALUE")
    np.testing.assert_array_equal(t, [1.25, 0.5, 1.0])
    np.testing.assert_array_equal(a, [0.25, -1.5, 0.5])


@pytest.mark.parametrize("k", range(int(G["n_cat"])))
def test_categorical_sampler_equals_the_reference(k):
    p = G["cat%d_p" % k]
    want = G["cat%d_train" % k]
    np.random.seed(int(G["cat%d_seed" % k]))
    u = np.random.random_sample(len(want))                 # what len(want) successive np.random.choice calls draw
    assert [oa.categorical_choice(p, x) for x in u] == want.tolist()
    assert int(np.argmax(p)) == int(G["cat%d_eval" % k])


def test_lockstep_schedule_with_one_stream_is_the_reference_schedule():
    """the cut rule of policy_optimization_agent.py:85-135, which A3C shares with N-step Q: with E = 1 the lock-step
    schedule is the reference's (no target network: only the cuts)"""
    from oracle import nstep_q as oq
    eps = [1, 3, 5, 6, 10, 11, 23]
    for t_max in (5, 20):
        done = np.zeros((sum(eps), 1), dtype=bool)
        done[np.cumsum(eps) - 1, 0] = True
        segs, _, _ = oq.schedule(eps, t_max, "EnvironmentSteps", 10 ** 9)
        got = [(t + 1, closed[0][1]) for t, closed in oq.lockstep_schedule(done, t_max) if closed]
        assert got == [(s[2], s[1] - s[0]) for s in segs]


def test_defaults_and_presets_equal_the_reference():
    from coach_b200.agents.actor_critic_agent import ActorCriticAgentParameters
    ap = ActorCriticAgentParameters()
    alg, net = ap.algorithm, ap.network_wrappers["main"]
    assert [alg.num_steps_between_gradient_updates, alg.apply_gradients_every_x_episodes, alg.beta_entropy,
            alg.gae_lambda, float(alg.estimate_state_value_using_gae), alg.discount] == G["par_algorithm"].tolist()
    assert alg.policy_gradient_rescaler.name == str(G["par_rescaler"])
    assert [net.learning_rate, net.adam_optimizer_beta1, net.adam_optimizer_beta2, net.optimizer_epsilon,
            float(net.replace_mse_with_huber_loss), float(net.create_target_network), float(net.async_training),
            net.clip_gradients] + net.head_loss_weights == G["par_network"].tolist()
    assert [h + "Parameters" for h in net.heads_parameters] == G["par_heads"].tolist()
    from coach_b200.presets import Atari_A3C, CartPole_A3C
    for tag, mod in (("cartpole", CartPole_A3C), ("atari", Atari_A3C)):
        p = mod.agent_params
        n, a = p.network_wrappers["main"], p.algorithm
        assert [n.learning_rate, a.discount, a.num_steps_between_gradient_updates, a.apply_gradients_every_x_episodes,
                a.beta_entropy, a.gae_lambda] == G["pre_%s" % tag].tolist()
        assert a.policy_gradient_rescaler.name == str(G["pre_%s_rescaler" % tag])
    rf = CartPole_A3C.agent_params.input_filter._reward_filters
    assert [f.rescale_factor for f in rf.values()] == G["pre_cartpole_reward_rescale"].tolist()
    assert CartPole_A3C.num_envs == int(G["pre_cartpole_workers"])


def test_actor_critic_network_layout():
    import torch
    from coach_b200.architectures.q_network import QNetworkDef
    for obs, K in (((4,), 512), ((84, 84, 4), 512)):
        a, b = QNetworkDef("cpu", obs, 6), QNetworkDef("cpu", obs, 6, value_head=True)
        ea, eb = list(a.store.entries.items()), list(b.store.entries.items())
        assert [n for n, _ in ea[:-3]] == [n for n, _ in eb[:-4]] and [s for _, (_, s) in ea[:-3]] == \
            [s for _, (_, s) in eb[:-4]]
        assert [s for _, (_, s) in eb[-4:]] == [(K, 7), (7,), (), ()]
        assert [n.split("/")[-1] for n, _ in eb[-2:]] == ["gradients_from_head_0-0_rescalers",
                                                          "gradients_from_head_1-0_rescalers"]
        b.store.init_glorot(torch.Generator().manual_seed(0))
        w = b.store.view(b.store.theta, b.trunk.names[-1][0]).numpy()
        assert abs(float((w[:, 0].astype(np.float64) ** 2).sum()) - 1.0) < 1e-5      # normalized_columns(1.0)
        assert np.abs(w[:, 1:]).max() <= np.sqrt(6.0 / (K + 6)) and np.abs(w[:, 1:]).max() > 0.9 * np.sqrt(6.0 / (K + 6))
        assert not b.store.view(b.store.theta, b.trunk.names[-1][1]).numpy().any()
        assert [float(b.store.view(b.store.theta, n)[0]) for n, _ in eb[-2:]] == [1.0, 1.0]
    # the default network is unchanged
    a = QNetworkDef("cpu", (4,), 2)
    assert [n.split("/")[-1] for n in a.store.entries][-3:] == ["kernel", "bias", "gradients_from_head_0-0_rescalers"]


@pytest.mark.parametrize("field,value", [("apply_gradients_every_x_episodes", 5), ("policy_gradient_rescaler", "TD")])
def test_refusals(field, value):
    from coach_b200.agents.actor_critic_agent import (ActorCriticAgent, ActorCriticAgentParameters,
                                                      PolicyGradientRescaler)
    ap = ActorCriticAgentParameters()
    ap.algorithm.apply_gradients_every_x_episodes = 1
    setattr(ap.algorithm, field, PolicyGradientRescaler.TD_RESIDUAL if value == "TD" else value)
    with pytest.raises(ValueError) as e:
        ActorCriticAgent(ap, observation_shape=(4,), num_actions=2, device="cpu")
    if field == "apply_gradients_every_x_episodes":
        assert "default is 5" in str(e.value) and "set 1" in str(e.value)


def test_continuous_actions_and_many_ranks_are_refused(monkeypatch):
    from coach_b200 import parallel
    from coach_b200.presets.CartPole_A3C import agent_params
    from coach_b200.agents.actor_critic_agent import ActorCriticAgent
    with pytest.raises(ValueError):
        ActorCriticAgent(agent_params, observation_shape=(17,), action_dim=6, device="cpu")
    monkeypatch.setattr(parallel, "is_distributed", lambda: True)
    with pytest.raises(ValueError):
        ActorCriticAgent(agent_params, observation_shape=(4,), num_actions=2, device="cpu")
