"""N-step Q-learning without a GPU: the oracle (oracle/nstep_q.py) against the reference fixture (tests/golden/nstep_q.npz,
written by oracle/make_golden_nstep_q.py from the unmodified agent), the defaults and presets, a hand-worked segment,
and the agent's refusals."""
import os

import numpy as np
import pytest

from oracle import nstep_q as oq

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nstep_q.npz")))


def _case(c):
    return (G["c%d_q_online" % c], G["c%d_actions" % c], G["c%d_rewards" % c], G["c%d_game_overs" % c],
            float(G["c%d_discount" % c]), G["c%d_q_next" % c])


@pytest.mark.parametrize("c", range(int(G["n_cases"])))
@pytest.mark.parametrize("horizon", ["N-Step", "1-Step", "none"])
def test_oracle_targets_equal_the_reference_bit_for_bit(c, horizon):
    q, a, r, d, disc, qn = _case(c)
    got, _ = oq.segment_targets(q, a, r, d, disc, horizon, qn)
    want = G["c%d_%s_targets" % (c, horizon.lower().replace("-", ""))]
    assert got.dtype == np.float32
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))


def test_fp32_first_step_is_what_the_fixture_pins():
    """the all-fp64 recurrence differs from the reference on some bootstrapped segment of the fixture"""
    differs = False
    for c in range(int(G["n_cases"])):
        q, a, r, d, disc, qn = _case(c)
        if d[-1]:
            continue
        want = G["c%d_nstep_targets" % c]
        R = np.float64(np.max(qn[-1]))
        t = q.copy()
        for i in reversed(range(len(a))):
            R = np.float64(r[i]) + np.float64(disc) * R
            t[i, a[i]] = R
        differs |= not np.array_equal(t.view(np.uint32), want.view(np.uint32))
    assert differs


def test_hand_worked_segment():
    q = np.zeros((3, 2), dtype=np.float32)
    qn = np.array([[9, 9], [9, 9], [1.5, 2.5]], dtype=np.float32)
    t, boot = oq.segment_targets(q, np.array([0, 1, 0]), np.array([1.0, 0.0, -1.0]), np.zeros(3, bool), 0.5, "N-Step",
                                 qn)
    assert boot == np.float32(2.5)
    # R = -1 + 0.5 * 2.5 = 0.25; R = 0 + 0.5 * 0.25 = 0.125; R = 1 + 0.0625
    np.testing.assert_array_equal(t, np.array([[1.0625, 0], [0, 0.125], [0.25, 0]], dtype=np.float32))
    t, _ = oq.segment_targets(q, np.array([0, 1, 0]), np.array([1.0, 0.0, -1.0]), np.array([0, 0, 1], bool), 0.5,
                              "N-Step", qn)
    # terminal: R = -1; R = 0 + 0.5 * -1 = -0.5; R = 1 + 0.5 * -0.5 = 0.75
    np.testing.assert_array_equal(t, np.array([[0.75, 0], [0, -0.5], [-1, 0]], dtype=np.float32))
    t, boot = oq.segment_targets(q, np.array([0, 1, 0]), np.array([1.0, 0.0, -1.0]), np.array([0, 0, 1], bool), 0.5,
                                 "1-Step", qn)
    np.testing.assert_array_equal(boot, [9, 9, 2.5])
    np.testing.assert_array_equal(t, np.array([[5.5, 0], [0, 4.5], [-1, 0]], dtype=np.float32))


@pytest.mark.parametrize("t_max", [5, 3])
@pytest.mark.parametrize("tag,method,steps", [("env7", "EnvironmentSteps", 7), ("train3", "TrainingSteps", 3)])
def test_schedule_equals_the_reference(t_max, tag, method, steps):
    segs, copies, it = oq.schedule(G["sch_episodes"].tolist(), t_max, method, steps)
    key = "sch_t%d_%s" % (t_max, tag)
    assert [list(s) for s in segs] == G[key + "_segments"].tolist()
    assert copies == G[key + "_copies"].tolist()
    assert it == int(G[key + "_training_iteration"])


def test_lockstep_schedule_with_one_stream_is_the_reference_schedule():
    eps = G["sch_episodes"].tolist()
    done = np.zeros((sum(eps), 1), dtype=bool)
    done[np.cumsum(eps) - 1, 0] = True
    segs, _, _ = oq.schedule(eps, 5, "EnvironmentSteps", 7)
    got = [(t + 1, closed[0][1]) for t, closed in oq.lockstep_schedule(done, 5) if closed]
    assert got == [(s[2], s[1] - s[0]) for s in segs]


def test_defaults_and_presets_equal_the_reference():
    from coach_b200.agents.n_step_q_agent import NStepQAgentParameters
    ap = NStepQAgentParameters()
    alg, net = ap.algorithm, ap.network_wrappers["main"]
    assert [alg.num_steps_between_gradient_updates, alg.apply_gradients_every_x_episodes,
            alg.num_steps_between_copying_online_weights_to_target.num_steps, alg.discount,
            alg.rate_for_copying_weights_to_target] == G["par_algorithm"].tolist()
    assert type(alg.num_steps_between_copying_online_weights_to_target).__name__ == str(G["par_copy_method"])
    assert alg.targets_horizon == str(G["par_horizon"])
    assert [net.learning_rate, net.adam_optimizer_beta1, net.adam_optimizer_beta2, net.optimizer_epsilon,
            float(net.replace_mse_with_huber_loss), float(net.create_target_network), float(net.async_training),
            float(net.shared_optimizer)] == G["par_network"].tolist()
    sch = ap.exploration.epsilon_schedule
    assert [sch.initial_value, sch.final_value, sch.decay_steps, ap.exploration.evaluation_epsilon] == \
        G["par_epsilon"].tolist()
    from coach_b200.presets import Atari_NStepQ, CartPole_NStepQ
    for tag, mod in (("cartpole", CartPole_NStepQ), ("atari", Atari_NStepQ)):
        p = mod.agent_params
        n, a = p.network_wrappers["main"], p.algorithm
        assert [n.learning_rate, a.discount, a.num_steps_between_copying_online_weights_to_target.num_steps,
                a.num_steps_between_gradient_updates] == G["pre_%s" % tag].tolist()
        emb = n.input_embedders_parameters["observation"].scheme
        assert ([[c.num_filters, c.kernel_size, c.strides] for c in emb] if isinstance(emb, list) else []) == \
            G["pre_%s_embedder" % tag].tolist()
        mid = n.middleware_parameters.scheme
        assert ([d.units for d in mid] if isinstance(mid, list) else []) == G["pre_%s_middleware" % tag].tolist()
    rf = CartPole_NStepQ.agent_params.input_filter._reward_filters
    assert [f.rescale_factor for f in rf.values()] == G["pre_cartpole_reward_rescale"].tolist()
    assert CartPole_NStepQ.num_envs == int(G["pre_cartpole_workers"])


def test_default_network_scheme_is_the_medium_network():
    from coach_b200.base_parameters import Conv2d, Dense, middleware_units, scheme_layers
    from coach_b200.architectures.q_network import QNetworkDef
    for obs in ((4,), (84, 84, 4)):
        a = QNetworkDef("cpu", obs, 6)
        spec = [Conv2d(32, 8, 4), Conv2d(64, 4, 2), Conv2d(64, 3, 1)] if len(obs) == 3 else [Dense(256)]
        b = QNetworkDef("cpu", obs, 6, embedder_scheme=spec)
        assert list(a.store.entries.items()) == list(b.store.entries.items())
    assert scheme_layers("Medium") is None and middleware_units([Dense(256)]) == (256,)
    atari = QNetworkDef("cpu", (84, 84, 4), 6, middleware_units=(256,),
                        embedder_scheme=[Conv2d(16, 8, 4), Conv2d(32, 4, 2)])
    shapes = [s for _, s in atari.store.entries.values()]
    assert shapes[:6] == [(8, 8, 4, 16), (16,), (4, 4, 16, 32), (32,), (2592, 256), (256,)]
    with pytest.raises(ValueError):
        scheme_layers("Deep")


@pytest.mark.parametrize("field,value", [("apply_gradients_every_x_episodes", 2), ("targets_horizon", "3-Step")])
def test_refusals(field, value):
    from coach_b200.agents.n_step_q_agent import NStepQAgent, NStepQAgentParameters
    ap = NStepQAgentParameters()
    setattr(ap.algorithm, field, value)
    with pytest.raises(ValueError):
        NStepQAgent(ap, observation_shape=(4,), num_actions=2, device="cpu")


def test_dueling_head_is_refused():
    from coach_b200.agents.n_step_q_agent import NStepQAgent, NStepQAgentParameters
    ap = NStepQAgentParameters()
    ap.network_wrappers["main"].heads_parameters = ["DuelingQHead"]
    with pytest.raises(ValueError):
        NStepQAgent(ap, observation_shape=(4,), num_actions=2, device="cpu")
