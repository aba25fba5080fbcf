"""Quantile Regression DQN pinned to the reference on the host: the oracle prologue (TD targets, midpoints, target
actions) and the parameter defaults against tests/golden/qr_dqn.npz (written from the unmodified reference by
oracle/make_golden_qr_dqn.py), the oracle's loss and gradient against a hand-worked case, and the refusals."""
import importlib
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qr_dqn.npz")
CASES = ["a2_n50", "a6_n200", "a18_n7", "a2_n1", "a6_n7"]


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLDEN))


def _case(g, tag):
    p = "c_%s_" % tag
    return {k: g[p + k] for k in ("next", "online", "actions", "rewards", "dones", "discount", "targets",
                                  "output_0_0", "output_0_1", "target_actions")}


@pytest.mark.parametrize("tag", CASES)
def test_oracle_prologue_equals_the_reference_bit_for_bit(g, tag):
    from oracle.qr_dqn import qr_targets
    c = _case(g, tag)
    t, ta, tau = qr_targets(c["next"], c["online"], c["actions"], c["rewards"], c["dones"], float(c["discount"]))
    np.testing.assert_array_equal(t.view(np.uint64), c["targets"].view(np.uint64))
    np.testing.assert_array_equal(t.astype(np.float32).view(np.uint32),
                                  c["targets"].astype(np.float32).view(np.uint32))
    np.testing.assert_array_equal(tau.view(np.uint64), c["output_0_1"].view(np.uint64))
    np.testing.assert_array_equal(tau.astype(np.float32).view(np.uint32),
                                  c["output_0_1"].astype(np.float32).view(np.uint32))
    np.testing.assert_array_equal(ta, c["target_actions"])
    B = len(c["actions"])
    np.testing.assert_array_equal(c["output_0_0"], np.stack([np.arange(B), c["actions"]], axis=1))


def test_fixture_covers_terminal_rows_rewards_one_atom_and_the_permutation_quirk(g):
    from oracle.qr_dqn import rank_midpoints
    d, r = g["c_a6_n200_dones"], g["c_a6_n200_rewards"]
    assert d.any() and (~d.astype(bool)).any()
    assert (r < 0).any() and (np.abs(r) > 1e5).any() and (r != np.round(r)).any()
    assert g["c_a2_n1_output_0_1"].shape[1] == 1 and (g["c_a2_n1_output_0_1"] == 0.5).all()
    # the reference's tau_hat[sigma(i)] is not the rank assignment tau_hat[sigma^-1(i)] the paper intends
    c = _case(g, "a6_n200")
    rank = rank_midpoints(c["online"], c["actions"])
    assert not np.array_equal(rank, c["output_0_1"])
    # ... and every taken row of every case is tie-free, so argsort's kind does not matter there
    for tag in CASES:
        c = _case(g, tag)
        rows = c["online"][np.arange(len(c["actions"])), c["actions"]]
        assert all(len(np.unique(x)) == x.size for x in rows)


def _values(ap):
    net, alg, ex = ap.network_wrappers["main"], ap.algorithm, ap.exploration
    return [net.learning_rate, net.optimizer_epsilon, net.adam_optimizer_beta1, net.adam_optimizer_beta2,
            net.batch_size, float(net.replace_mse_with_huber_loss), float(net.create_target_network),
            alg.atoms, alg.huber_loss_interval, alg.discount,
            alg.num_steps_between_copying_online_weights_to_target.num_steps,
            alg.num_consecutive_playing_steps.num_steps, alg.num_consecutive_training_steps,
            ap.memory.max_size[0].value, ap.memory.max_size[1],
            ex.epsilon_schedule.initial_value, ex.epsilon_schedule.final_value,
            ex.epsilon_schedule.decay_steps, ex.evaluation_epsilon]


def test_parameter_classes_equal_the_reference_defaults(g):
    from coach_b200.agents.qr_dqn_agent import QuantileRegressionDQNAgentParameters
    from coach_b200.utils import short_dynamic_import
    ap = QuantileRegressionDQNAgentParameters()
    np.testing.assert_array_equal(_values(ap), g["par_defaults"])
    assert type(ap.memory).__name__ == str(g["par_memory"])
    assert type(ap.algorithm.num_steps_between_copying_online_weights_to_target).__name__ == str(g["par_copy_unit"])
    assert short_dynamic_import(ap.path).__name__ == "QuantileRegressionDQNAgent"
    assert short_dynamic_import(ap.path).__module__ == "coach_b200.agents.qr_dqn_agent"
    assert short_dynamic_import(ap.exploration.path).__name__ == "BatchedEGreedy"
    assert short_dynamic_import(ap.memory.path).__module__.startswith("coach_b200.memories")
    assert ap.network_wrappers["main"].heads_parameters == ["QuantileRegressionQHead"]


@pytest.mark.parametrize("tag,preset,shape", [("atari", "Atari_QR_DQN", ((84, 84, 4), 6)),
                                              ("cartpole", "CartPole_QR_DQN", ((4,), 2))])
def test_presets_equal_the_reference_agent_parameters(g, tag, preset, shape):
    from coach_b200.utils import short_dynamic_import
    mod = importlib.import_module("coach_b200.presets." + preset)
    assert (mod.observation_shape, mod.num_actions) == shape
    np.testing.assert_array_equal(_values(mod.agent_params), g["pre_" + tag])
    assert short_dynamic_import(mod.agent_params.path).__name__ == str(g["pre_%s_path" % tag])


def test_oracle_loss_and_gradient_hand_worked():
    """N = 3, kappa = 1, theta = (0, 1, 2) (sorted: tau = tau_hat = (1/6, 1/2, 5/6)), T = (-1, 0.5, 3):
    per-i pair sums 41/48, 75/48, 48/48 -> L = (41/12) / 3 = 41/36;
    d L / d theta = -(1/3) (-7/12, -1/4, 1/2) = (7/36, 1/12, -1/6)"""
    from oracle.qr_dqn import qr_loss_grad, quantile_midpoints
    theta = torch.tensor([[0.0, 1.0, 2.0]], dtype=torch.float64)
    t = torch.tensor([[-1.0, 0.5, 3.0]], dtype=torch.float64)
    tau = torch.from_numpy(quantile_midpoints(3)[None, :])
    np.testing.assert_allclose(tau.numpy(), [[1 / 6, 1 / 2, 5 / 6]], rtol=1e-15)
    loss, grad = qr_loss_grad(theta, t, tau, 1.0)
    np.testing.assert_allclose(float(loss), 41.0 / 36.0, rtol=1e-14)
    np.testing.assert_allclose(grad.numpy(), [[7 / 36, 1 / 12, -1 / 6]], rtol=1e-14)
    # the gradient is the derivative of the loss away from the kinks (central differences in fp64)
    h = 1e-6
    for i in range(3):
        dp, dm = theta.clone(), theta.clone()
        dp[0, i] += h
        dm[0, i] -= h
        fd = (float(qr_loss_grad(dp, t, tau, 1.0)[0]) - float(qr_loss_grad(dm, t, tau, 1.0)[0])) / (2 * h)
        np.testing.assert_allclose(fd, float(grad[0, i]), rtol=1e-6)


def test_kappa_zero_gives_zero_loss_and_gradient():
    """huber_loss_interval = 0, the docstring's "strict quantile loss": h = 0 (a - 0) + 0.5 * 0^2 = 0 everywhere"""
    from oracle.qr_dqn import qr_loss_grad
    rng = np.random.RandomState(0)
    for dtype in (torch.float32, torch.float64):
        theta = torch.from_numpy(rng.randn(4, 9)).to(dtype)
        t = torch.from_numpy(rng.randn(4, 9) * 10).to(dtype)
        tau = torch.from_numpy(rng.rand(4, 9)).to(dtype)
        loss, grad = qr_loss_grad(theta, t, tau, 0.0)
        assert float(loss) == 0.0 and not grad.abs().max().item()


def test_refuses_a_prioritized_replay_and_a_dueling_head():
    """no GPU needed: the refusals come before any device work"""
    from coach_b200.agents.qr_dqn_agent import QuantileRegressionDQNAgent, QuantileRegressionDQNAgentParameters
    from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplayParameters
    ap = QuantileRegressionDQNAgentParameters()
    ap.memory = PrioritizedExperienceReplayParameters()
    with pytest.raises(NotImplementedError, match="prioritized"):
        QuantileRegressionDQNAgent(ap, observation_shape=(4,), num_actions=2, device="cpu")
    ap = QuantileRegressionDQNAgentParameters()
    ap.network_wrappers["main"].heads_parameters = ["DuelingQHead"]
    with pytest.raises(NotImplementedError, match="dueling"):
        QuantileRegressionDQNAgent(ap, observation_shape=(4,), num_actions=2, device="cpu")
    ap = QuantileRegressionDQNAgentParameters()
    ap.algorithm.atoms = 1025
    with pytest.raises(ValueError):
        QuantileRegressionDQNAgent(ap, observation_shape=(4,), num_actions=2, device="cpu")
