"""NAF pinned to the reference on the host: the oracle's TD targets, BatchedOUProcess, the parameter classes and the
Mujoco_NAF preset against tests/golden/naf.npz (written from the unmodified reference by oracle/make_golden_naf.py), and
the oracle's L packing against a hand-worked case."""
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "naf.npz")


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLDEN))


@pytest.mark.parametrize("key", ["a1", "a1_g09", "a6", "a6_g09"])
def test_oracle_td_targets_equal_the_reference_bit_for_bit(g, key):
    from oracle.rl_math import ac_td_targets
    p = "td_%s_" % key
    y = ac_td_targets(g[p + "rewards"], g[p + "dones"], g[p + "v"], float(g[p + "discount"]))
    np.testing.assert_array_equal(y.view(np.uint64), g[p + "targets"].view(np.uint64))
    # what the fp32 feed receives, and the head input is the batch actions unchanged
    np.testing.assert_array_equal(y.astype(np.float32).view(np.uint32),
                                  g[p + "targets"].astype(np.float32).view(np.uint32))
    np.testing.assert_array_equal(g[p + "output_0_0"], g[p + "actions"])


def test_fixture_covers_terminal_rows_and_large_rewards(g):
    d, r = g["td_a6_dones"], g["td_a6_rewards"]
    assert d.any() and (~d.astype(bool)).any()
    assert (r < 0).any() and (np.abs(r) > 1e5).any() and (r != np.round(r)).any()


@pytest.mark.parametrize("A", [1, 3, 6])
def test_batched_ou_process_reproduces_the_reference_actions(g, A):
    from coach_b200.exploration_policies.e_greedy import RunPhase
    from coach_b200.exploration_policies.ou_process import BatchedOUProcess
    mus, want = g["ou_a%d_mu" % A], g["ou_a%d_actions" % A]
    steps, E = mus.shape[0], mus.shape[1]
    resets = {}
    for s, e in g["ou_resets"]:
        resets.setdefault(int(s), []).append(int(e))
    test_steps = set(int(s) for s in g["ou_test_steps"])
    pol = BatchedOUProcess(A, E)
    np.random.seed(int(g["ou_seed_base"]) + A)
    for step in range(steps):
        for e in resets.get(step, ()):
            pol.reset(e)
        pol.change_phase(RunPhase.TEST if step in test_steps else RunPhase.TRAIN)
        got = pol.get_actions(mus[step])
        np.testing.assert_array_equal(got.view(np.uint64), want[step].view(np.uint64), err_msg="step %d" % step)
    # the TEST phase adds no noise
    for s in test_steps:
        np.testing.assert_array_equal(want[s], mus[s].astype(np.float64))


def test_parameter_classes_equal_the_reference_defaults(g):
    from coach_b200.agents.naf_agent import NAFAgentParameters
    from coach_b200.base_parameters import MiddlewareScheme
    from coach_b200.exploration_policies.ou_process import OUProcessParameters
    from coach_b200.utils import short_dynamic_import
    ap = NAFAgentParameters()
    net, alg = ap.network_wrappers["main"], ap.algorithm
    np.testing.assert_array_equal([net.learning_rate, net.adam_optimizer_beta1, net.adam_optimizer_beta2,
                                   net.optimizer_epsilon, net.batch_size, float(net.replace_mse_with_huber_loss),
                                   float(net.create_target_network)], g["par_network"])
    np.testing.assert_array_equal([alg.num_consecutive_training_steps,
                                   alg.num_steps_between_copying_online_weights_to_target.num_steps,
                                   alg.rate_for_copying_weights_to_target, alg.discount], g["par_algorithm"])
    assert type(alg.num_steps_between_copying_online_weights_to_target).__name__ == str(g["par_copy_unit"])
    assert type(ap.memory).__name__ == str(g["par_memory"])
    assert [ap.memory.max_size[0].value, ap.memory.max_size[1]] == list(g["par_max_size"])
    # embedder scheme Medium = [Dense(256)], middleware Medium = [Dense(512)]
    assert [str(s) for s in g["par_schemes"]] == ["Medium", "Medium"]
    assert tuple(net.embedder_units) == (256,) and net.middleware_parameters.scheme == MiddlewareScheme.Medium
    ou = OUProcessParameters()
    np.testing.assert_array_equal([ou.mu, ou.theta, ou.sigma, ou.dt], g["par_ou"])
    assert isinstance(ap.exploration, OUProcessParameters)
    assert str(g["par_head_activation"]) == "tanh"
    assert short_dynamic_import(ap.path).__name__ == "NAFAgent"
    assert short_dynamic_import(ap.path).__module__ == "coach_b200.agents.naf_agent"
    assert short_dynamic_import(ap.exploration.path).__name__ == "BatchedOUProcess"
    assert short_dynamic_import(ap.memory.path).__module__.startswith("coach_b200.memories")


def test_mujoco_naf_preset():
    from coach_b200.presets import Mujoco_NAF as preset
    from coach_b200.utils import short_dynamic_import
    ap = preset.agent_params
    net = ap.network_wrappers["main"]
    assert tuple(net.embedder_units) == (200,) and list(net.middleware_parameters.scheme) == [200]
    assert net.gradients_clipping_method == "ClipByValue" and net.clip_gradients == 1000
    assert short_dynamic_import(ap.path).__module__ == "coach_b200.agents.naf_agent"
    assert short_dynamic_import(ap.memory.path).__name__ == "EpisodicExperienceReplay"
    assert short_dynamic_import(ap.exploration.path).__name__ == "BatchedOUProcess"


def test_oracle_l_packing_hand_worked():
    """A = 3, l = [l0 .. l5]: column 0 = [e^l0, l1, l2], column 1 = [0, e^l3, l4], column 2 = [0, 0, e^l5]"""
    from oracle.naf import unpack_l
    lv = torch.tensor([[0.0, 2.0, 3.0, np.log(4.0), 5.0, np.log(6.0)]], dtype=torch.float64)
    L = unpack_l(lv, 3)[0].numpy()
    want = np.array([[1.0, 0.0, 0.0],
                     [2.0, 4.0, 0.0],
                     [3.0, 5.0, 6.0]])
    np.testing.assert_allclose(L, want, rtol=1e-15)
    # the oracle's advantage: d = (0, 0, 1) -> L^T d = (3, 5, 6), A = -0.5 * 70; d = (1, 0, 0) -> L^T d = (1, 0, 0)
    from oracle.naf import naf_forward
    h = torch.zeros((2, 1), dtype=torch.float64)
    params = [torch.zeros((1, 1), dtype=torch.float64), torch.zeros(1, dtype=torch.float64),       # trunk Dense(1)
              torch.zeros((1, 1), dtype=torch.float64), torch.zeros(1, dtype=torch.float64),       # V
              torch.zeros((1, 3), dtype=torch.float64), torch.zeros(3, dtype=torch.float64),       # mu_unscaled
              torch.zeros((1, 6), dtype=torch.float64), lv[0]]                                     # l_vector
    u = torch.tensor([[0.0, 0.0, 1.0], [1.0, 0.0, 0.0]], dtype=torch.float64)
    f = naf_forward(params, h, u, torch.ones(3, dtype=torch.float64), 1, 3)
    np.testing.assert_allclose(f["q"].numpy().ravel(), [-35.0, -0.5], rtol=1e-15)


def test_naf_refuses_what_it_cannot_run():
    """no GPU needed: the refusals come before any device work"""
    from coach_b200.agents.naf_agent import NAFAgent, NAFAgentParameters
    for kwargs in (dict(action_dim=33), dict(action_dim=0), dict(action_dim=3, continuous_actions=False)):
        with pytest.raises(ValueError):
            NAFAgent(NAFAgentParameters(), observation_dim=11, device="cpu", **kwargs)
    ap = NAFAgentParameters()
    ap.network_wrappers["main"].clip_gradients = 5.0
    ap.network_wrappers["main"].gradients_clipping_method = "ClipByNorm"
    with pytest.raises(NotImplementedError):
        NAFAgent(ap, observation_dim=11, action_dim=3, device="cpu")
