"""Actor-Critic (A3C) with continuous actions, without a GPU: the oracle (oracle/a3c_continuous.py) against the reference
fixture (tests/golden/a3c_continuous.npz, written by oracle/make_golden_a3c_continuous.py from the unmodified agent), the
ContinuousEntropy sampler, the network layout and its three initialisers, the defaults and the Mujoco_A3C preset, and
the agent's refusals (including a segment that overruns max_episode_steps)."""
import copy
import os

import numpy as np
import pytest
import torch

from oracle import a3c as oa, a3c_continuous as oc

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "a3c_continuous.npz")))
MODES = ("A_VALUE", "GAE", "GAE_VALUE")


@pytest.mark.parametrize("c", range(int(G["n_cases"])))
@pytest.mark.parametrize("mode", MODES)
def test_oracle_targets_advantages_and_fed_actions_equal_the_reference(c, mode):
    v, b, r, d = G["c%d_values" % c], G["c%d_boot" % c], G["c%d_rewards" % c], G["c%d_game_overs" % c]
    t, a = oa.segment_targets(v, b, r, d, float(G["c%d_discount" % c]), mode, float(G["c%d_lambda" % c]))
    for got, key in ((t, "targets"), (a, "advantages")):
        want = G["c%d_%s_%s" % (c, mode.lower(), key)]
        np.testing.assert_array_equal(got.view(np.uint64), want.view(np.uint64), err_msg=key)
    D = int(G["c%d_dim" % c])
    acts = G["c%d_actions" % c]
    fed = oc.fed_actions(acts[:, 0] if D == 1 else acts, D)
    want = G["c%d_fed_actions" % c].astype(np.float32)         # the float32 placeholder's rounding
    assert fed.shape == want.shape == (len(r), D)
    np.testing.assert_array_equal(fed.view(np.uint32), want.view(np.uint32))


def test_fixture_covers_whole_episodes():
    lengths = [len(G["c%d_rewards" % c]) for c in range(int(G["n_cases"]))]
    assert min(lengths) == 1 and max(lengths) == 1000
    assert {int(G["c%d_dim" % c]) for c in range(int(G["n_cases"]))} >= {1, 17}


@pytest.mark.parametrize("k", range(int(G["n_acting"])))
def test_sampler_equals_the_reference_draws(k):
    means, stds, want = G["act%d_means" % k], G["act%d_stds" % k], G["act%d_train" % k]
    E, D = means.shape
    np.random.seed(int(G["act%d_seed" % k]))
    n = np.random.standard_normal((E, D))                      # what E successive np.random.normal calls draw
    got = oc.normal_action(means, stds, n)
    np.testing.assert_array_equal(got.view(np.uint64), want.view(np.uint64))
    np.testing.assert_array_equal(G["act%d_eval" % k], means)
    # E steps of LinearSchedule(0.5, 0.1, 7) in training, none in evaluation
    from coach_b200.schedules import LinearSchedule
    s = LinearSchedule(0.5, 0.1, 7)
    for _ in range(E):
        s.step()
    assert float(s.current_value) == float(G["act%d_noise_after" % k]) == float(G["act%d_noise_after_eval" % k])


def test_tf_softplus_regions():
    x = torch.tensor([-30.0, -13.9, -1.0, 0.0, 2.0, 13.9, 30.0], dtype=torch.float64)
    y = oc.softplus_tf(x).numpy()
    t = oc.SOFTPLUS_THRESHOLD
    assert -14.0 < t < -13.9
    assert y[0] == np.exp(-30.0) and y[-1] == 30.0
    np.testing.assert_allclose(y[1:-1], np.log1p(np.exp(x.numpy()[1:-1])), rtol=1e-10)


def test_gaussian_terms_hand_worked():
    # one dimension, range 2: z_mean = 0 -> mean 0; z_std = 0 -> std = log 2 + eps; x = 1
    z = torch.tensor([[0.5, 0.0, 0.0]], dtype=torch.float64)
    v, mean, std, logp, ent = oc.gaussian_terms(z, np.array([1.0]), np.array([2.0], np.float32))
    s = np.log(2.0) + oc.EPS32
    assert float(v[0]) == 0.5 and float(mean[0, 0]) == 0.0
    np.testing.assert_allclose(float(std[0, 0]), s, rtol=1e-15)
    np.testing.assert_allclose(float(logp[0]), -0.5 / s ** 2 - np.log(s) - 0.5 * np.log(2 * np.pi), rtol=1e-14)
    np.testing.assert_allclose(float(ent[0]), 0.5 * (1 + np.log(2 * np.pi)) + np.log(s), rtol=1e-14)


@pytest.mark.parametrize("obs,D,K", [((4,), 1, 512), ((376,), 17, 512), ((11,), 3, 512)])
def test_gaussian_network_layout_and_initialisers(obs, D, K):
    from coach_b200.architectures.q_network import QNetworkDef
    net = QNetworkDef("cpu", obs, 2 * D, value_head=True, gaussian_policy=True)
    disc = QNetworkDef("cpu", obs, 2 * D, value_head=True)
    assert [(n, s) for n, (_, s) in net.store.entries.items()] == [(n, s) for n, (_, s) in disc.store.entries.items()]
    kname, bname = net.trunk.names[-1]
    assert net.store.entries[kname][1] == (K, 1 + 2 * D)
    net.store.init_glorot(torch.Generator().manual_seed(0))
    w = net.store.view(net.store.theta, kname).numpy().astype(np.float64)
    norms = np.sqrt((w ** 2).sum(0))
    assert abs(norms[0] - 1.0) < 1e-5                                        # V: normalized_columns(1.0)
    np.testing.assert_allclose(norms[1 + D:], 0.01, rtol=1e-5)              # fc_std: normalized_columns(0.01)
    limit = np.sqrt(6.0 / (K + D))                                           # fc_mean: Glorot over (K, D)
    assert np.abs(w[:, 1:1 + D]).max() <= limit and np.abs(w[:, 1:1 + D]).max() > 0.9 * limit
    assert not net.store.view(net.store.theta, bname).numpy().any()
    with pytest.raises(ValueError):
        QNetworkDef("cpu", obs, 2 * D + 1, value_head=True, gaussian_policy=True)


def test_discrete_initialisation_is_unchanged():
    """the discrete head's draws: uniform over the kernel, then randn for column 0 (the parent's single block)"""
    from coach_b200.architectures.q_network import QNetworkDef
    net = QNetworkDef("cpu", (4,), 2, value_head=True)
    net.store.init_glorot(torch.Generator().manual_seed(3))
    kname = net.trunk.names[-1][0]
    g = torch.Generator().manual_seed(3)
    want = {}
    for name, (_, shape) in net.store.entries.items():
        if name.endswith("kernel"):
            fi, fo = net.store.glorot_fans.get(name, shape)
            cpu = (torch.rand(shape, generator=g, dtype=torch.float32) * 2 - 1) * float(np.sqrt(6.0 / (fi + fo)))
            if name == kname:
                c = torch.randn((shape[0], 1), generator=g, dtype=torch.float32)
                cpu[:, :1] = c * (1.0 / torch.sqrt((c * c).sum(dim=0, keepdim=True)))
            want[name] = cpu
    for name, t in want.items():
        assert torch.equal(net.store.view(net.store.theta, name), t), name


def test_defaults_and_preset_equal_the_reference():
    from coach_b200.agents.actor_critic_agent import ActorCriticAgentParameters, CategoricalParameters
    from coach_b200.exploration_policies.additive_noise import ContinuousEntropyParameters
    ap = ActorCriticAgentParameters()
    assert sorted("%s:%s" % (k, type(v).__name__) for k, v in ap.exploration.items()) == G["par_exploration"].tolist()
    assert isinstance(ap.exploration["DiscreteActionSpace"], CategoricalParameters)
    box = ap.exploration["BoxActionSpace"]
    assert isinstance(box, ContinuousEntropyParameters) and box.path == str(G["par_box_path"])
    s = box.noise_schedule
    assert [s.initial_value, s.final_value, s.decay_steps, box.evaluation_noise,
            float(box.noise_as_percentage_from_action_space)] == G["par_box_noise"].tolist()
    from coach_b200.presets import Mujoco_A3C as m
    n, a = m.agent_params.network_wrappers["main"], m.agent_params.algorithm
    assert [n.learning_rate, a.discount, a.num_steps_between_gradient_updates, a.apply_gradients_every_x_episodes,
            a.beta_entropy, a.gae_lambda] == G["pre_mujoco"].tolist()
    assert a.policy_gradient_rescaler.name == str(G["pre_mujoco_rescaler"])
    rf = m.agent_params.input_filter._reward_filters
    assert [f.rescale_factor for f in rf.values()] == G["pre_mujoco_reward_rescale"].tolist()
    of = m.agent_params.input_filter._observation_filters
    assert [type(f).__name__ for flt in of.values() for f in flt.values()] == \
        G["pre_mujoco_observation_filters"].tolist()
    assert m.num_envs == int(G["pre_mujoco_workers"])
    assert str(G["pre_mujoco_reward_test_level"]) == "inverted_pendulum"
    assert (m.observation_shape, m.action_dim, m.max_episode_steps) == ((4,), 1, 1000)
    assert m.action_low.tolist() == [-3.0] and m.action_high.tolist() == [3.0]


def _params():
    from coach_b200.presets.Mujoco_A3C import agent_params
    return copy.deepcopy(agent_params)


def _agent(ap=None, **kw):
    from coach_b200.agents.actor_critic_agent import ActorCriticAgent
    args = dict(observation_shape=(4,), action_dim=1, action_low=[-3.0], action_high=[3.0], device="cpu")
    args.update(kw)
    return ActorCriticAgent(ap if ap is not None else _params(), **args)


@pytest.mark.parametrize("case", ["no_bounds", "low_only", "infinite", "dim18", "features", "additive_noise"])
def test_refusals(case):
    from coach_b200.base_parameters import MiddlewareParameters
    from coach_b200.exploration_policies.additive_noise import AdditiveNoiseParameters
    ap, kw = _params(), {}
    if case == "no_bounds":
        kw = dict(action_low=None, action_high=None)
    elif case == "low_only":
        kw = dict(action_high=None)
    elif case == "infinite":
        kw = dict(action_high=[np.inf])
    elif case == "dim18":
        kw = dict(action_dim=18, action_low=-np.ones(18), action_high=np.ones(18))
    elif case == "features":
        ap.network_wrappers["main"].middleware_parameters = MiddlewareParameters("Shallow")
    else:
        ap.exploration["BoxActionSpace"] = AdditiveNoiseParameters()
    with pytest.raises(ValueError):
        _agent(ap, **kw)


def test_many_ranks_are_refused(monkeypatch):
    from coach_b200 import parallel
    monkeypatch.setattr(parallel, "is_distributed", lambda: True)
    with pytest.raises(ValueError):
        _agent()


def test_a_segment_overrunning_max_episode_steps_is_refused_before_a_row_is_overwritten(monkeypatch):
    from coach_b200 import _lib
    from coach_b200.memories.lockstep_segments import LockstepSegments

    class Lib(object):                                         # the rollout ring's scatter, counted on the host
        calls = 0

        def cb200_scatter_ring(self, *a):
            Lib.calls += 1
            return 0

    class Event(object):
        def record(self):
            pass

        def synchronize(self):
            pass
    monkeypatch.setattr(_lib, "current_stream", lambda: None)
    monkeypatch.setattr(torch.cuda, "Event", Event)
    seg = LockstepSegments(Lib(), "cpu", (3,), 2, 10 ** 7, action_dim=2, depth=4)
    obs = np.zeros((2, 3), np.float32)
    step = lambda done: seg.observe(obs, np.zeros((2, 2)), np.zeros(2), obs, np.array(done))   # noqa: E731
    for _ in range(3):
        step([False, False])
    step([True, False])                                       # stream 0 closes at 4 rows
    assert seg.close()[0].tolist() == [0]
    with pytest.raises(ValueError, match=r"stream\(s\) \[1\]"):
        step([False, False])                                  # stream 1 holds 4 open rows: the next would overwrite
    assert Lib.calls == 4 and seg.t == 4
    assert seg.rollout["state"].shape[0] == 4 * 2 and seg.max_rows == 32
    # depth defaults to t_max: the other agents' rings are unchanged
    assert LockstepSegments(Lib(), "cpu", (3,), 2, 5).rollout["state"].shape[0] == 10


def test_bucket_rows_is_shared():
    from coach_b200.agents import policy_gradients_agent as pg
    from coach_b200.memories import lockstep_segments as ls
    assert pg.bucket_rows is ls.bucket_rows
    assert [ls.bucket_rows(n) for n in (1, 256, 257, 1000, 8000)] == [32, 256, 320, 1024, 8192]
