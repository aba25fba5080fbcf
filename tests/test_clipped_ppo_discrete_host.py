"""Discrete ClippedPPO without a GPU: the oracle (oracle/clipped_ppo_discrete.py) against the reference fixture
(tests/golden/clipped_ppo_discrete.npz, written by oracle/make_golden_clipped_ppo_discrete.py from the unmodified agent)
-- Categorical acting draws, the clipping schedule's trajectory, what each minibatch feeds -- plus the defaults, the
CartPole_ClippedPPO preset and the agent's refusals."""
import importlib
import os
import random

import numpy as np
import pytest

from oracle import clipped_ppo_discrete as oc

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clipped_ppo_discrete.npz")))


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({8: np.uint64, 4: np.uint32}[a.dtype.itemsize])


@pytest.mark.parametrize("k", range(int(G["n_acting"])))
def test_acting_draws_and_schedule_equal_the_reference(k):
    from coach_b200.schedules import LinearSchedule
    g = lambda n: G["act%d_%s" % (k, n)]      # noqa: E731
    probs = g("probs")
    E = probs.shape[0]
    np.random.seed(int(g("seed")))
    u = np.random.random_sample(E)                # what E successive np.random.choice calls draw
    np.testing.assert_array_equal(oc.act(probs, u), g("train"))
    np.testing.assert_array_equal(oc.act(probs), g("eval"))
    # one step per choose_action, in training and in evaluation
    sched = LinearSchedule(*[float(x) for x in g("schedule")[:2]], int(g("schedule")[2]))
    np.testing.assert_array_equal(_bits(oc.schedule_values(sched, 2 * E)), _bits(g("clipping")))


def test_acting_fixture_covers_schedule_ends_and_wide_action_sets():
    ks = range(int(G["n_acting"]))
    assert max(G["act%d_probs" % k].shape[1] for k in ks) == 18
    assert any(G["act%d_clipping" % k][-1] == G["act%d_schedule" % k][1] for k in ks)     # a schedule reaching its end
    assert any(not np.array_equal(G["act%d_train" % k], G["act%d_eval" % k]) for k in ks)


@pytest.mark.parametrize("c", range(int(G["n_train"])))
def test_minibatch_feeds_equal_the_reference(c):
    g = lambda n: G["train%d_%s" % (c, n)]      # noqa: E731
    N, A, B, epochs = (int(x) for x in g("shape"))
    from oracle.make_golden_clipped_ppo_discrete import TRAIN
    random.seed(TRAIN[c][5])
    rows = oc.shuffled_rows(N, B, epochs)
    np.testing.assert_array_equal(rows, g("rows"))
    assert list(g("keys")) == ["observation", "output_1_0", "output_1_1", "output_1_2"]
    assert (g("fed_actions_ndim") == 1).all()                   # discrete actions are fed 1-D, not [B, 1]
    for i, r in enumerate(rows):
        feeds = oc.minibatch_feeds(r, g("actions"), g("probs"), float(g("rescaler")))
        assert list(feeds) == ["output_1_0", "output_1_1", "output_1_2"]
        np.testing.assert_array_equal(feeds["output_1_0"], g("fed_actions")[i])
        np.testing.assert_array_equal(_bits(feeds["output_1_1"]), _bits(g("fed_old")[i]))
        assert feeds["output_1_2"] == g("fed_rescaler")[i]


def test_clip_bounds_are_the_fp32_product():
    lo, hi = oc.clip_bounds(0.2, 0.3)
    e = np.float32(np.float32(0.2) * np.float32(0.3))
    assert lo == float(np.float32(1) - e) and hi == float(np.float32(1) + e)
    assert lo != 1 - 0.2 * 0.3                                   # the fp64 product rounds differently here


def test_exploration_defaults_equal_the_reference():
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgentParameters
    ap = ClippedPPOAgentParameters()
    got = sorted("%s:%s" % (k, type(v).__name__) for k, v in ap.exploration.items())
    assert got == list(G["par_exploration"])


def test_preset_equals_the_reference():
    mod = importlib.import_module("coach_b200.presets.CartPole_ClippedPPO")
    ap = mod.agent_params
    net, alg = ap.network_wrappers['main'], ap.algorithm
    np.testing.assert_array_equal([net.learning_rate, net.batch_size, net.optimizer_epsilon,
                                   net.adam_optimizer_beta2], G["pre_cartpole_network"])
    assert [net.hidden_units, net.hidden_units] == list(G["pre_cartpole_widths"])
    assert list(G["pre_cartpole_activations"]) == ["tanh", "tanh"]        # the agent's networks are tanh throughout
    np.testing.assert_array_equal([alg.clip_likelihood_ratio_using_epsilon, alg.beta_entropy, alg.gae_lambda,
                                   alg.discount, alg.optimization_epochs, float(alg.estimate_state_value_using_gae),
                                   alg.num_steps_between_copying_online_weights_to_target.num_steps],
                                  G["pre_cartpole_algorithm"])
    sched = alg.clipping_decay_schedule
    assert type(sched).__name__ == str(G["pre_cartpole_schedule"][0])
    np.testing.assert_array_equal([sched.initial_value, sched.final_value, sched.decay_steps],
                                  G["pre_cartpole_schedule_values"])
    filters = [type(f).__name__ for flt in ap.pre_network_filter._observation_filters.values() for f in flt.values()]
    assert filters == list(G["pre_cartpole_observation_filters"])
    assert (mod.observation_dim, mod.num_actions) == (4, 2)


def test_preset_resolves_to_the_device_classes():
    from coach_b200.utils import short_dynamic_import
    ap = importlib.import_module("coach_b200.presets.CartPole_ClippedPPO").agent_params
    cls = short_dynamic_import(ap.path)
    assert cls.__module__ == "coach_b200.agents.clipped_ppo_agent" and cls.__name__ == "ClippedPPOAgent"
    assert short_dynamic_import(ap.memory.path).__module__.startswith("coach_b200.memories")


def _refuse(match, **kw):
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgent, ClippedPPOAgentParameters
    with pytest.raises(ValueError, match=match):
        ClippedPPOAgent(ClippedPPOAgentParameters(), observation_dim=4, **kw)


def test_refusals():
    _refuse("exactly one")
    _refuse("exactly one", num_actions=2, action_dim=2)
    _refuse("1 .. 18 actions", num_actions=33)
    _refuse("1 .. 18 actions", num_actions=19)
    _refuse("1 .. 18 actions", num_actions=0)


def test_refuses_discrete_actions_on_several_ranks(monkeypatch):
    from coach_b200 import parallel
    monkeypatch.setattr(parallel, "world", lambda: (0, 2))
    _refuse("one rank", num_actions=2)


@pytest.mark.parametrize("low, high", [(None, None), (-1.0, None), (-np.inf, 1.0), (np.array([-1.0, -1.0]),
                                                                                     np.array([1.0, np.nan]))])
def test_continuous_acting_needs_finite_bounds(low, high):
    """refused at the call, before any network runs (the agent itself is never built here)"""
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgent
    ag = ClippedPPOAgent.__new__(ClippedPPOAgent)
    ag.discrete = False
    ag.action_low = None if low is None or high is None else np.broadcast_to(np.asarray(low, np.float64), (2,))
    ag.action_high = None if low is None or high is None else np.broadcast_to(np.asarray(high, np.float64), (2,))
    with pytest.raises(ValueError, match="bounded"):
        ag.choose_actions(np.zeros((1, 4), np.float32))
