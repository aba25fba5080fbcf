"""PAL and Mixed Monte Carlo pinned to the reference on the host: the oracle prologues and the parameter defaults against
tests/golden/pal_mmc.npz (written from the unmodified reference by oracle/make_golden_pal_mmc.py)."""
import importlib
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pal_mmc.npz")


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLDEN))


def _common(g):
    return dict(q_next=g["q_next"], q_select=g["q_select"], q_online=g["q_online"], actions=g["actions"],
                rewards=g["rewards"], game_overs=g["game_overs"], returns=g["returns"], discount=float(g["discount"]))


@pytest.mark.parametrize("tag", ["", "_b"])
def test_oracle_reproduces_every_fixture_target(g, tag):
    from oracle.pal_mmc import mmc_targets, pal_targets
    alpha, rate = (float(x) for x in g["alpha_rate" + tag])
    want = {"mmc": mmc_targets(mixing_rate=rate, **_common(g))}
    for persistent in (False, True):
        want["pal_persistent" if persistent else "pal"] = pal_targets(
            q_target_s=g["q_target_s"], alpha=alpha, persistent=persistent, mixing_rate=rate, **_common(g))
    for name, t in want.items():
        assert t.dtype == np.float32
        np.testing.assert_array_equal(t.view(np.uint32), g["%s%s_targets" % (name, tag)].view(np.uint32), err_msg=name)


def test_fixture_covers_the_crafted_rows(g):
    qs, qn, qt, a = g["q_select"], g["q_next"], g["q_target_s"], g["actions"]
    B = len(a)
    sel = np.argmax(qs, 1)
    adv = np.max(qt, 1) - qt[np.arange(B), a]
    nadv = np.max(qn, 1) - qn[np.arange(B), sel]
    assert (adv == nadv).any() and (adv < nadv).any() and (adv > nadv).any()
    assert g["game_overs"].any() and (np.abs(g["returns"]) > 1e5).any()
    assert any((qs[i] == qs[i].max()).sum() > 1 for i in range(B))                  # argmax ties
    # the persistent rule differs from the regular one somewhere, and the mixing rate reaches every taken action
    assert not np.array_equal(g["pal_targets"], g["pal_persistent_targets"])
    rows = np.arange(B)
    assert (g["mmc_targets"][rows, a] != g["q_online"][rows, a]).all()


def test_parameter_classes_equal_the_reference_defaults(g):
    from coach_b200.agents.mmc_agent import MixedMonteCarloAgentParameters
    from coach_b200.agents.pal_agent import PALAgentParameters
    from coach_b200.utils import short_dynamic_import
    pal, mmc = PALAgentParameters(), MixedMonteCarloAgentParameters()
    alg = pal.algorithm
    np.testing.assert_array_equal([alg.pal_alpha, float(alg.persistent_advantage_learning),
                                   alg.monte_carlo_mixing_rate, alg.discount], g["par_pal"])
    np.testing.assert_array_equal([mmc.algorithm.monte_carlo_mixing_rate, mmc.algorithm.discount], g["par_mmc"])
    for tag, ap, cls in (("pal", pal, "PALAgent"), ("mmc", mmc, "MixedMonteCarloAgent")):
        assert type(ap.memory).__name__ == str(g["par_%s_memory" % tag])
        assert [ap.memory.max_size[0].value, ap.memory.max_size[1]] == list(g["par_%s_max_size" % tag])
        assert ap.algorithm.num_steps_between_copying_online_weights_to_target.num_steps == \
            g["par_%s_copy_steps" % tag]
        assert short_dynamic_import(ap.path).__name__ == cls
        assert short_dynamic_import(ap.memory.path).__module__.startswith("coach_b200.memories")


@pytest.mark.parametrize("tag,preset,shape", [("cartpole_pal", "CartPole_PAL", ((4,), 2)),
                                              ("doom_mmc", "Doom_Health_MMC", ((60, 76, 3), 4))])
def test_presets_equal_the_reference_agent_parameters(g, tag, preset, shape):
    from coach_b200.utils import short_dynamic_import
    mod = importlib.import_module("coach_b200.presets." + preset)
    ap = mod.agent_params
    assert (mod.observation_shape, mod.num_actions) == shape
    net, alg = ap.network_wrappers["main"], ap.algorithm
    got = [net.learning_rate, float(net.replace_mse_with_huber_loss), alg.discount,
           alg.num_steps_between_copying_online_weights_to_target.num_steps, alg.num_consecutive_playing_steps.num_steps,
           ap.memory.max_size[0].value, ap.memory.max_size[1], net.batch_size]
    np.testing.assert_array_equal(got, g["pre_" + tag])
    assert short_dynamic_import(ap.path).__name__ == str(g["pre_%s_path" % tag])


def test_episodic_fixture_counts_like_the_reference_length(g):
    """the fixture's reference counters: length() counts the open episode only when it is non-empty, so at most k - 1
    complete episodes stay listed while one is being filled"""
    k, c = int(g["ep_k"]), g["ep_counters"]
    assert (c[:, 2] <= k).all() and (c[:, 3] <= k).all()
    open_len = c[:, 0] - c[:, 1]
    assert (c[open_len > 0, 2] <= k - 1).all() and (c[open_len == 0, 2] == k).any()
