"""tests/head_ref.py pinned to what is already pinned to the reference agents: the oracle restatements
(oracle/nets.dqn_targets, oracle/pal_mmc, oracle/bootstrapped, oracle/c51) and the fixtures written from the unmodified
reference (tests/golden/agent_prologues.npz, pal_mmc.npz, bootstrapped.npz), target bits where the fixtures have them.
So the reference the fused-head kernel tests compare against is not a second, unchecked opinion."""
import os

import numpy as np
import pytest

import head_ref as hr

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _npz(name):
    return dict(np.load(os.path.join(GOLDEN, name)))


def _bits(x):
    x = np.asarray(x)
    return x.view(np.uint32 if x.dtype == np.float32 else np.uint64)


@pytest.mark.parametrize("tag", ["dqn", "ddqn"])
def test_dqn_rule_matches_the_oracle_and_the_fixture(tag):
    from oracle import nets as on
    fx = _npz("agent_prologues.npz")
    g = lambda k: fx[tag + "_" + k]                                                             # noqa: E731
    q_sel = g("q_select") if tag == "ddqn" else None
    targets, td, _ = hr.rule_targets(hr.TARGET_DQN, g("q_online"), g("q_next"), q_sel, g("actions"), g("rewards"),
                                     g("game_overs"), 0.99)
    want_t, want_td = on.dqn_targets(g("q_next"), g("q_next") if q_sel is None else q_sel, g("q_online"), g("actions"),
                                     g("rewards"), g("game_overs").astype(bool), 0.99)
    np.testing.assert_array_equal(_bits(targets), _bits(want_t))
    np.testing.assert_array_equal(_bits(td), _bits(want_td))
    np.testing.assert_array_equal(_bits(targets), _bits(g("targets")))
    np.testing.assert_array_equal(_bits(td), _bits(g("td_errors")))


@pytest.mark.parametrize("tag", ["", "_b"])
@pytest.mark.parametrize("rule", [hr.TARGET_MMC, hr.TARGET_PAL, hr.TARGET_PAL_PERSISTENT])
def test_mmc_and_pal_rules_match_the_oracle_and_the_fixture(rule, tag):
    from oracle.pal_mmc import mmc_targets, pal_targets
    g = _npz("pal_mmc.npz")
    alpha, rho = (float(x) for x in g["alpha_rate" + tag])
    common = dict(actions=g["actions"], rewards=g["rewards"], game_overs=g["game_overs"], returns=g["returns"],
                  discount=float(g["discount"]))
    targets, td, _ = hr.rule_targets(rule, g["q_online"], g["q_next"], g["q_select"], q_target_s=g["q_target_s"],
                                     alpha=alpha, rho=rho, **common)
    if rule == hr.TARGET_MMC:
        want = mmc_targets(g["q_next"], g["q_select"], g["q_online"], mixing_rate=rho, **common)
    else:
        want = pal_targets(g["q_next"], g["q_select"], g["q_target_s"], g["q_online"], alpha=alpha,
                           persistent=rule == hr.TARGET_PAL_PERSISTENT, mixing_rate=rho, **common)
    name = hr.RULE_NAMES[rule]
    np.testing.assert_array_equal(_bits(targets), _bits(want))
    np.testing.assert_array_equal(_bits(targets), _bits(g["%s%s_targets" % (name, tag)]))
    rows = np.arange(len(g["actions"]))
    want_td = np.abs(want[rows, g["actions"]].astype(np.float64) - g["q_online"][rows, g["actions"]])
    np.testing.assert_array_equal(_bits(td), _bits(want_td))


def test_rho_zero_reduces_mmc_and_pal_to_the_ddqn_rule():
    g = _npz("pal_mmc.npz")
    common = dict(actions=g["actions"], rewards=g["rewards"], game_overs=g["game_overs"], returns=g["returns"],
                  discount=float(g["discount"]), q_target_s=g["q_target_s"])
    ddqn = hr.rule_targets(hr.TARGET_DQN, g["q_online"], g["q_next"], g["q_select"], g["actions"], g["rewards"],
                           g["game_overs"], float(g["discount"]))[0]
    for rule in (hr.TARGET_MMC, hr.TARGET_PAL, hr.TARGET_PAL_PERSISTENT):
        t = hr.rule_targets(rule, g["q_online"], g["q_next"], g["q_select"], alpha=0.0, rho=0.0, **common)[0]
        np.testing.assert_array_equal(_bits(t), _bits(ddqn), err_msg=hr.RULE_NAMES[rule])


def test_out_of_range_actions_keep_the_row():
    rng = np.random.RandomState(0)
    q = rng.randn(4, 3).astype(np.float32)
    act = np.array([0, 3, -1, 2])
    for rule in (hr.TARGET_DQN, hr.TARGET_MMC, hr.TARGET_PAL, hr.TARGET_PAL_PERSISTENT):
        t, td, _ = hr.rule_targets(rule, q, q, q, act, np.ones(4), np.zeros(4, np.uint8), 0.99, q_target_s=q,
                                   returns=np.ones(4), alpha=0.5, rho=0.5)
        np.testing.assert_array_equal(t[1:3], q[1:3])
        assert td[1] == 0.0 and td[2] == 0.0 and td[0] > 0.0


def test_ensemble_targets_match_the_oracle_and_the_fixture():
    from oracle.bootstrapped import bootstrapped_targets
    g = _npz("bootstrapped.npz")
    H = g["pro_q_online"].shape[0]
    flat = lambda k: np.concatenate(list(g[k]), axis=1)                                          # noqa: E731
    targets, _ = hr.ensemble_targets(flat("pro_q_online"), flat("pro_q_next"), flat("pro_q_select"), g["pro_actions"],
                                     g["pro_rewards"], g["pro_game_overs"], g["pro_masks"], float(g["pro_discount"]), H)
    want = bootstrapped_targets(list(g["pro_q_next"]), list(g["pro_q_select"]), list(g["pro_q_online"]),
                                g["pro_actions"], g["pro_rewards"], g["pro_game_overs"], g["pro_masks"],
                                float(g["pro_discount"]))
    np.testing.assert_array_equal(_bits(targets), _bits(np.concatenate(want, axis=1)))
    np.testing.assert_array_equal(_bits(targets), _bits(flat("pro_targets")))


@pytest.mark.parametrize("tag", ["c51", "rainbow"])
def test_c51_projection_matches_the_oracle_and_the_fixture(tag):
    from oracle import c51
    fx = _npz("agent_prologues.npz")
    g = lambda k: fx[tag + "_" + k]                                                             # noqa: E731
    sel = g("dist_select") if tag == "rainbow" else None
    coef = g("bootstrap") * float(g("gamma_n"))
    r = hr.c51_head(g("dist_next"), g("dist_online"), sel, g("actions"), g("rewards"), coef, g("z"), next_is_prob=1)
    want_t, want_a, want_m = c51.c51_targets(g("dist_next"), g("dist_online"), sel, g("actions"), g("rewards"),
                                             g("bootstrap"), float(g("gamma_n")), g("z"))
    np.testing.assert_array_equal(r["sel"], want_a)
    np.testing.assert_array_equal(_bits(r["m"]), _bits(want_m))
    labels = np.array(g("dist_online"), dtype=np.float32, copy=True)
    labels[np.arange(len(r["sel"])), g("actions")] = r["m"]
    np.testing.assert_array_equal(_bits(labels), _bits(g("targets")))


def test_c51_bound_check_agrees_with_the_reference_index_error():
    """on a linspace support whose top bin position rounds above N - 1, a target clamped to v_max is an IndexError in
    the reference (oracle/c51.py restates its loop) and an AssertionError in head_ref unless the drop is asked for; the
    drop changes nothing inside the row but the share that would have landed on bin N"""
    from oracle import c51
    z = np.linspace(-10.0, 10.0, 101)
    assert hr.projection_overflow(z) and not hr.projection_overflow(np.linspace(-10.0, 10.0, 51))
    B, N = 3, z.size
    p = np.full((B, 1, N), 1.0 / N, dtype=np.float32)
    rewards = np.array([0.0, 50.0, -3.0])                  # row 1 clamps to v_max
    coef = np.array([0.99, 0.99, 0.0])
    with pytest.raises(IndexError):
        c51.c51_targets(p, p, None, np.zeros(B, np.int64), rewards, coef / 0.99, 0.99, z)
    with pytest.raises(AssertionError):
        hr.c51_project(p[:, 0], rewards, coef, z)
    m = hr.c51_project(p[:, 0], rewards, coef, z, allow_drop=True)
    ok = [0, 2]
    np.testing.assert_array_equal(m[ok], hr.c51_project(p[ok, 0], rewards[ok], coef[ok], z))


def test_categorical_agent_refuses_a_support_whose_top_bin_overflows():
    from coach_b200.agents.categorical_dqn_agent import CategoricalDQNAgent, CategoricalDQNAgentParameters
    ap = CategoricalDQNAgentParameters()
    ap.algorithm.atoms = 101
    with pytest.raises(ValueError, match="IndexError"):
        CategoricalDQNAgent(ap, observation_shape=(4,), num_actions=2, seed=0)


def test_fp32_emulation_of_the_head_stays_within_the_fp64_bound():
    """the emulation itself satisfies the bound the kernel is held to, so the bound is not vacuous for it"""
    rng = np.random.RandomState(1)
    B, K, A = 33, 256, 6
    h = np.maximum(rng.randn(B, K), 0).astype(np.float32)
    w = (rng.randn(K, A) * 0.1).astype(np.float32)
    b = (rng.randn(A) * 0.1).astype(np.float32)
    q32 = hr.head_q32(h, w, b)
    q64, S = hr.head_q64(h, w, b)
    assert np.all(np.abs(q32 - q64) <= hr.gamma(hr.dot_terms(K)) * S)
    tgt = q32 + rng.randn(B, A).astype(np.float32)
    dq, row = hr.loss_grad32(q32, tgt, None, True, B)
    np.testing.assert_allclose(dq, hr.dq64(q32, tgt, None, True, B), rtol=4 * hr.U32, atol=0)
    r = hr.backward32(h, w, dq, row, None, B)
    b64 = hr.backward64(h, w, dq)
    for k, n in (("dw", B + 8), ("db", B + 8), ("dh", A)):
        v, s = b64[k]
        assert np.all(np.abs(r[k] - v) <= hr.gamma(n) * s), k
    l64, ls = hr.loss64(q32, tgt, None, True, B)
    assert abs(float(r["loss"]) - l64) <= hr.gamma(B * A + 10) * ls
