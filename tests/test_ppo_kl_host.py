"""PPO (KL penalty) without a GPU: the oracle (oracle/ppo.py) against the reference fixture (tests/golden/ppo.npz, written
by oracle/make_golden_ppo.py from the unmodified agent) -- advantages, the minibatch plan and what it feeds, the KL
coefficient rule, the AdditiveNoise draw -- plus a hand-worked one-dimensional KL-penalty gradient, the defaults, the
Mujoco_PPO preset and the agent's refusals."""
import os

import numpy as np
import pytest

from oracle import ppo as op

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ppo.npz")))


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({8: np.uint64, 4: np.uint32}[a.dtype.itemsize])


@pytest.mark.parametrize("c", range(int(G["n_adv"])))
def test_oracle_advantages_equal_the_reference(c):
    g = lambda k: G["adv%d_%s" % (c, k)]      # noqa: E731
    got = op.fill_advantages(g("rewards"), g("values"), g("game_overs").astype(bool), g("returns"),
                             float(g("discount")), float(g("lambda")), str(g("rescaler")))
    np.testing.assert_array_equal(_bits(got), _bits(g("advantages")))


def test_fixture_covers_episode_lengths_and_rescalers():
    lengths = set()
    for c in range(int(G["n_adv"])):
        ends = np.nonzero(G["adv%d_game_overs" % c])[0]
        lengths |= set(np.diff(np.concatenate([[-1], ends])).tolist())
    assert min(lengths) == 1 and max(lengths) == 1000
    assert {str(G["adv%d_rescaler" % c]) for c in range(int(G["n_adv"]))} == {"GAE", "A_VALUE"}
    assert {float(G["adv%d_lambda" % c]) for c in range(int(G["n_adv"])) if str(G["adv%d_rescaler" % c]) == "GAE"} \
        == {0.96, 1.0}


@pytest.mark.parametrize("c", range(int(G["n_train"])))
def test_oracle_minibatch_plan_and_feeds_equal_the_reference(c):
    g = lambda k: G["train%d_%s" % (c, k)]    # noqa: E731
    N, A = len(g("rewards")), int(g("dim"))
    assert N > 5000 and N % 128 != 0
    plan = op.minibatches(N, 128, 5000)
    rows = np.concatenate([np.arange(lo, hi) for lo, hi in plan])
    assert len(plan) == 39                                    # floor(5000 / 128): the tail rows are dropped
    np.testing.assert_array_equal(g("critic_rows"), rows)     # in order, not shuffled
    np.testing.assert_array_equal(g("actor_rows"), rows)
    np.testing.assert_array_equal(_bits(g("critic_targets")), _bits(g("returns")[rows][:, None]))
    np.testing.assert_array_equal(_bits(g("actor_actions")), _bits(g("actions")[rows].reshape(-1, A)))
    adv = op.fill_advantages(g("rewards"), g("values"), g("game_overs").astype(bool), g("returns"), 0.99,
                             float(g("lambda")), str(g("rescaler")))
    np.testing.assert_array_equal(_bits(g("actor_advantages")), _bits(adv[rows]))
    # the old policy is the actor's target network on the minibatch's own rows (the stand-in's per-row values)
    want = np.stack([np.sin(rows + j).astype(np.float32) for j in range(A)], 1)
    np.testing.assert_array_equal(g("actor_old_mean"), want)
    assert g("actor_old_std").shape == (len(rows), A)
    # post_training_commands: the coefficient update on the last epoch's KL mean, then memory.clean()
    k = op.update_kl_coefficient(g("kl_before"), float(np.float32(g("kl_value"))), 0.01)
    assert _bits(np.float32(k)) == _bits(np.float32(g("kl_after")))
    assert list(g("memory_calls")) == ["clean"]


@pytest.mark.parametrize("c", range(int(G["n_kl"])))
def test_oracle_kl_coefficient_trajectories_equal_the_reference(c):
    k = G["kl%d_initial" % c]
    got = []
    for m in G["kl%d_means" % c]:
        k = op.update_kl_coefficient(k, m, float(G["kl%d_target" % c]))
        got.append(k)
    np.testing.assert_array_equal(_bits(np.array(got, np.float32)), _bits(G["kl%d_coefficients" % c]))


def test_kl_trajectories_move_both_ways():
    c = G["kl1_coefficients"]
    assert c[19] < G["kl1_initial"] < c[-1]


@pytest.mark.parametrize("k", range(int(G["n_acting"])))
def test_normal_draw_equals_the_reference(k):
    means, stds = G["act%d_means" % k], G["act%d_stds" % k]
    E, A = means.shape
    np.random.seed(int(G["act%d_seed" % k]))
    n = np.random.standard_normal((E, A))                  # what E successive np.random.normal calls draw
    np.testing.assert_array_equal(_bits(op.normal_action(means, stds, n)), _bits(G["act%d_train" % k]))
    np.testing.assert_array_equal(G["act%d_eval" % k], means)
    from coach_b200.schedules import LinearSchedule
    s = LinearSchedule(0.5, 0.1, 7)
    for _ in range(E):
        s.step()
    assert float(s.current_value) == float(G["act%d_noise_after" % k])


@pytest.mark.parametrize("kl_coef,cutoff,use_kl", [(0.5, 1.0, True), (0.5, 0.001, True), (0.5, 0.001, False)])
def test_kl_head_gradient_hand_worked(kl_coef, cutoff, use_kl):
    """A = 1, B = 2 by hand: KL_i = log(s / so) + (so^2 + (mo_i - m_i)^2) / (2 s^2) - 1/2 with s = e^l + eps"""
    eps, hp, beta = 1e-15, 1000.0, 0.01
    mu, mo, a, adv = np.array([0.3, -0.2]), np.array([0.1, 0.0]), np.array([0.5, -1.0]), np.array([1.5, -0.5])
    l, lo = 0.2, 0.0
    s, so = np.exp(l) + eps, np.exp(lo) + eps
    kl = np.log(s / so) + (so ** 2 + (mo - mu) ** 2) / (2 * s ** 2) - 0.5
    klbar = kl.mean()
    logp = -0.5 * ((a - mu) / s) ** 2 - np.log(s) - 0.5 * np.log(2 * np.pi)
    logpo = -0.5 * ((a - mo) / so) ** 2 - np.log(so) - 0.5 * np.log(2 * np.pi)
    ratio = np.exp(logp - logpo)
    f = (kl_coef + 2 * hp * max(0.0, klbar - cutoff)) if use_kl else 0.0
    d_mu = (-adv * ratio * (a - mu) / s ** 2 + f * (mu - mo) / s ** 2) / 2
    ds = (s - eps) / s
    d_l = ((-adv * ratio * (((a - mu) / s) ** 2 - 1)).sum() / 2 + f * (1 - (so / s) ** 2 - ((mu - mo) / s) ** 2).sum() / 2
           - beta) * ds
    entropy = 0.5 * (1 + np.log(2 * np.pi)) + np.log(s)
    surrogate = -(ratio * adv).mean()
    loss = surrogate - beta * entropy + ((kl_coef * klbar + hp * max(0.0, klbar - cutoff) ** 2) if use_kl else 0.0)
    g_mu, g_l, sc = op.kl_head(mu[:, None], [l], a[:, None], mo[:, None], [lo], adv, kl_coef, cutoff, hp, use_kl,
                               beta)
    np.testing.assert_allclose(g_mu[:, 0], d_mu, rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(g_l, [d_l], rtol=1e-12, atol=1e-15)
    np.testing.assert_allclose(sc, [loss, klbar, entropy, ratio.mean(), surrogate], rtol=1e-12, atol=1e-15)
    assert (klbar > cutoff) == (cutoff < 0.01)


def test_defaults_equal_the_reference():
    from coach_b200.agents.ppo_agent import PPOAgentParameters, network_widths
    ap = PPOAgentParameters()
    alg = ap.algorithm
    got = [alg.gae_lambda, alg.target_kl_divergence, alg.initial_kl_coefficient, alg.high_kl_penalty_coefficient,
           alg.value_targets_mix_fraction, alg.beta_entropy, alg.num_consecutive_playing_steps.num_steps,
           alg.discount, alg.num_consecutive_training_steps]
    np.testing.assert_array_equal(np.array(got, np.float64), G["par_algorithm"])
    assert [alg.clip_likelihood_ratio_using_epsilon is None, alg.estimate_state_value_using_gae,
            alg.use_kl_regularization, alg.act_for_full_episodes] == list(G["par_flags"])
    assert alg.policy_gradient_rescaler.name == str(G["par_rescaler"])
    for row, name in zip(G["par_networks"], ("critic", "actor")):
        n = ap.network_wrappers[name]
        np.testing.assert_array_equal([n.batch_size, n.learning_rate, n.optimizer_epsilon, n.adam_optimizer_beta1,
                                       n.adam_optimizer_beta2, float(n.create_target_network), n.l2_regularization],
                                      row)
        assert n.optimizer_type == str(G["par_%s_optimizer" % name])
        assert list(G["par_%s_schemes" % name]) == ["Medium", "Medium"]
        assert network_widths(n) == (256, 512)
    assert type(ap.exploration).__name__ == str(G["par_box_exploration"])
    s = ap.exploration.noise_schedule
    np.testing.assert_array_equal([s.initial_value, s.final_value, s.decay_steps, ap.exploration.evaluation_noise,
                                   float(ap.exploration.noise_as_percentage_from_action_space)], G["par_box_noise"])
    assert ap.path == 'coach_b200.agents.ppo_agent:PPOAgent'


def test_preset_equals_the_reference():
    import importlib
    from coach_b200.agents.ppo_agent import network_widths
    mod = importlib.import_module("coach_b200.presets.Mujoco_PPO")
    ap = mod.agent_params
    np.testing.assert_array_equal([ap.network_wrappers['actor'].learning_rate,
                                   ap.network_wrappers['critic'].learning_rate, ap.algorithm.initial_kl_coefficient,
                                   ap.algorithm.gae_lambda], G["pre_mujoco"])
    for row, name in zip(G["pre_mujoco_widths"], ("actor", "critic")):
        assert network_widths(ap.network_wrappers[name]) == tuple(row)
    assert [type(f).__name__ for flt in ap.input_filter._observation_filters.values() for f in flt.values()] == \
        list(G["pre_mujoco_observation_filters"])
    assert str(G["pre_mujoco_reward_test_level"]) == "inverted_pendulum"
    assert (mod.observation_dim, mod.action_dim) == (4, 1)


def _params():
    from coach_b200.agents.ppo_agent import PPOAgentParameters
    return PPOAgentParameters()


def _refuse(ap, match, **kw):
    from coach_b200.agents import ppo_agent
    args = dict(observation_dim=4, action_dim=1, action_low=-1.0, action_high=1.0, device="cpu")
    args.update(kw)
    with pytest.raises(ValueError, match=match):
        ppo_agent.PPOAgent(ap, **args)


def test_refusals():
    from coach_b200.agents.actor_critic_agent import PolicyGradientRescaler
    from coach_b200.base_parameters import Dense, MiddlewareScheme
    _refuse(_params(), "continuous", continuous_actions=False)
    _refuse(_params(), "bounded", action_low=None)
    _refuse(_params(), "bounded", action_high=np.array([np.inf]))
    _refuse(_params(), "action dimensions", action_dim=33)
    ap = _params()
    ap.algorithm.clip_likelihood_ratio_using_epsilon = 0.2
    _refuse(ap, "clip_likelihood_ratio_using_epsilon")
    for name in ("actor", "critic"):
        ap = _params()
        ap.network_wrappers[name].optimizer_type = 'LBFGS'
        _refuse(ap, "Adam only")
    for r in (PolicyGradientRescaler.FUTURE_RETURN, PolicyGradientRescaler.TD_RESIDUAL):
        ap = _params()
        ap.algorithm.policy_gradient_rescaler = r
        _refuse(ap, "GAE or A_VALUE")
    for emb, mid in (([Dense(64)], MiddlewareScheme.Medium), ([Dense(128)], [Dense(128)]),
                     ([Dense(64), Dense(64)], [Dense(64)]), ("Medium", MiddlewareScheme.Deep)):
        ap = _params()
        ap.network_wrappers["critic"].input_embedders_parameters['observation'].scheme = emb
        ap.network_wrappers["critic"].middleware_parameters.scheme = mid
        _refuse(ap, "widths")
    ap = _params()
    ap.network_wrappers["critic"].batch_size = 64
    _refuse(ap, "batch sizes")


def test_refuses_several_ranks(monkeypatch):
    from coach_b200 import parallel
    monkeypatch.setattr(parallel, "world", lambda: (0, 2))
    _refuse(_params(), "one rank")

