"""Policy Gradients (REINFORCE) without a GPU: the oracle (oracle/pg.py) against the reference fixture
(tests/golden/pg.npz, written by oracle/make_golden_pg.py from the unmodified agent) bit for bit -- the returns, the four
rescalers, numpy's pairwise mean and std, the per-timestep table over a sequence of episodes, AdditiveNoise -- a
hand-worked episode, the split of closed episodes into learn steps, the defaults and presets and the agent's
refusals."""
import os

import numpy as np
import pytest

from oracle import pg as op

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pg.npz")))


def bits(x):
    return np.asarray(x, dtype=np.float64).view(np.uint64)


@pytest.mark.parametrize("c", range(int(G["n_cases"])))
def test_oracle_returns_and_targets_equal_the_reference_bit_for_bit(c):
    r, disc = G["c%d_rewards" % c], float(G["c%d_discount" % c])
    R = op.episode_returns(r, disc)
    np.testing.assert_array_equal(bits(R), bits(G["c%d_returns" % c]))
    for name in op.RESCALERS:
        t = op.episode_targets(R, name, op.TimestepTable(1000))
        np.testing.assert_array_equal(bits(t), bits(G["c%d_%s" % (c, name.lower())]), err_msg=name)


def test_zero_std_episode_gets_zero_targets():
    c = [k for k in range(int(G["n_cases"])) if not G["c%d_rewards" % k].any()][0]
    assert not G["c%d_future_return_normalized_by_episode" % c].any()
    assert op.mean_std(G["c%d_returns" % c])[1] == 0


@pytest.mark.parametrize("n", [1, 2, 7, 8, 9, 15, 16, 17, 127, 128, 129, 130, 255, 256, 257, 1000, 1001, 4099, 20000])
def test_pairwise_sum_mean_and_std_are_numpys(n):
    rng = np.random.RandomState(n)
    for x in (rng.randn(n) * 10 ** rng.randint(-3, 4), rng.choice([0.1, 1 / 3., 1e8, -1e-8], n)):
        assert bits(op.pairwise_sum(x)) == bits(np.add.reduce(x))
        m, s = op.mean_std(x)
        assert bits(m) == bits(np.mean(x)) and bits(s) == bits(np.std(x))


def test_pairwise_order_is_not_a_running_sum():
    x = np.array([1e16] + [1.0] * 200 + [-1e16])
    assert op.pairwise_sum(x) == np.add.reduce(x) and op.pairwise_sum(x) != sum(x.tolist())


def test_table_sequence_equals_the_reference():
    table = op.TimestepTable(1000)
    for k in range(int(G["n_seq"])):
        R = op.episode_returns(G["seq%d_rewards" % k], 0.99)
        table.fold(R)
        n = len(G["seq%d_mean_table" % k])
        np.testing.assert_array_equal(bits(table.mean[:n]), bits(G["seq%d_mean_table" % k]))
        np.testing.assert_array_equal(bits(table.count[:n]), bits(G["seq%d_count_table" % k]))
        np.testing.assert_array_equal(bits(op.mean_std(R)), bits(G["seq%d_mean_std" % k]))


def test_timestep_targets_along_the_sequence_equal_the_reference():
    """the default rescaler on the reference's running table: the targets learn_from_batch handed over"""
    table = op.TimestepTable(1000)
    nonzero = 0
    for k in range(int(G["n_seq"])):
        R = op.episode_returns(G["seq%d_rewards" % k], 0.99)
        t = op.episode_targets(R, "FUTURE_RETURN_NORMALIZED_BY_TIMESTEP", table)
        np.testing.assert_array_equal(bits(t), bits(G["seq%d_targets" % k]))
        nonzero += int((t != 0).sum())
    assert nonzero > 300


def test_bucket_rows():
    from coach_b200.agents.policy_gradients_agent import bucket_rows
    assert [bucket_rows(n) for n in (1, 32, 33, 256, 257, 320, 321, 513, 1000, 1025, 5000)] == \
        [32, 32, 64, 256, 320, 320, 384, 640, 1024, 1280, 5120]
    sizes = {bucket_rows(n) for n in range(1, 100001)}
    assert len(sizes) <= 4 * 9 + 8                            # 32-row steps to 256, then four per doubling
    assert all(bucket_rows(n) >= n and bucket_rows(n) <= max(1.25 * n, n + 31) for n in range(1, 100001, 7))


def test_additive_noise_equals_the_reference():
    means = G["noise_means"]
    np.random.seed(int(G["noise_seed"]))
    z = np.random.standard_normal(len(means))                  # what successive np.random.normal calls draw
    got = op.additive_noise(means[:, 0], float(G["noise_value"]), G["noise_low"], G["noise_high"], z)
    np.testing.assert_array_equal(bits(got), bits(G["noise_train"][:, 0]))
    assert G["noise_eval"].dtype == np.float32
    np.testing.assert_array_equal(G["noise_eval"], means)


def test_hand_worked_episode():
    # rewards [1, 0, 2], discount 0.5: R = [1 + 0 + 0.5, 0 + 1, 2] = [1.5, 1, 2]
    R = op.episode_returns(np.array([1.0, 0.0, 2.0]), 0.5)
    np.testing.assert_array_equal(R, [1.5, 1.0, 2.0])
    np.testing.assert_array_equal(op.episode_targets(R, "TOTAL_RETURN"), [1.5, 1.5, 1.5])
    np.testing.assert_array_equal(op.episode_targets(R, "FUTURE_RETURN"), R)
    # mean 1.5, std sqrt((0 + 0.25 + 0.25) / 3)
    t = op.episode_targets(R, "FUTURE_RETURN_NORMALIZED_BY_EPISODE")
    np.testing.assert_array_equal(t, (R - 1.5) / np.sqrt(0.5 / 3))
    table = op.TimestepTable(4)
    np.testing.assert_array_equal(op.episode_targets(R, "FUTURE_RETURN_NORMALIZED_BY_TIMESTEP", table), [0, 0, 0])
    # a second episode [3, 3]: m = [(1.5 + 3) / 2, (1 + 3) / 2] = [2.25, 2]; targets [0.75, 1]
    R2 = np.array([3.0, 3.0])
    np.testing.assert_array_equal(op.episode_targets(R2, "FUTURE_RETURN_NORMALIZED_BY_TIMESTEP", table), [0.75, 1.0])
    np.testing.assert_array_equal(table.count, [2, 2, 1, 0])


def test_closed_episodes_split_at_multiples_of_x():
    assert op.split_parts(0, 12, 5) == [5, 5, 2]
    assert op.split_parts(3, 4, 5) == [2, 2]
    assert op.split_parts(4, 1, 5) == [1]
    assert op.split_parts(7, 3, 1) == [1, 1, 1]
    assert op.split_parts(0, 3, 5) == [3]


def test_defaults_and_presets_equal_the_reference():
    from coach_b200.agents.policy_gradients_agent import PolicyGradientsAgentParameters
    ap = PolicyGradientsAgentParameters()
    alg, net = ap.algorithm, ap.network_wrappers["main"]
    assert [alg.num_steps_between_gradient_updates, alg.apply_gradients_every_x_episodes, alg.beta_entropy,
            alg.discount, alg.n_step] == G["par_algorithm"].tolist()
    assert alg.policy_gradient_rescaler.name == str(G["par_rescaler"])
    assert [net.learning_rate, net.adam_optimizer_beta1, net.adam_optimizer_beta2, net.optimizer_epsilon,
            float(net.async_training), -1.0 if net.clip_gradients is None else net.clip_gradients,
            net.head_loss_weights[0]] == G["par_network"].tolist()
    assert [h + "Parameters" for h in net.heads_parameters] == G["par_heads"].tolist()
    assert sorted(type(v).__name__ for v in ap.exploration.values()) == G["par_exploration"].tolist()
    from coach_b200.presets import CartPole_PG, InvertedPendulum_PG
    for tag, mod in (("cartpole", CartPole_PG), ("pendulum", InvertedPendulum_PG)):
        p = mod.agent_params
        n, a = p.network_wrappers["main"], p.algorithm
        assert [n.learning_rate, a.discount, a.num_steps_between_gradient_updates, a.apply_gradients_every_x_episodes,
                a.beta_entropy] == G["pre_%s" % tag].tolist()
        assert a.policy_gradient_rescaler.name == str(G["pre_%s_rescaler" % tag])
        rf = p.input_filter._reward_filters
        assert [f.rescale_factor for f in rf.values()] == G["pre_%s_reward_rescale" % tag].tolist()
        obs = [type(f).__name__ for f in p.input_filter._observation_filters.get("observation", {}).values()] or [""]
        assert obs == G["pre_%s_observation_filters" % tag].tolist()
    assert InvertedPendulum_PG.observation_shape == (4,) and InvertedPendulum_PG.action_dim == 1
    assert InvertedPendulum_PG.action_high.tolist() == [3.0] and InvertedPendulum_PG.action_low.tolist() == [-3.0]


def test_rescaler_stays_importable_from_the_actor_critic_module():
    from coach_b200.agents import actor_critic_agent, policy_gradients_agent
    assert policy_gradients_agent.PolicyGradientRescaler is actor_critic_agent.PolicyGradientRescaler


def _agent(**kw):
    from coach_b200.agents.policy_gradients_agent import PolicyGradientsAgent
    from coach_b200.presets.CartPole_PG import agent_params
    import copy
    ap = copy.deepcopy(agent_params)
    for k, v in kw.pop("alg", {}).items():
        setattr(ap.algorithm, k, v)
    for k, v in kw.pop("net", {}).items():
        setattr(ap.network_wrappers["main"], k, v)
    args = dict(observation_shape=(4,), num_actions=2, device="cpu")
    args.update(kw)
    return PolicyGradientsAgent(ap, **args)


@pytest.mark.parametrize("case", ["rescaler", "n_step", "clip", "unbounded", "no_bounds"])
def test_refusals(case):
    from coach_b200.agents.actor_critic_agent import PolicyGradientRescaler
    kw = {"rescaler": dict(alg=dict(policy_gradient_rescaler=PolicyGradientRescaler.GAE)),
          "n_step": dict(alg=dict(n_step=5)),
          "clip": dict(net=dict(clip_gradients=40.0)),
          "unbounded": dict(num_actions=None, action_dim=1, action_low=[-np.inf], action_high=[np.inf]),
          "no_bounds": dict(num_actions=None, action_dim=1)}[case]
    with pytest.raises(ValueError):
        _agent(**kw)


def test_many_ranks_are_refused(monkeypatch):
    from coach_b200 import parallel
    monkeypatch.setattr(parallel, "is_distributed", lambda: True)
    with pytest.raises(ValueError):
        _agent()
