"""Bootstrapped DQN pinned to the reference on the host: the oracle prologue, the bootstrap-mask draw, the batched
Bootstrapped / UCB exploration and the parameter defaults against tests/golden/bootstrapped.npz (written from the
unmodified reference by oracle/make_golden_bootstrapped.py)."""
import importlib
import os

import numpy as np
import pytest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bootstrapped.npz")


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLDEN))


def test_oracle_prologue_equals_the_reference_targets(g):
    from oracle.bootstrapped import bootstrapped_targets
    K = g["pro_q_online"].shape[0]
    t = bootstrapped_targets(list(g["pro_q_next"]), list(g["pro_q_select"]), list(g["pro_q_online"]),
                             g["pro_actions"], g["pro_rewards"], g["pro_game_overs"], g["pro_masks"],
                             float(g["pro_discount"]))
    assert len(t) == K
    for h in range(K):
        assert t[h].dtype == np.float32
        np.testing.assert_array_equal(t[h].view(np.uint32), g["pro_targets"][h].view(np.uint32))
    # the fixture covers what it should: unmasked heads, terminal transitions, a transition no head learns from
    assert 0 < g["pro_masks"].mean() < 1 and g["pro_game_overs"].any() and not g["pro_masks"][0].any()
    np.testing.assert_array_equal(g["pro_targets"][:, 0], g["pro_q_online"][:, 0])


@pytest.mark.parametrize("tag,p", [("p1", 1.0), ("p05", 0.5)])
def test_bootstrap_masks_draw_like_observe(g, tag, p):
    from coach_b200.agents.bootstrapped_dqn_agent import draw_bootstrap_masks
    np.random.seed(77)
    m = draw_bootstrap_masks(12, p, 10)
    assert m.dtype == np.uint8
    np.testing.assert_array_equal(m, g["masks_" + tag])
    assert np.random.rand() == g["masks_%s_next_rand" % tag]       # same stream position, even at p = 1


def _policy(g, tag):
    from coach_b200.exploration_policies.bootstrapped import BatchedBootstrapped, BatchedUCB
    from coach_b200.schedules import LinearSchedule
    E = int(g["pol_E"])
    K, A = g["pol_%s_q" % tag].shape[2:]
    lo, hi, n = g["pol_eps"]
    sched = LinearSchedule(float(lo), float(hi), int(n))
    if tag == "boot":
        return BatchedBootstrapped(A, E, sched, float(g["pol_eval_eps"]), K)
    return BatchedUCB(A, E, sched, float(g["pol_eval_eps"]), K, float(g["pol_lamb"]))


@pytest.mark.parametrize("tag", ["boot", "ucb"])
def test_batched_policies_select_the_reference_actions(g, tag):
    """host [E, K, A] values through ensemble_values + get_actions: the reference's actions, last_action_values, heads,
    final epsilon and random-stream position"""
    from coach_b200.exploration_policies.e_greedy import RunPhase
    q, resets = g["pol_%s_q" % tag], g["pol_resets"]
    T, E = resets.shape
    T_train = T - T // 3                          # the fixture runs 2/3 of its steps in TRAIN, then TEST
    np.random.seed(123)
    pol = _policy(g, tag)
    want_lav = g["pol_%s_last_values" % tag]
    for t in range(T):
        if t == T_train:
            pol.change_phase(RunPhase.TEST)
        for e in range(E):
            if resets[t, e]:
                pol.select_head(e)
        actions, _ = pol.get_actions(pol.ensemble_values(q[t]))
        np.testing.assert_array_equal(actions, g["pol_%s_actions" % tag][t], err_msg="step %d" % t)
        if tag == "boot":
            np.testing.assert_array_equal(pol.selected_head, g["pol_boot_heads"][t])
        for e in range(E):
            v = pol.last_action_values[e]
            if np.isnan(want_lav[t, e]).all():
                assert v is None or np.isscalar(v), (t, e)
            else:
                np.testing.assert_array_equal(np.asarray(v, dtype=np.float64), want_lav[t, e], err_msg=str((t, e)))
    np.testing.assert_array_equal([s.current_value for s in pol.epsilon_schedules], g["pol_%s_final_eps" % tag])
    assert np.random.rand() == g["pol_%s_next_rand" % tag]


def test_presets_resolve_to_device_classes_with_the_reference_parameters(g):
    from coach_b200.utils import short_dynamic_import
    for name, expl in (("Atari_Bootstrapped_DQN", "BatchedBootstrapped"), ("Atari_UCB_with_Q_Ensembles", "BatchedUCB")):
        mod = importlib.import_module("coach_b200.presets." + name)
        ap = mod.agent_params
        assert (mod.observation_shape, mod.num_actions) == ((84, 84, 4), 6)
        assert short_dynamic_import(ap.path).__name__ == "BootstrappedDQNAgent"
        assert short_dynamic_import(ap.memory.path).__module__.startswith("coach_b200.memories")
        assert short_dynamic_import(ap.exploration.path).__name__ == expl
        net = ap.network_wrappers["main"]
        assert net.learning_rate == 0.00025
        assert net.num_output_head_copies == g["par_head_copies"]
        assert net.rescale_gradient_from_head_by_factor == g["par_rescale"]
        assert net.batch_size == g["par_batch_size"] and ap.memory.max_size[1] == g["par_memory_size"]
        ex = ap.exploration
        assert ex.architecture_num_q_heads == g["par_num_q_heads"]
        assert ex.bootstrapped_data_sharing_probability == g["par_share_prob"]
        if expl == "BatchedBootstrapped":
            s = ex.epsilon_schedule
            assert [s.initial_value, s.final_value, s.decay_steps] == list(g["par_boot_eps"])
            assert ex.evaluation_epsilon == g["par_eval_eps"]
        else:
            assert ex.lamb == g["par_ucb_lamb"] and ex.evaluation_epsilon == g["par_ucb_eval_eps"]
            got = [[sc.initial_value, sc.final_value, sc.decay_steps, st.num_steps]
                   for sc, st in ex.epsilon_schedule.schedules]
            np.testing.assert_array_equal(got, g["par_ucb_eps"])


def test_ensemble_network_layout_and_init():
    """one Dense(K A) head with per-block Glorot fans and K rescalers at r; K = 1 keeps the DQN layout"""
    import torch
    from coach_b200.architectures.q_network import QNetworkDef
    one = QNetworkDef("cpu", (84, 84, 4), 6)
    base = QNetworkDef("cpu", (84, 84, 4), 6, head_copies=1, head_grad_rescale=1.0)
    assert list(one.store.entries.items()) == list(base.store.entries.items())
    q = QNetworkDef("cpu", (84, 84, 4), 6, head_copies=10, head_grad_rescale=0.1)
    names = list(q.store.entries)
    assert names[-10:] == ["main/online/network_0/gradients_from_head_0-%d_rescalers" % k for k in range(10)]
    assert q.store.entries[names[-12]][1] == (512, 60)
    q.store.init_glorot(torch.Generator().manual_seed(0))
    named = q.store.export_named()
    w = named[names[-12]]
    assert np.abs(w).max() <= np.sqrt(6.0 / (512 + 6)) and np.abs(w).max() > np.sqrt(6.0 / (512 + 60))
    assert all(named[n][0] == np.float32(0.1) for n in names[-10:])
