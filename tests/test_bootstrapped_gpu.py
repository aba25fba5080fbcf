"""Bootstrapped DQN on the GPU: the learn step against the oracle restatement (oracle/bootstrapped.py, whose prologue
tests/test_bootstrapped_host.py pins to the reference), the bootstrap masks and the gradient rescale, the K = 1 anchor
against DDQN, CUDA-graph replay, ensemble acting, and the ``info:mask`` replay column through store, gather and
checkpoints."""
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

def close(got, want, rtol=1e-5, name="", atol=0.0):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    err = np.abs(got - want).max() if got.size else 0.0
    tol = rtol * np.abs(want).max() + atol
    assert err <= tol, "%s: max abs err %.3e > %.3e" % (name, err, tol)


def _agent(obs, A, B, K=10, p=1.0, r=None, huber=True, seed=0):
    from coach_b200.agents.bootstrapped_dqn_agent import BootstrappedDQNAgent, BootstrappedDQNAgentParameters
    from coach_b200.memories.memory import MemoryGranularity
    ap = BootstrappedDQNAgentParameters()
    ap.memory.max_size = (MemoryGranularity.Transitions, 1024)
    net = ap.network_wrappers["main"]
    net.batch_size = B
    net.replace_mse_with_huber_loss = huber
    net.num_output_head_copies = K
    net.rescale_gradient_from_head_by_factor = 1.0 / K if r is None else r
    ap.exploration.architecture_num_q_heads = K
    ap.exploration.bootstrapped_data_sharing_probability = p
    return BootstrappedDQNAgent(ap, observation_shape=obs, num_actions=A, seed=seed)


def _data(obs, A, n, seed=5):
    rng = np.random.RandomState(seed)
    if len(obs) == 3:
        s = rng.randint(0, 256, (n,) + obs).astype(np.uint8)
        s2 = rng.randint(0, 256, (n,) + obs).astype(np.uint8)
    else:
        s = rng.uniform(-1, 1, (n,) + obs).astype(np.float32)
        s2 = rng.uniform(-1, 1, (n,) + obs).astype(np.float32)
    return {"state:observation": s, "next_state:observation": s2, "action": rng.randint(0, A, n).astype(np.int64),
            "reward": rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], n).astype(np.float64),
            "game_over": (rng.rand(n) < 0.2).astype(np.uint8)}


def _fill(agent, obs, A, n, seed=5):
    cols = _data(obs, A, n, seed)
    np.random.seed(seed)
    cols["info:mask"] = agent.draw_bootstrap_masks(n)
    agent.memory.store_columns(cols)
    return cols


def _oracle_check(agent, obs, A, B, K, steps=2):
    from oracle import bootstrapped as ob, nets as on
    from test_learn_gpu import _device_relu_masks
    store, net = agent.net_def.store, agent.networks["main"]
    net.theta_target.copy_(store.theta * 0.9 + 0.01)
    net.target_changed()
    o32 = on.QNetOracle(obs, K * A, False, torch.float32)
    o64 = on.QNetOracle(obs, K * A, False, torch.float64)
    huber = bool(net.params.replace_mse_with_huber_loss)
    for step in range(steps):
        online_named, target_named = store.export_named(), store.export_named(net.theta_target)
        if step == 0:
            opt32 = on.AdamTF([torch.from_numpy(v) for v in online_named.values()], 2.5e-4, 0.9, 0.99, 1e-4)
            opt64 = on.AdamTF([torch.from_numpy(v).double() for v in online_named.values()], 2.5e-4, 0.9, 0.99, 1e-4,
                              dtype=torch.float64)
        random.seed(20 + step)
        np.random.seed(20 + step)
        batch = agent.sample_batch()
        total, losses, gnorm = agent.learn_from_batch(batch)
        torch.cuda.synchronize()
        for k in ("state:observation", "next_state:observation"):
            batch.column(k)
        cols = {k: v.cpu().numpy() for k, v in batch.columns.items()}
        ob_ = dict(states=cols["state:observation"], next_states=cols["next_state:observation"], actions=cols["action"],
                   rewards=cols["reward"], game_overs=cols["game_over"], masks=cols["info:mask"])
        masks = _device_relu_masks(agent)
        k32, k64 = dict(masks=masks, tol=1e-5), dict(masks=masks, tol=1e-5)
        ref = ob.bootstrapped_learn_step(o32, o32.cast(online_named), o32.cast(target_named), opt32, ob_, 0.99, K,
                                         agent.grad_rescale, huber, kink=k32)
        ref64 = ob.bootstrapped_learn_step(o64, o64.cast(online_named), o64.cast(target_named), opt64, ob_, 0.99, K,
                                           agent.grad_rescale, huber, kink=k64)
        assert k32.get("hard", 0) == 0 and k64.get("hard", 0) == 0, "ReLU masks differ away from the kink"
        # targets: the oracle prologue on the device's own Q values, bit for bit
        qo, qn, qs = (t.cpu().numpy() for t in (net.online_s.q, net.target_s2.q, agent.q_select))
        want_t = ob.bootstrapped_targets(ob.split_heads(qn, K), ob.split_heads(qs, K), ob.split_heads(qo, K),
                                         ob_["actions"], ob_["rewards"], ob_["game_overs"], ob_["masks"], 0.99)
        got_t = ob.split_heads(agent.targets.cpu().numpy(), K)
        for h in range(K):
            np.testing.assert_array_equal(got_t[h].view(np.uint32), want_t[h].view(np.uint32))
        close(qo, ref["q_online"], name="q_online", atol=1e-6)
        assert len(losses) == K
        for h in range(K):
            assert abs(losses[h] - ref["losses"][h]) <= 1e-5 * max(1.0, abs(ref["losses"][h])), (h, losses[h])
        assert abs(total - ref["loss"]) <= 1e-5 * max(1.0, abs(ref["loss"]))
        close(gnorm, ref["grad_norm"], name="grad_norm", rtol=2e-5)
        got_grads = store.export_named(store.grad)
        for name in ref["grads"]:
            want = ref["grads"][name].numpy()
            e_ours = np.abs(got_grads[name] - ref64["grads"][name].numpy()).max()
            e_orc = np.abs(want - ref64["grads"][name].numpy()).max()
            try:
                close(got_grads[name], want, name="grad " + name)
            except AssertionError as exc:
                assert e_ours <= 1.5 * e_orc, "%s; vs fp64: ours %.3e, fp32 oracle %.3e" % (exc, e_ours, e_orc)
            assert e_ours <= 4 * e_orc + 2e-6 * (np.abs(want).max() + 1e-30), (name, e_ours, e_orc)
        got_params = store.export_named()
        for name in ref["new_params"]:
            want = ref["new_params"][name].numpy()
            try:
                close(got_params[name], want, name="param " + name)
            except AssertionError as exc:
                w64 = ref64["new_params"][name].numpy()
                e_ours, e_orc = np.abs(got_params[name] - w64).max(), np.abs(want - w64).max()
                assert e_ours <= 2 * e_orc, "%s; vs fp64: ours %.3e, fp32 oracle %.3e" % (exc, e_ours, e_orc)


@pytest.mark.parametrize("obs,A,B,p,huber", [((4,), 2, 32, 1.0, False), ((84, 84, 4), 6, 32, 0.5, True),
                                             ((84, 84, 4), 6, 128, 0.5, True), ((84, 84, 4), 6, 128, 1.0, True)],
                         ids=["cartpole_B32_mse", "atari_B32_p05", "atari_B128_p05", "atari_B128_p1"])
def test_bootstrapped_learn_step_matches_oracle(obs, A, B, p, huber):
    torch.manual_seed(0)
    agent = _agent(obs, A, B, K=10, p=p, huber=huber)
    assert agent.head_desc is not None and agent.networks["main"].online_s.q.shape == (B, 10 * A)
    if B >= 128 and len(obs) == 3:
        assert agent.s2d is not None                               # the fused s2d input path
    _fill(agent, obs, A, max(256, 2 * B))
    _oracle_check(agent, obs, A, B, 10)


def test_masked_head_has_zero_gradient_and_rescale_only_reaches_the_trunk():
    obs, A, B, K = (84, 84, 4), 6, 32, 4
    cols = _data(obs, A, 256)
    mask = np.ones((256, K), dtype=np.uint8)
    mask[:, 2] = 0                                                 # head 2 never learns
    grads = []
    for r in (0.1, 1.0):
        agent = _agent(obs, A, B, K=K, r=r, seed=3)
        agent.memory.store_columns(dict(cols, **{"info:mask": mask}))
        np.random.seed(1)
        agent.learn_from_batch(agent.sample_batch())
        torch.cuda.synchronize()
        g = agent.net_def.store.export_named(agent.net_def.store.grad)
        wname, bname = agent.net_def.trunk.names[-1]
        np.testing.assert_array_equal(g[wname][:, 2 * A:3 * A], 0)
        np.testing.assert_array_equal(g[bname][2 * A:3 * A], 0)
        np.testing.assert_array_equal(agent.networks["main"].online_s.dq.cpu().numpy()[:, 2 * A:3 * A], 0)
        grads.append((g, wname, bname))
    (g1, wname, bname), (g2, _, _) = grads
    assert np.array_equal(g1[wname], g2[wname]) and np.array_equal(g1[bname], g2[bname])
    trunk = [n for n in g1 if n not in (wname, bname) and not n.endswith("rescalers")]
    for n in trunk:                                               # trunk gradients scale with r (linear in dh)
        close(g1[n], 0.1 * g2[n], rtol=2e-4, name=n, atol=1e-12)


def test_single_head_anchor_matches_ddqn():
    from test_learn_gpu import _make_agent
    obs, A, B = (84, 84, 4), 6, 32
    boot = _agent(obs, A, B, K=1, r=1.0, p=1.0, seed=7)
    ddqn = _make_agent(obs, A, B, False, True, False, seed=7)
    ddqn.net_def.store.theta.copy_(boot.net_def.store.theta)
    ddqn.networks["main"].online_changed()
    ddqn.networks["main"].sync()
    cols = _data(obs, A, 256)
    ddqn.memory.store_columns(cols)
    boot.memory.store_columns(dict(cols, **{"info:mask": np.ones((256, 1), dtype=np.uint8)}))
    np.random.seed(4)
    lb, lsb, _ = boot.learn_from_batch(boot.sample_batch())
    np.random.seed(4)
    ld, _, _ = ddqn.learn_from_batch(ddqn.sample_batch())
    assert abs(lb - ld) <= 1e-6 * abs(ld) and abs(lsb[0] - ld) <= 1e-6 * abs(ld)
    gb = boot.net_def.store.export_named(boot.net_def.store.grad)
    gd = ddqn.net_def.store.export_named(ddqn.net_def.store.grad)
    for n in gd:
        close(gb[n], gd[n], rtol=1e-6, name=n)


def test_graph_replay_is_bit_identical_to_eager(monkeypatch):
    results = []
    for graph in (0, 1):
        monkeypatch.setenv("CB200_DQN_GRAPH", str(graph))
        torch.manual_seed(0)
        agent = _agent((84, 84, 4), 6, 128, K=10, p=0.5)
        assert agent.use_graph == bool(graph)
        _fill(agent, (84, 84, 4), 6, 512, seed=3)
        out = []
        for step in range(6):                          # 2 eager steps, capture, 3 replays
            random.seed(20 + step)
            np.random.seed(20 + step)
            out.append(agent.learn_from_batch(agent.sample_batch())[:2])
        torch.cuda.synchronize()
        if graph:
            assert agent._graphs is not None and agent.graph_kernel_launches > 0
        results.append((out, agent.net_def.store.theta.clone()))
    assert results[0][0] == results[1][0]
    assert torch.equal(results[0][1], results[1][1])


def test_ensemble_action_values_kernel_matches_numpy():
    from coach_b200 import _lib
    lib = _lib.load()
    rng = np.random.RandomState(2)
    for E, K, A in ((64, 10, 6), (5, 3, 2), (7, 16, 8), (3, 1, 4)):
        q = rng.randn(E, K, A).astype(np.float32)
        q[::2] = (rng.randint(-2, 3, q[::2].shape) * 0.5).astype(np.float32)      # ties
        heads = rng.randint(0, K, E).astype(np.int32)
        qd, hd = torch.from_numpy(q).cuda(), torch.from_numpy(heads).cuda()
        out = torch.zeros((E, A), dtype=torch.float32, device="cuda")
        want = {
            _lib.ENSEMBLE_SELECT: q[np.arange(E), heads],
            _lib.ENSEMBLE_UCB: np.stack([np.mean(q[e], axis=0) + 0.1 * np.std(q[e], axis=0) for e in range(E)]),
            _lib.ENSEMBLE_MEAN: np.stack([np.mean(q[e], axis=0) for e in range(E)]),
            _lib.ENSEMBLE_VOTE: np.stack([np.eye(A)[np.argmax(np.bincount(np.argmax(q[e], axis=-1)))]
                                          for e in range(E)]).astype(np.float32),
        }
        for mode, w in want.items():
            _lib.check(lib.cb200_ensemble_action_values(qd.data_ptr(), E, K, A, mode, hd.data_ptr(), 0.1,
                                                        out.data_ptr(), _lib.current_stream()))
            got = out.cpu().numpy()
            assert w.dtype == np.float32
            np.testing.assert_array_equal(got.view(np.uint32), w.view(np.uint32), err_msg="mode %d %s" % (mode, (E, K, A)))


@pytest.mark.parametrize("tag", ["boot", "ucb"])
def test_choose_actions_reproduces_the_reference_actions(tag):
    """the fixture's [E, K, A] values, planted as the head's bias on an all-zero network, through choose_actions"""
    import os
    from coach_b200.exploration_policies.bootstrapped import BatchedBootstrapped, BatchedUCB
    from coach_b200.exploration_policies.e_greedy import RunPhase
    from coach_b200.schedules import LinearSchedule
    g = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bootstrapped.npz")))
    q, resets = g["pol_%s_q" % tag], g["pol_resets"]
    T, E = resets.shape
    K, A = q.shape[2:]
    agent = _agent((4,), A, 32, K=K)
    store = agent.net_def.store
    wname, bname = agent.net_def.trunk.names[-1]
    store.view(store.theta, wname).zero_()
    agent.networks["main"].online_changed()
    lo, hi, n = g["pol_eps"]
    np.random.seed(123)
    if tag == "boot":
        pol = BatchedBootstrapped(A, E, LinearSchedule(lo, hi, int(n)), float(g["pol_eval_eps"]), K)
    else:
        pol = BatchedUCB(A, E, LinearSchedule(lo, hi, int(n)), float(g["pol_eval_eps"]), K, float(g["pol_lamb"]))
    x = np.zeros((E, 4), dtype=np.float32)
    for t in range(T):
        if t == T - T // 3:
            pol.change_phase(RunPhase.TEST)
        for e in range(E):
            if resets[t, e]:
                pol.select_head(e)
        # one environment per call (the planted bias is shared by a batch): the epsilon-greedy draws of environment e
        # run on a one-environment view of the policy
        acts = np.zeros(E, dtype=np.int64)
        for e in range(E):
            store.view(store.theta, bname).copy_(torch.from_numpy(q[t, e].reshape(-1)))
            agent.networks["main"].online_changed()
            acts[e] = agent.choose_actions(x[:1], _OneEnv(pol, e))[0][0]
        np.testing.assert_array_equal(acts, g["pol_%s_actions" % tag][t], err_msg="step %d" % t)
    assert np.random.rand() == g["pol_%s_next_rand" % tag]


class _OneEnv(object):
    """environment e of a batched ensemble policy, as a policy over one environment"""

    def __init__(self, pol, e):
        self.pol, self.e = pol, e
        self.lamb = pol.lamb
        self.selected_head = pol.selected_head[e:e + 1]

    def ensemble_mode(self):
        return self.pol.ensemble_mode()

    def get_actions(self, v):
        from coach_b200.exploration_policies.e_greedy import RunPhase
        p, e = self.pol, self.e
        exploit = p.current_random_value[e] >= p.epsilon(e)
        p._observe_values(e, v[0], bool(exploit))
        eps = p.epsilon(e)
        if p.current_random_value[e] < eps:
            a = np.random.choice(np.arange(p.num_actions))
        else:
            a = np.argmax(np.random.random(v[0].shape) * (np.isclose(v[0], v[0].max())))
        if p.phase == RunPhase.TRAIN:
            p.epsilon_schedules[e].step()
        p.current_random_value[e] = np.random.rand()
        return np.array([a]), None


def test_choose_actions_runs_forward_and_ensemble_values():
    from coach_b200.exploration_policies.bootstrapped import BootstrappedParameters, UCBParameters
    agent = _agent((4,), 3, 32, K=5)
    x = np.random.RandomState(0).uniform(-1, 1, (6, 4)).astype(np.float32)
    for params in (BootstrappedParameters(), UCBParameters()):
        params.architecture_num_q_heads = 5
        np.random.seed(0)
        pol = params.make(3, 6)
        for e in range(6):
            pol.select_head(e)
        q = agent.get_all_q_values_for_states(x).cpu().numpy()
        assert q.shape == (6, 5, 3)
        want_v = pol.ensemble_values(q)
        acts, v = agent.choose_actions(x, pol)
        np.testing.assert_array_equal(v.view(np.uint32), want_v.view(np.uint32))
        assert acts.shape == (6,) and ((0 <= acts) & (acts < 3)).all()


def test_mask_column_through_store_gather_and_transitions():
    from coach_b200.core_types import Transition
    agent = _agent((4,), 2, 32, K=10, p=0.5)
    mem = agent.memory
    rng = np.random.RandomState(0)
    masks = []
    for i in range(40):
        m = rng.binomial(1, 0.5, 10)
        masks.append(m.astype(np.uint8))
        mem.store(Transition(state={"observation": rng.randn(4)}, action=int(rng.randint(2)), reward=1.0,
                             next_state={"observation": rng.randn(4)}, game_over=False, info={"mask": m}))
    cols = _data((4,), 2, 24)
    cm = rng.randint(0, 2, (24, 10)).astype(np.uint8)
    mem.store_columns(dict(cols, **{"info:mask": cm}))
    want = np.concatenate([np.stack(masks), cm])
    ts = [mem.get_transition(i) for i in range(64)]
    np.testing.assert_array_equal(np.stack([t.info["mask"] for t in ts]), want)
    np.random.seed(3)
    batch = agent.sample_batch()
    idx = batch.columns["idx"].cpu().numpy()
    np.testing.assert_array_equal(batch.columns["info:mask"].cpu().numpy(), want[idx])
    np.testing.assert_array_equal(np.stack([t.info["mask"] for t in batch.to_transitions()]), want[idx])
    with pytest.raises(ValueError):                    # the declared column has no source in this transition
        mem.store(Transition(state={"observation": rng.randn(4)}, action=0, reward=1.0,
                             next_state={"observation": rng.randn(4)}, game_over=False))
        mem._flush()


def test_undeclared_source_column_raises():
    from coach_b200.core_types import Transition
    from coach_b200.memories.experience_replay import ExperienceReplay
    from coach_b200.memories.memory import MemoryGranularity
    mem = ExperienceReplay((MemoryGranularity.Transitions, 64))
    mem.declare_schema({"state:observation": ((4,), np.float32), "next_state:observation": ((4,), np.float32),
                        "action": ((), np.int64), "reward": ((), np.float64), "game_over": ((), np.uint8),
                        "priority_hint": ((), np.float32)})
    with pytest.raises(ValueError):
        mem.store(Transition(state={"observation": np.zeros(4)}, action=0, reward=0.0,
                             next_state={"observation": np.zeros(4)}, game_over=True))


def test_checkpoint_restores_masks_and_continues_bit_identically(tmp_path):
    from coach_b200 import checkpoint
    obs, A, B = (84, 84, 4), 6, 32
    a = _agent(obs, A, B, K=10, p=0.5, seed=1)
    _fill(a, obs, A, 300, seed=2)

    def steps(agent, n, seed):
        out = []
        for k in range(n):
            np.random.seed(seed + k)
            out.append(agent.learn_from_batch(agent.sample_batch())[:2])
        return out
    steps(a, 3, 10)
    name = checkpoint.save_checkpoint(a, str(tmp_path), checkpoint_id=1)
    want = steps(a, 3, 40)
    b = _agent(obs, A, B, K=10, p=0.5, seed=9)
    checkpoint.restore_checkpoint(b, str(tmp_path), name)
    assert torch.equal(b.memory.ring.columns["info:mask"], a.memory.ring.columns["info:mask"])
    got = steps(b, 3, 40)
    assert got == want
    assert torch.equal(b.net_def.store.theta, a.net_def.store.theta)
