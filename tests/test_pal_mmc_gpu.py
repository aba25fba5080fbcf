"""PAL and Mixed Monte Carlo on the GPU: the fused head's target rules against the reference fixture
(tests/golden/pal_mmc.npz) and the oracle (oracle/pal_mmc.py, pinned to the reference by tests/test_pal_mmc_host.py),
whole learn steps against the fp32 / fp64 oracle, the DDQN anchors, CUDA-graph replay, and the episodic replay's
fused sample path, Monte Carlo returns, Episodes granularity and checkpoints."""
import ctypes
import os
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pal_mmc.npz")
RULES = ["mmc", "pal", "pal_persistent"]


def close(got, want, rtol=1e-5, name="", atol=0.0):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    err = np.abs(got - want).max() if got.size else 0.0
    tol = rtol * np.abs(want).max() + atol
    assert err <= tol, "%s: max abs err %.3e > %.3e" % (name, err, tol)


@pytest.fixture(scope="module")
def g():
    return dict(np.load(GOLDEN))


def _agent(rule, obs, A, B, huber=True, alpha=0.9, rate=0.1, seed=0, memory=None, discount=0.99):
    from coach_b200.agents.mmc_agent import MixedMonteCarloAgent, MixedMonteCarloAgentParameters
    from coach_b200.agents.pal_agent import PALAgent, PALAgentParameters
    from coach_b200.memories.memory import MemoryGranularity
    ap = MixedMonteCarloAgentParameters() if rule == "mmc" else PALAgentParameters()
    ap.memory.max_size = memory or (MemoryGranularity.Transitions, 1024)
    if memory is not None and memory[0] == MemoryGranularity.Episodes:
        ap.memory.transition_capacity = 1024
    ap.algorithm.monte_carlo_mixing_rate = rate
    ap.algorithm.discount = discount
    if rule != "mmc":
        ap.algorithm.pal_alpha = alpha
        ap.algorithm.persistent_advantage_learning = rule == "pal_persistent"
    net = ap.network_wrappers["main"]
    net.batch_size = B
    net.replace_mse_with_huber_loss = huber
    cls = MixedMonteCarloAgent if rule == "mmc" else PALAgent
    return cls(ap, observation_shape=obs, num_actions=A, seed=seed)


def _data(obs, A, n, seed=5):
    """n transitions in episodes of 1..12 steps, the last one closed"""
    rng = np.random.RandomState(seed)
    if len(obs) == 3:
        s = rng.randint(0, 256, (n,) + obs).astype(np.uint8)
        s2 = rng.randint(0, 256, (n,) + obs).astype(np.uint8)
    else:
        s = rng.uniform(-1, 1, (n,) + obs).astype(np.float32)
        s2 = rng.uniform(-1, 1, (n,) + obs).astype(np.float32)
    done = np.zeros(n, dtype=np.uint8)
    i = -1
    while i < n - 1:
        i = min(n - 1, i + int(rng.randint(1, 13)))
        done[i] = 1
    return {"state:observation": s, "next_state:observation": s2, "action": rng.randint(0, A, n).astype(np.int64),
            "reward": rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], n).astype(np.float64), "game_over": done}


# ---- the head kernel on the fixture's crafted rows ---------------------------------------------------------------------
def _head_call(lib, rule, q, actions, rewards, dones, returns, discount, alpha, rate):
    """cb200_dqn_head_fused on planted Q values: h = [Q | 0] and W = [I; 0], so every Q value the kernel computes is
    the planted one (one product by 1 plus zeros)"""
    from coach_b200 import _lib
    B, A = actions.shape[0], q["q_online"].shape[1]
    F = 256
    dev = "cuda"

    def feat(x):
        h = np.zeros((B, F), dtype=np.float32)
        h[:, :A] = x
        return torch.from_numpy(h).to(dev)
    w = np.zeros((F, A), dtype=np.float32)
    w[:A] = np.eye(A, dtype=np.float32)
    keep = dict(h_next=feat(q["q_next"]), h_online=feat(q["q_online"]), h_select=feat(q["q_select"]),
                h_target_s=feat(q["q_target_s"]), w=torch.from_numpy(w).to(dev),
                b=torch.zeros(A, dtype=torch.float32, device=dev), actions=torch.from_numpy(actions).to(dev),
                rewards=torch.from_numpy(rewards).to(dev), dones=torch.from_numpy(dones).to(dev),
                returns=torch.from_numpy(np.ascontiguousarray(returns)).to(dev))
    outs = {k: torch.zeros((B, A), dtype=torch.float32, device=dev) for k in
            ("q_online", "q_next", "targets", "dq", "q_select", "q_target_s")}
    td = torch.zeros(B, dtype=torch.float64, device=dev)
    dw, db = torch.zeros((F, A), device=dev), torch.zeros(A, device=dev)
    ws = torch.zeros(((B + 15) // 16) * 8 * (F * A + A + 1), device=dev)
    d = _lib.DqnHeadDesc()
    d.h_next, d.h_online, d.h_select = (keep[k].data_ptr() for k in ("h_next", "h_online", "h_select"))
    d.w_target = d.w_online = keep["w"].data_ptr()
    d.b_target = d.b_online = keep["b"].data_ptr()
    d.actions, d.rewards, d.game_overs = (keep[k].data_ptr() for k in ("actions", "rewards", "dones"))
    d.discount, d.huber, d.batch, d.features, d.n_actions = discount, 1, B, F, A
    for k in ("q_online", "q_next", "targets", "dq", "q_select", "q_target_s"):
        setattr(d, k, outs[k].data_ptr())
    d.td_err, d.dw, d.db, d.workspace = td.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr()
    d.target_rule = {"dqn": _lib.TARGET_DQN, "mmc": _lib.TARGET_MMC, "pal": _lib.TARGET_PAL,
                     "pal_persistent": _lib.TARGET_PAL_PERSISTENT}[rule]
    d.h_target_s, d.mc_returns = keep["h_target_s"].data_ptr(), keep["returns"].data_ptr()
    d.pal_alpha, d.mc_mixing_rate = alpha, rate
    _lib.check(lib.cb200_dqn_head_fused(ctypes.byref(d), _lib.current_stream()))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in outs.items()}


@pytest.mark.parametrize("tag", ["", "_b"])
@pytest.mark.parametrize("rule", RULES)
def test_head_kernel_targets_equal_the_reference_bit_for_bit(g, rule, tag):
    from coach_b200 import _lib
    from oracle.pal_mmc import mmc_targets, pal_targets
    lib = _lib.load()
    alpha, rate = (float(x) for x in g["alpha_rate" + tag])
    q = {k: g[k] for k in ("q_next", "q_select", "q_target_s", "q_online")}
    out = _head_call(lib, rule, q, g["actions"], g["rewards"], g["game_overs"], g["returns"], float(g["discount"]),
                     alpha, rate)
    for k in ("q_online", "q_next", "q_select") + (("q_target_s",) if rule != "mmc" else ()):
        np.testing.assert_array_equal(out[k], q[k], err_msg=k)             # the planted values came through exactly
    common = dict(actions=g["actions"], rewards=g["rewards"], game_overs=g["game_overs"], returns=g["returns"],
                  discount=float(g["discount"]), mixing_rate=rate)
    if rule == "mmc":
        want = mmc_targets(out["q_next"], out["q_select"], out["q_online"], **common)
    else:
        want = pal_targets(out["q_next"], out["q_select"], out["q_target_s"], out["q_online"], alpha=alpha,
                           persistent=rule == "pal_persistent", **common)
    np.testing.assert_array_equal(out["targets"].view(np.uint32), want.view(np.uint32))
    np.testing.assert_array_equal(out["targets"].view(np.uint32), g["%s%s_targets" % (rule, tag)].view(np.uint32))


def test_head_refuses_a_descriptor_without_its_inputs():
    from coach_b200 import _lib
    lib = _lib.load()
    d = _lib.DqnHeadDesc()
    x = torch.zeros(4096, device="cuda")
    for f in ("h_next", "h_online", "h_select", "w_target", "b_target", "w_online", "b_online", "actions", "rewards",
              "game_overs", "q_online", "targets", "td_err", "dq", "dw", "db", "workspace"):
        setattr(d, f, x.data_ptr())
    d.batch, d.features, d.n_actions = 8, 256, 4
    d.target_rule = _lib.TARGET_PAL
    d.mc_returns = x.data_ptr()
    assert lib.cb200_dqn_head_fused(ctypes.byref(d), _lib.current_stream()) != 0        # no h_target_s
    d.target_rule, d.mc_returns = _lib.TARGET_MMC, None
    assert lib.cb200_dqn_head_fused(ctypes.byref(d), _lib.current_stream()) != 0        # no mc_returns
    d.mc_returns, d.h_select = x.data_ptr(), None
    assert lib.cb200_dqn_head_fused(ctypes.byref(d), _lib.current_stream()) != 0        # no h_select
    d.target_rule = 7
    assert lib.cb200_dqn_head_fused(ctypes.byref(d), _lib.current_stream()) != 0


# ---- whole learn steps against the oracle ------------------------------------------------------------------------------
def _oracle_check(agent, rule, obs, A, steps=2):
    from oracle import nets as on, pal_mmc as op
    from test_learn_gpu import _device_relu_masks
    store, net = agent.net_def.store, agent.networks["main"]
    net.theta_target.copy_(store.theta * 0.9 + 0.01)
    net.target_changed()
    o32 = on.QNetOracle(obs, A, False, torch.float32)
    o64 = on.QNetOracle(obs, A, False, torch.float64)
    huber = bool(net.params.replace_mse_with_huber_loss)
    alpha, rate = getattr(agent, "alpha", 0.9), agent.mixing_rate
    for step in range(steps):
        online_named, target_named = store.export_named(), store.export_named(net.theta_target)
        if step == 0:
            opt32 = on.AdamTF([torch.from_numpy(v) for v in online_named.values()], 2.5e-4, 0.9, 0.99, 1e-4)
            opt64 = on.AdamTF([torch.from_numpy(v).double() for v in online_named.values()], 2.5e-4, 0.9, 0.99, 1e-4,
                              dtype=torch.float64)
        random.seed(20 + step)
        np.random.seed(20 + step)
        batch = agent.sample_batch()
        total, _, gnorm = agent.learn_from_batch(batch)
        torch.cuda.synchronize()
        for k in ("state:observation", "next_state:observation"):
            batch.column(k)
        cols = {k: v.cpu().numpy() for k, v in batch.columns.items()}
        ob = dict(states=cols["state:observation"], next_states=cols["next_state:observation"], actions=cols["action"],
                  rewards=cols["reward"], game_overs=cols["game_over"], returns=cols["n_step_discounted_rewards"])
        masks = _device_relu_masks(agent)
        k32, k64 = dict(masks=masks, tol=1e-5), dict(masks=masks, tol=1e-5)
        kw = dict(alpha=alpha, mixing_rate=rate, huber_loss=huber)
        ref = op.learn_step(o32, o32.cast(online_named), o32.cast(target_named), opt32, ob, 0.99, rule, kink=k32, **kw)
        ref64 = op.learn_step(o64, o64.cast(online_named), o64.cast(target_named), opt64, ob, 0.99, rule, kink=k64,
                              **kw)
        assert k32.get("hard", 0) == 0 and k64.get("hard", 0) == 0, "ReLU masks differ away from the kink"
        # targets: the oracle prologue on the device's own Q values, bit for bit
        qo, qn, qs = (t.cpu().numpy() for t in (net.online_s.q, net.target_s2.q, agent.q_select))
        common = dict(actions=ob["actions"], rewards=ob["rewards"], game_overs=ob["game_overs"], returns=ob["returns"],
                      discount=0.99, mixing_rate=rate)
        if rule == "mmc":
            want_t = op.mmc_targets(qn, qs, qo, **common)
        else:
            want_t = op.pal_targets(qn, qs, agent.q_target_s.cpu().numpy(), qo, alpha=alpha,
                                    persistent=rule == "pal_persistent", **common)
            close(agent.q_target_s.cpu().numpy(), ref["q_target_s"], name="q_target_s", atol=1e-6)
        np.testing.assert_array_equal(agent.targets.cpu().numpy().view(np.uint32), want_t.view(np.uint32))
        close(qo, ref["q_online"], name="q_online", atol=1e-6)
        assert abs(total - ref["loss"]) <= 1e-5 * max(1.0, abs(ref["loss"])), (total, ref["loss"])
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


@pytest.mark.parametrize("rule", RULES)
@pytest.mark.parametrize("obs,A,B,huber", [((4,), 2, 32, False), ((84, 84, 4), 6, 32, True),
                                           ((84, 84, 4), 6, 128, True), ((60, 76, 3), 4, 32, False)],
                         ids=["cartpole_B32_mse", "atari_B32", "atari_B128", "doom_B32_mse"])
def test_learn_step_matches_oracle(rule, obs, A, B, huber):
    torch.manual_seed(0)
    agent = _agent(rule, obs, A, B, huber=huber)
    assert agent.head_desc is not None
    assert (agent.networks["main"].target_s is not None) == (rule != "mmc")
    if B >= 128 and len(obs) == 3:
        assert agent.s2d is not None                               # the fused s2d input path through the episodic replay
    agent.memory.store_columns(_data(obs, A, max(256, 2 * B)))
    _oracle_check(agent, rule, obs, A)


@pytest.mark.parametrize("rule", RULES)
def test_zero_alpha_and_mixing_equal_ddqn(rule):
    from test_learn_gpu import _make_agent
    obs, A, B = (84, 84, 4), 6, 32
    agent = _agent(rule, obs, A, B, alpha=0.0, rate=0.0, seed=7)
    ddqn = _make_agent(obs, A, B, False, True, False, seed=7)
    for a in (agent, ddqn):
        a.networks["main"].theta_target.copy_(a.net_def.store.theta * 0.9 + 0.01)
        a.networks["main"].target_changed()
    cols = _data(obs, A, 256)
    agent.memory.store_columns(cols)
    ddqn.memory.store_columns(cols)
    for step in range(2):
        np.random.seed(4 + step)
        la, _, ga = agent.learn_from_batch(agent.sample_batch())
        np.random.seed(4 + step)
        ld, _, gd = ddqn.learn_from_batch(ddqn.sample_batch())
        assert (la, ga) == (ld, gd)
        assert torch.equal(agent.targets, ddqn.targets)
        assert torch.equal(agent.net_def.store.theta, ddqn.net_def.store.theta)


@pytest.mark.parametrize("rule", ["pal", "mmc"])
def test_graph_replay_is_bit_identical_to_eager(monkeypatch, rule):
    results = []
    for graph in (0, 1):
        monkeypatch.setenv("CB200_DQN_GRAPH", str(graph))
        torch.manual_seed(0)
        agent = _agent(rule, (84, 84, 4), 6, 128)
        assert agent.use_graph == bool(graph) and agent.s2d is not None
        agent.memory.store_columns(_data((84, 84, 4), 6, 512, seed=3))
        out = []
        for step in range(6):                          # 2 eager steps, capture, 3 replays
            np.random.seed(20 + step)
            out.append(agent.learn_from_batch(agent.sample_batch())[:2])
        torch.cuda.synchronize()
        if graph:
            assert agent._graphs is not None and agent.graph_kernel_launches > 0
        results.append((out, agent.net_def.store.theta.clone(), agent.targets.clone()))
    assert results[0][0] == results[1][0]
    assert torch.equal(results[0][1], results[1][1]) and torch.equal(results[0][2], results[1][2])


def test_refusals():
    from coach_b200.agents.pal_agent import PALAgent, PALAgentParameters
    from coach_b200.memories.experience_replay import ExperienceReplayParameters
    from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplayParameters
    for mem in (PrioritizedExperienceReplayParameters(), ExperienceReplayParameters()):
        ap = PALAgentParameters()
        ap.memory = mem
        with pytest.raises(NotImplementedError):
            PALAgent(ap, observation_shape=(4,), num_actions=2)
    ap = PALAgentParameters()
    ap.network_wrappers["main"].heads_parameters = ["DuelingQHead"]
    with pytest.raises(NotImplementedError):
        PALAgent(ap, observation_shape=(4,), num_actions=2)
    ap = PALAgentParameters()
    ap.memory.max_size = (ap.memory.max_size[0], 256)
    with pytest.raises(NotImplementedError):                       # more actions than the fused head takes
        PALAgent(ap, observation_shape=(4,), num_actions=9)
    agent = _agent("mmc", (4,), 2, 32)
    agent.memory.store_columns(_data((4,), 2, 64))
    batch = agent.sample_batch()
    del batch.columns["n_step_discounted_rewards"]
    with pytest.raises(ValueError):
        agent.learn_from_batch(batch)


# ---- the episodic replay -----------------------------------------------------------------------------------------------
def test_s2d_sample_equals_sample_then_convert():
    from coach_b200 import _lib
    agent = _agent("pal", (84, 84, 4), 6, 128)
    assert agent.s2d is not None
    agent.memory.store_columns(_data((84, 84, 4), 6, 400))
    np.random.seed(11)
    fused = agent.sample_batch()
    planes = {k: v.to_dense().clone() if hasattr(v, "to_dense") else v.clone() for k, v in agent.s2d["columns"].items()}
    idx = fused.columns["idx"].clone()
    np.random.seed(11)
    plain = agent.memory.sample_batch(128)
    assert torch.equal(plain.columns["idx"], idx)
    H, W, C, S = agent.s2d["geometry"]
    for k, want in planes.items():
        x = plain.columns[k].contiguous()
        _lib.check(agent.lib.cb200_u8_s2d_planes(x.data_ptr(), 128, H, W, C, S, agent.s2d["columns"][k].ptr,
                                                 _lib.current_stream()))
        got = agent.s2d["columns"][k]
        got = got.to_dense() if hasattr(got, "to_dense") else got
        assert torch.equal(got, want), k
        assert torch.equal(fused.column(k), x)
    for k in ("action", "reward", "game_over", "n_step_discounted_rewards"):
        assert torch.equal(fused.columns[k], plain.columns[k]), k
    mem = agent.memory
    assert torch.equal(fused.columns["n_step_discounted_rewards"], mem._returns[idx])
    assert fused.columns["n_step_discounted_rewards"].data_ptr() == \
        agent.batch_buffers["n_step_discounted_rewards"].data_ptr()


def test_episodes_granularity_reproduces_the_reference_session(g):
    """an MMC agent with discount 0.95 on an Episodes-sized replay: the reference's counters after every store and its
    seeded samples with their returns -- discounted by 0.99, the Episode default, whatever the agent's discount"""
    from coach_b200.core_types import Transition
    from coach_b200.memories.memory import MemoryGranularity
    k = int(g["ep_k"])
    agent = _agent("mmc", (1,), 2, 32, memory=(MemoryGranularity.Episodes, k), discount=0.95)
    mem = agent.memory
    counters, checks = g["ep_counters"], list(g["ep_sample_at"])
    sid, c = 0, 0
    for L in g["ep_lengths"]:
        for j in range(int(L)):
            mem.store(Transition(state={"observation": np.array([sid], dtype=np.float32)}, action=0,
                                 reward=float(g["ep_rewards"][sid]),
                                 next_state={"observation": np.array([sid + 1], dtype=np.float32)},
                                 game_over=j == L - 1))
            got = [mem.num_transitions(), mem.num_transitions_in_complete_episodes(), mem.num_complete_episodes(),
                   mem.length()]
            assert got == list(counters[sid]), (sid, got, counters[sid])
            sid += 1
            if checks and checks[0] == sid:
                checks.pop(0)
                np.random.seed(1000 + sid)
                b = mem.sample_batch(7)
                ids = b.columns["state:observation"].cpu().numpy()[:, 0]
                rets = b.columns["n_step_discounted_rewards"].cpu().numpy()
                np.testing.assert_array_equal(ids, g["ep_samples"][c][:, 0])
                np.testing.assert_allclose(rets, g["ep_samples"][c][:, 1], rtol=1e-12, atol=1e-12)
                assert torch.equal(b.columns["n_step_discounted_rewards"], mem._returns[b.columns["idx"]])
                c += 1
    assert c == len(g["ep_samples"])


def test_episodes_granularity_refuses_to_overwrite_listed_episodes():
    from coach_b200.core_types import Transition
    from coach_b200.memories.episodic_experience_replay import EpisodicExperienceReplay
    from coach_b200.memories.memory import MemoryGranularity
    with pytest.raises(ValueError):
        EpisodicExperienceReplay((MemoryGranularity.Episodes, 2))
    mem = EpisodicExperienceReplay((MemoryGranularity.Episodes, 2), transition_capacity=8)
    mk = lambda i, done: Transition(state={"observation": np.zeros(2)}, action=0, reward=1.0,   # noqa: E731
                                    next_state={"observation": np.zeros(2)}, game_over=done)
    for i in range(5):
        mem.store(mk(i, i == 4))
    with pytest.raises(ValueError):
        for i in range(4):
            mem.store(mk(i, False))                     # 5 listed + 4 open > 8 slots


def test_checkpoint_restore_continues_bit_identically(tmp_path):
    from coach_b200 import checkpoint
    obs, A, B = (84, 84, 4), 6, 32
    a = _agent("pal_persistent", obs, A, B, seed=1)
    a.memory.store_columns(_data(obs, A, 300, seed=2))

    def steps(agent, n, seed):
        out = []
        for k in range(n):
            np.random.seed(seed + k)
            out.append(agent.learn_from_batch(agent.sample_batch())[:2])
        return out
    steps(a, 3, 10)
    a.networks["main"].update_target_network(1.0)
    steps(a, 1, 30)
    name = checkpoint.save_checkpoint(a, str(tmp_path), checkpoint_id=1)
    want = steps(a, 3, 40)
    b = _agent("pal_persistent", obs, A, B, seed=9)
    checkpoint.restore_checkpoint(b, str(tmp_path), name)
    assert b.memory.episode_lengths == a.memory.episode_lengths
    got = steps(b, 3, 40)
    assert got == want
    assert torch.equal(b.net_def.store.theta, a.net_def.store.theta)
    assert torch.equal(b.targets, a.targets)
