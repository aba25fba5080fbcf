"""N-step Q-learning on the GPU: cb200_nstep_q_head at the C ABI (the reference fixture's targets and bootstrap values
bit for bit, random segment tables against an fp64 evaluation, exact probes, repeat-call bits, argument errors) and the
agent (the reference schedule and the fp32 / fp64 oracle at E = 1, the segment mean at E = 16 / 64, graph replay
against eager steps, acting, checkpoint restore)."""
import ctypes
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "nstep_q.npz")))
EPS32 = 2.0 ** -24
HOR = {"N-Step": 1, "1-Step": 2, "none": 0}


def close(got, want, rtol=1e-5, name="", atol=0.0):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    err = np.abs(got - want).max() if got.size else 0.0
    tol = rtol * np.abs(want).max() + atol
    assert err <= tol, "%s: max abs err %.3e > %.3e" % (name, err, tol)


# ---- the head at the C ABI --------------------------------------------------------------------------------------------
def head(h, hb, w_t, b_t, w_o, b_o, actions, rewards, dones, offsets, lengths, discount, horizon, huber=0, rows=None,
         planes=False):
    """one cb200_nstep_q_head call on host arrays; returns every output as numpy"""
    from coach_b200 import _lib as L
    lib, dev = L.load(), "cuda"
    rows = rows or h.shape[0]
    K, A, S = h.shape[1], w_o.shape[1], len(offsets)
    T = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x, dtype=dt)).to(dev)       # noqa: E731
    t = dict(h=T(h, np.float32), hb=T(hb, np.float32), wt=T(w_t, np.float32), bt=T(b_t, np.float32),
             wo=T(w_o, np.float32), bo=T(b_o, np.float32), a=T(actions, np.int64), r=T(rewards, np.float64),
             d=T(dones, np.uint8), off=T(offsets, np.int32), len=T(lengths, np.int32))
    out = {k: torch.full(s, float("nan"), dtype=torch.float32, device=dev) for k, s in
           (("q", (rows, A)), ("dq", (rows, A)), ("loss", (1,)), ("targets", (rows, A)),
            ("boot", (S if horizon == 1 else rows,)), ("dh", (rows, K)), ("dw", (K, A)), ("db", (A,)))}
    ws = torch.full((((S + 3) // 4) * 4 * (K * A + A + 1),), float("nan"), device=dev)
    d = L.NstepQHeadDesc()
    d.h_online, d.h_boot = t["h"].data_ptr(), t["hb"].data_ptr()
    d.w_target, d.b_target, d.w_online, d.b_online = (t[k].data_ptr() for k in ("wt", "bt", "wo", "bo"))
    d.actions, d.rewards, d.game_overs = t["a"].data_ptr(), t["r"].data_ptr(), t["d"].data_ptr()
    d.seg_offsets, d.seg_lengths, d.segments, d.rows = t["off"].data_ptr(), t["len"].data_ptr(), S, rows
    d.discount, d.horizon, d.huber, d.features, d.n_actions = discount, horizon, huber, K, A
    d.q_online, d.dq, d.loss, d.targets = (out[k].data_ptr() for k in ("q", "dq", "loss", "targets"))
    d.bootstrap, d.dh, d.dw, d.db = (out[k].data_ptr() for k in ("boot", "dh", "dw", "db"))
    d.workspace = ws.data_ptr()
    pl = None
    if planes:
        pl = torch.zeros(3 * rows * K, dtype=torch.int16, device=dev)
        d.dh_planes, d.dh_plane_stride = pl.data_ptr(), rows * K
    L.check(lib.cb200_nstep_q_head(ctypes.byref(d), L.current_stream()))
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    res["_desc"], res["_keep"] = d, (t, out, ws, pl)
    return res


def planted(q, K):
    """h = [Q | 0] and W = [I; 0]: the head's Q values are exactly q"""
    n, A = q.shape
    h = np.zeros((n, K), dtype=np.float32)
    h[:, :A] = q
    w = np.zeros((K, A), dtype=np.float32)
    w[np.arange(A), np.arange(A)] = 1
    return h, w


@pytest.mark.parametrize("horizon", ["N-Step", "1-Step", "none"])
@pytest.mark.parametrize("K", [256, 512])
def test_fixture_targets_and_bootstrap_bit_for_bit(horizon, K):
    for c in range(int(G["n_cases"])):
        q, a, r = G["c%d_q_online" % c], G["c%d_actions" % c], G["c%d_rewards" % c]
        d, disc, qn = G["c%d_game_overs" % c], float(G["c%d_discount" % c]), G["c%d_q_next" % c]
        L, A = q.shape
        h, w = planted(q, K)
        hb, _ = planted(qn[-1:] if horizon == "N-Step" else qn, K)
        z = np.zeros(A, dtype=np.float32)
        o = head(h, hb, w, z, w, z, a, r.astype(np.float64), d, [0], [L], disc, HOR[horizon])
        want = G["c%d_%s_targets" % (c, horizon.lower().replace("-", ""))]
        np.testing.assert_array_equal(o["targets"].view(np.uint32), want.view(np.uint32), err_msg="case %d" % c)
        np.testing.assert_array_equal(o["q"], q)
        if horizon == "N-Step":
            assert o["boot"][0] == (0.0 if d[-1] else np.max(qn[-1]))
        elif horizon == "1-Step":
            np.testing.assert_array_equal(o["boot"], np.max(qn, axis=1))
        if horizon == "none":
            assert not o["dq"].any() and not o["dw"].any() and o["loss"][0] == 0


def _random(rng, S, K, A, maxlen=23, pad=0, mag=1.0):
    lengths = rng.randint(1, maxlen + 1, S)
    n = int(lengths.sum())
    rows = n + pad
    h = np.maximum(rng.randn(rows, K), 0).astype(np.float32) * mag
    hb = np.maximum(rng.randn(rows, K), 0).astype(np.float32)
    w_t, w_o = (rng.randn(2, K, A) * 0.05).astype(np.float32)
    b_t, b_o = (rng.randn(2, A) * 0.1).astype(np.float32)
    actions = rng.randint(0, A, rows).astype(np.int64)
    rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], rows)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int32)
    dones = np.zeros(rows, dtype=np.uint8)
    ends = offsets + lengths - 1
    dones[ends[rng.rand(S) < 0.4]] = 1
    perm = rng.permutation(S)                                  # the table's slot order is free
    return h, hb, w_t, b_t, w_o, b_o, actions, rewards, dones, offsets[perm], lengths[perm], rows


def _fp64_check(args, o, discount, horizon, huber):
    from oracle import nstep_q as oq
    h, hb, w_t, b_t, w_o, b_o, actions, rewards, dones, offsets, lengths, rows = args
    h64, w64 = h.astype(np.float64), w_o.astype(np.float64)
    q64 = h64 @ w64 + b_o
    S, A = len(offsets), w_o.shape[1]
    n = int(lengths.sum())
    sab = np.abs(h64) @ np.abs(w64) + np.abs(b_o)
    qb = (h.shape[1] + 2) * EPS32 * sab
    assert (np.abs(o["q"][:n] - q64[:n]) <= qb[:n]).all()
    # targets: the oracle on the kernel's own Q values and bootstrap maxima, bit for bit
    want_t = np.zeros_like(o["targets"])
    dq64 = np.zeros((rows, A))
    dqb = np.zeros((rows, A))
    loss64 = lossb = 0.0
    hz = "N-Step" if horizon == 1 else "1-Step"
    for s in range(S):
        o0, L = int(offsets[s]), int(lengths[s])
        sl = slice(o0, o0 + L)
        qn = np.full((L, A), o["boot"][s], np.float32) if horizon == 1 else \
            np.repeat(o["boot"][sl][:, None], A, axis=1)
        t, _ = oq.segment_targets(o["q"][sl], actions[sl], rewards[sl], dones[sl], discount, hz, qn)
        want_t[sl] = t
        e = (q64[sl] - t.astype(np.float64)) * (np.arange(A)[None, :] == actions[sl][:, None])   # 0 off the taken one
        if huber:
            g, l = np.clip(e, -1, 1), np.where(np.abs(e) <= 1, 0.5 * e * e, np.abs(e) - 0.5)
        else:
            g, l = 2 * e, e * e
        dq64[sl] = g / (S * L)
        dqb[sl] = (2 * qb[sl] + 4 * EPS32 * np.abs(g)) / (S * L)
        loss64 += l.sum() / L / S
        lossb += (np.abs(g) * qb[sl] + qb[sl] ** 2).sum() / L / S
    np.testing.assert_array_equal(o["targets"][:n].view(np.uint32), want_t[:n].view(np.uint32))
    assert np.isfinite(o["targets"]).all() and not o["targets"][n:].any() and not o["dq"][n:].any()
    err = np.abs(o["dq"] - dq64)
    assert (err <= dqb + 1e-30).all(), (err / (dqb + 1e-30)).max()
    dw64, dwb = h64.T @ dq64, np.abs(h64).T @ dqb + (rows + 2) * EPS32 * (np.abs(h64).T @ np.abs(dq64))
    db64, dbb = dq64.sum(0), dqb.sum(0) + (rows + 2) * EPS32 * np.abs(dq64).sum(0)
    dh64 = (dq64 @ w64.T) * (h > 0)
    dhb = (dqb @ np.abs(w64).T + 4 * EPS32 * np.abs(dq64) @ np.abs(w64).T) * (h > 0)
    for name, got, want, bound in (("dW", o["dw"], dw64, dwb), ("db", o["db"], db64, dbb), ("dh", o["dh"], dh64, dhb)):
        e = np.abs(got - want)
        ratio = (e / (bound + 1e-30)).max()
        print("%s: observed error / bound = %.3f" % (name, ratio))
        assert ratio <= 1.0, name
    lb = lossb + (rows + 8) * EPS32 * abs(loss64)
    print("loss: observed error / bound = %.3f" % (abs(o["loss"][0] - loss64) / (lb + 1e-30)))
    assert abs(o["loss"][0] - loss64) <= lb + 1e-30


@pytest.mark.parametrize("seed", range(6))
def test_random_segment_tables_against_fp64(seed):
    rng = np.random.RandomState(seed)
    S = [1, 3, 17, 64, 40, 8][seed]
    K = [256, 512][seed % 2]
    A = [1, 2, 6, 18, 18, 6][seed]
    horizon = 1 if seed % 3 else 2
    huber = seed % 2
    args = _random(rng, S, K, A, pad=[0, 5, 31, 7, 0, 19][seed])
    o = head(*args[:11], 0.99, horizon, huber, rows=args[11])
    _fp64_check(args, o, 0.99, horizon, huber)
    assert np.isfinite(o["dh"]).all() and not o["dh"][int(args[10].sum()):].any()


def test_dyadic_probe_is_exact():
    """small-integer features and dyadic weights: every product and sum is exact in fp32, so the kernel's outputs
    equal the fp64 evaluation exactly"""
    rng = np.random.RandomState(7)
    K, A, S = 256, 6, 4
    lengths = np.array([1, 2, 4, 1])
    rows = 8
    h = rng.randint(0, 4, (rows, K)).astype(np.float32)
    w = (rng.randint(-4, 5, (K, A)) / 64.0).astype(np.float32)
    b = np.zeros(A, np.float32)
    actions = rng.randint(0, A, rows)
    rewards = rng.randint(-2, 3, rows).astype(np.float64)
    offsets = np.array([0, 1, 3, 7], np.int32)
    dones = np.zeros(rows, np.uint8)
    dones[[0, 6]] = 1
    o = head(h, h, w, b, w, b, actions, rewards, dones, offsets, lengths, 0.5, 1, 0)
    q64 = h.astype(np.float64) @ w
    np.testing.assert_array_equal(o["q"], q64)
    dq = np.zeros((rows, A))
    for s in range(S):
        for i in range(offsets[s], offsets[s] + lengths[s]):
            dq[i, actions[i]] = 2 * (o["q"][i, actions[i]] - np.float64(o["targets"][i, actions[i]])) / (S * lengths[s])
    sc = np.abs(dq).max()
    assert np.abs(o["dq"] - dq).max() <= 4 * EPS32 * sc


def test_repeat_calls_and_planes_give_identical_bits():
    rng = np.random.RandomState(3)
    args = _random(rng, 33, 512, 18, pad=9)
    args = args[:11] + (args[11] + (-args[11]) % 8,)
    a = head(*args[:11], 0.99, 1, 1, rows=args[11])
    b = head(*args[:11], 0.99, 1, 1, rows=args[11], planes=True)
    for k in ("q", "dq", "loss", "targets", "boot", "dh", "dw", "db"):
        np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32), err_msg=k)
    t, out, ws, pl = b["_keep"]
    from coach_b200 import _lib as L
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.check(L.load().cb200_nstep_q_head(ctypes.byref(b["_desc"]), L.current_stream()))
    for v in out.values():
        v.fill_(float("nan"))
    graph.replay()
    torch.cuda.synchronize()
    for k in ("q", "dq", "loss", "dh", "dw", "db"):
        np.testing.assert_array_equal(out[k].cpu().numpy().view(np.uint32), a[k].view(np.uint32), err_msg=k)
    hi = pl.view(3, -1)[0].cpu().numpy().astype(np.uint16)
    dh = a["dh"].view(np.uint32)
    rows, K = dh.shape
    r, c = np.meshgrid(np.arange(rows), np.arange(K), indexing="ij")
    tiled = ((r // 8) * (K // 8) + c // 8) * 64 + (r % 8) * 8 + c % 8
    np.testing.assert_array_equal(hi[tiled], (dh >> 16).astype(np.uint16))


def test_argument_errors():
    from coach_b200 import _lib as L
    lib = L.load()
    rng = np.random.RandomState(1)
    args = _random(rng, 2, 256, 6)
    o = head(*args[:11], 0.99, 1, 0, rows=args[11])
    d = o["_desc"]
    call = lambda: L.check(lib.cb200_nstep_q_head(ctypes.byref(d), L.current_stream()))      # noqa: E731
    for field, bad in (("n_actions", 19), ("n_actions", 0), ("features", 128), ("horizon", 3), ("segments", 0),
                       ("rows", 0), ("h_online", None), ("workspace", None), ("seg_lengths", None)):
        old = getattr(d, field)
        setattr(d, field, bad)
        with pytest.raises(ValueError):
            call()
        setattr(d, field, old)
    d.dh_planes, d.dh_plane_stride = 256, 12
    with pytest.raises(ValueError):
        call()
    d.dh_planes = None
    call()


# ---- the agent --------------------------------------------------------------------------------------------------------
def _agent(obs, A, E=1, horizon="N-Step", t_max=5, copy=7, seed=0, atari_scheme=False, lr=2.5e-4):
    from coach_b200.agents.n_step_q_agent import NStepQAgent, NStepQAgentParameters
    from coach_b200.base_parameters import Conv2d, Dense, EnvironmentSteps
    ap = NStepQAgentParameters()
    ap.algorithm.targets_horizon = horizon
    ap.algorithm.num_steps_between_gradient_updates = t_max
    ap.algorithm.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(copy)
    ap.network_wrappers["main"].learning_rate = lr
    if atari_scheme:
        ap.network_wrappers["main"].input_embedders_parameters["observation"].scheme = [Conv2d(16, 8, 4),
                                                                                         Conv2d(32, 4, 2)]
        ap.network_wrappers["main"].middleware_parameters.scheme = [Dense(256)]
    return NStepQAgent(ap, observation_shape=obs, num_actions=A, num_envs=E, seed=seed)


def _stream(obs, A, E, steps, seed, p_end=0.15):
    rng = np.random.RandomState(seed)
    mk = (lambda n: rng.randint(0, 256, (n, E) + obs).astype(np.uint8)) if len(obs) == 3 else \
        (lambda n: rng.uniform(-1, 1, (n, E) + obs).astype(np.float32))
    s = mk(steps + 1)
    return dict(states=s[:-1], next_states=s[1:], actions=rng.randint(0, A, (steps, E)),
                rewards=rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], (steps, E)), dones=rng.rand(steps, E) < p_end)


def _oracle(agent, obs):
    from oracle import nets as on, nstep_q as oq
    nd = agent.net_def
    strides = tuple(l.S for l in nd.trunk.layers if hasattr(l, "S"))
    n_embed = sum(1 for l in nd.trunk.layers[:-1] if not hasattr(l, "S")) - len(nd.middleware_units)
    mk = lambda dt: oq.NStepQNetOracle(obs, agent.num_actions, dt, strides=strides or (4, 2, 1),      # noqa: E731
                                       n_embed=max(n_embed, 1), middleware=bool(nd.middleware_units))
    o32, o64 = mk(torch.float32), mk(torch.float64)
    named = nd.store.export_named()
    lr = agent.ap.network_wrappers["main"].learning_rate
    opt32 = on.AdamTF([torch.from_numpy(v) for v in named.values()], lr, 0.9, 0.99, 1e-4)
    opt64 = on.AdamTF([torch.from_numpy(v).double() for v in named.values()], lr, 0.9, 0.99, 1e-4,
                      dtype=torch.float64)
    return o32, o64, opt32, opt64


def _run_and_check(agent, obs, st, steps, horizon="N-Step"):
    """drive observe_batch / train over the stream; at every learn step compare the new parameters with the fp32 /
    fp64 oracle (1e-5, else no farther from fp64 than the fp32 oracle).  Returns the learned (step, [(stream, rows)])."""
    from oracle import nstep_q as oq
    o32, o64, opt32, opt64 = _oracle(agent, obs)
    net = agent.networks["main"]
    E = agent.num_envs
    hist = []
    learned, copies = [], []
    for t in range(steps):
        agent.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t], st["dones"][t])
        hist.append(t)
        before_on = agent.net_def.store.export_named()
        last_copy = agent.last_target_network_update_step
        tgt_named = None
        loss = agent.train()
        if agent.last_target_network_update_step != last_copy:
            copies.append(agent.total_steps_counter)
        if not agent.learned_segments:
            continue
        tgt_named = agent.net_def.store.export_named(net.theta_target)
        segs = []
        closed = [(e, end - start) for e, start, end in agent.learned_segments]
        learned.append((t, closed))
        for e, L in closed:
            ts = list(range(t - L + 1, t + 1))
            segs.append(dict(states=st["states"][ts, e], next_states=st["next_states"][ts, e],
                             actions=st["actions"][ts, e], rewards=st["rewards"][ts, e],
                             game_overs=st["dones"][ts, e].astype(np.uint8)))
        ref = oq.learn_step(o32, o32.cast(before_on), o32.cast(tgt_named), opt32, segs, 0.99, horizon)
        ref64 = oq.learn_step(o64, o64.cast(before_on), o64.cast(tgt_named), opt64, segs, 0.99, horizon)
        assert abs(loss - ref["loss"]) <= 1e-5 * max(1.0, abs(ref["loss"])), (loss, ref["loss"])
        got = agent.net_def.store.export_named()
        for name in ref["new_params"]:
            want = ref["new_params"][name].numpy()
            try:
                close(got[name], want, name="param " + name)
            except AssertionError as exc:
                w64 = ref64["new_params"][name].numpy()
                e_ours, e_orc = np.abs(got[name] - w64).max(), np.abs(want - w64).max()
                assert e_ours <= 2 * e_orc, "%s; vs fp64: ours %.3e, fp32 oracle %.3e" % (exc, e_ours, e_orc)
    return learned, copies


@pytest.mark.parametrize("obs,A,atari", [((4,), 2, False), ((84, 84, 4), 6, True)], ids=["cartpole", "atari"])
def test_one_stream_follows_the_reference_schedule_and_the_oracle(obs, A, atari):
    from oracle import nstep_q as oq
    torch.manual_seed(0)
    eps = G["sch_episodes"].tolist()
    steps = sum(eps)
    agent = _agent(obs, A, E=1, atari_scheme=atari, seed=1)
    st = _stream(obs, A, 1, steps, seed=4)
    st["dones"][:] = False
    st["dones"][np.cumsum(eps) - 1, 0] = True
    learned, copies = _run_and_check(agent, obs, st, steps)
    want = G["sch_t5_env7_segments"].tolist()
    assert [(t + 1, closed[0][1]) for t, closed in learned] == [(s[2], s[1] - s[0]) for s in want]
    assert copies == G["sch_t5_env7_copies"].tolist()
    assert agent.training_iteration == int(G["sch_t5_env7_training_iteration"])
    segs, _, _ = oq.schedule(eps, 5, "EnvironmentSteps", 7)
    assert [s[1] - s[0] for s in segs] == [c[0][1] for _, c in learned]


@pytest.mark.parametrize("E,horizon", [(16, "N-Step"), (16, "1-Step"), (64, "N-Step")])
def test_many_streams_learn_the_segment_mean(E, horizon):
    from oracle import nstep_q as oq
    torch.manual_seed(0)
    obs, A = (4,), 2
    steps = 14
    agent = _agent(obs, A, E=E, horizon=horizon, seed=2)
    st = _stream(obs, A, E, steps, seed=5)
    learned, _ = _run_and_check(agent, obs, st, steps, horizon)
    assert [(t, sorted(c)) for t, c in learned] == [(t, sorted(c)) for t, c in oq.lockstep_schedule(st["dones"], 5)
                                                     if c]


def test_graph_replay_is_bit_identical_to_eager(monkeypatch):
    obs, A, E, steps = (4,), 2, 60, 20          # every stream cuts at steps 5, 10, ...: 300 rows, a 320-row bucket

    def run(graph):
        monkeypatch.setenv("CB200_NSTEP_GRAPH", "1" if graph else "0")
        a = _agent(obs, A, E=E, seed=3)
        st = _stream(obs, A, E, steps, seed=6, p_end=0.0)
        losses = []
        for t in range(steps):
            a.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t], st["dones"][t])
            losses.append(a.train())
        return a, losses
    g, lg = run(True)
    e, le = run(False)
    assert g.graph_kernel_launches > 0 and e.graph_kernel_launches == 0
    assert lg == le
    assert torch.equal(g.net_def.store.theta, e.net_def.store.theta)


def test_acting_matches_the_oracle_forward():
    from oracle import nstep_q as oq
    from coach_b200.exploration_policies.e_greedy import EGreedyParameters
    obs, A, E = (84, 84, 4), 6, 16
    agent = _agent(obs, A, E=E, atari_scheme=True, seed=4)
    x = np.random.RandomState(0).randint(0, 256, (E,) + obs).astype(np.uint8)
    pol = EGreedyParameters().make(A, E)
    actions, q = agent.choose_actions(x, pol)
    o = oq.NStepQNetOracle(obs, A, torch.float64, strides=(4, 2))
    ref = o.forward(o.cast(agent.net_def.store.export_named()), x).numpy()
    close(q, ref, rtol=1e-5, name="q")
    assert actions.shape == (E,) and ((actions >= 0) & (actions < A)).all()


def test_checkpoint_restore_continues_identically(tmp_path):
    from coach_b200 import checkpoint
    obs, A, E, steps = (4,), 2, 1, 30
    st = _stream(obs, A, E, 2 * steps, seed=8, p_end=0.0)
    a = _agent(obs, A, E=E, seed=5)

    def run(agent, lo, hi):
        out = []
        for t in range(lo, hi):
            agent.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t],
                                st["dones"][t])
            out.append(agent.train())
        return out
    run(a, 0, steps)                                           # 30 steps at t_max 5: the last step closed a segment
    name = checkpoint.save_checkpoint(a, str(tmp_path), checkpoint_id=1)
    want = run(a, steps, 2 * steps)
    b = _agent(obs, A, E=E, seed=9)
    checkpoint.restore_checkpoint(b, str(tmp_path), name)
    got = run(b, steps, 2 * steps)
    assert got == want
    assert torch.equal(b.net_def.store.theta, a.net_def.store.theta)
    assert b.training_iteration == a.training_iteration
