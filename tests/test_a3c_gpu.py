"""Actor-Critic (A3C) on the GPU: cb200_actor_critic_head at the C ABI (the reference fixture's targets and advantages
bit for bit, random segment tables against an fp64 evaluation, an exact dyadic probe, repeat-call and graph-replay bits,
argument errors), cb200_categorical_act, and the agent (the fp32 / fp64 oracle at E = 1 on the CartPole_A3C and
Atari_A3C shapes, the segment mean at E = 16 / 64, graph replay against eager steps, acting, checkpoint restore)."""
import ctypes
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "a3c.npz")))
EPS32 = 2.0 ** -24
MODE = {"A_VALUE": 0, "GAE": 1, "GAE_VALUE": 2}


def close(got, want, rtol=1e-5, name="", atol=0.0):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    err = np.abs(got - want).max() if got.size else 0.0
    tol = rtol * np.abs(want).max() + atol
    assert err <= tol, "%s: max abs err %.3e > %.3e" % (name, err, tol)


# ---- the head at the C ABI --------------------------------------------------------------------------------------------
def head(h, hb, w, b, actions, rewards, dones, offsets, lengths, discount, mode, lam=0.96, beta=0.01, huber=0,
         rows=None, planes=False):
    """one cb200_actor_critic_head call on host arrays; returns every output as numpy"""
    from coach_b200 import _lib as L
    lib, dev = L.load(), "cuda"
    rows = rows or h.shape[0]
    K, N, S = h.shape[1], w.shape[1], len(offsets)
    A = N - 1
    T = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x, dtype=dt)).to(dev)       # noqa: E731
    t = dict(h=T(h, np.float32), hb=T(hb, np.float32), w=T(w, np.float32), b=T(b, np.float32),
             a=T(actions, np.int64), r=T(rewards, np.float64), d=T(dones, np.uint8), off=T(offsets, np.int32),
             len=T(lengths, np.int32))
    out = {k: torch.full(s, float("nan"), dtype=torch.float32, device=dev) for k, s in
           (("z", (rows, N)), ("dz", (rows, N)), ("loss", (1,)), ("probs", (rows, A)), ("targets", (rows,)),
            ("adv", (rows,)), ("boot", (S,)), ("dh", (rows, K)), ("dw", (K, N)), ("db", (N,)))}
    ws = torch.full((((S + 3) // 4) * 4 * (K * N + N + 1),), float("nan"), device=dev)
    d = L.ActorCriticHeadDesc()
    d.h, d.h_boot, d.w, d.b = (t[k].data_ptr() for k in ("h", "hb", "w", "b"))
    d.actions, d.rewards, d.game_overs = t["a"].data_ptr(), t["r"].data_ptr(), t["d"].data_ptr()
    d.seg_offsets, d.seg_lengths, d.segments, d.rows = t["off"].data_ptr(), t["len"].data_ptr(), S, rows
    d.discount, d.gae_lambda, d.mode, d.huber = discount, lam, mode, huber
    d.beta_entropy, d.v_weight, d.p_weight, d.features, d.n_actions = beta, 0.5, 1.0, K, A
    d.z, d.dz, d.loss, d.probs = (out[k].data_ptr() for k in ("z", "dz", "loss", "probs"))
    d.targets, d.advantages, d.bootstrap = (out[k].data_ptr() for k in ("targets", "adv", "boot"))
    d.dh, d.dw, d.db = (out[k].data_ptr() for k in ("dh", "dw", "db"))
    d.workspace = ws.data_ptr()
    pl = None
    if planes:
        pl = torch.zeros(3 * rows * K, dtype=torch.int16, device=dev)
        d.dh_planes, d.dh_plane_stride = pl.data_ptr(), rows * K
    L.check(lib.cb200_actor_critic_head(ctypes.byref(d), L.current_stream()))
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    res["_desc"], res["_keep"] = d, (t, out, ws, pl)
    return res


@pytest.mark.parametrize("mode", list(MODE))
@pytest.mark.parametrize("K", [256, 512])
def test_fixture_targets_and_advantages_bit_for_bit(mode, K):
    """V planted exactly: h = [V | 0], W = e_0 (column 0), zero logits"""
    for c in range(int(G["n_cases"])):
        v, boot, r = G["c%d_values" % c], G["c%d_boot" % c], G["c%d_rewards" % c]
        d, disc, lam = G["c%d_game_overs" % c], float(G["c%d_discount" % c]), float(G["c%d_lambda" % c])
        L = len(v)
        h = np.zeros((L, K), np.float32)
        h[:, 0] = v
        hb = np.zeros((1, K), np.float32)
        hb[0, 0] = boot
        w = np.zeros((K, 5), np.float32)
        w[0, 0] = 1
        o = head(h, hb, w, np.zeros(5, np.float32), np.zeros(L), r.astype(np.float64), d, [0], [L], disc, MODE[mode],
                 lam)
        np.testing.assert_array_equal(o["z"][:, 0], v)
        for key, got in (("targets", o["targets"]), ("advantages", o["adv"])):
            want = G["c%d_%s_%s" % (c, mode.lower(), key)].astype(np.float32)
            np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg="case %d %s" % (c, key))
        assert o["boot"][0] == (0.0 if d[-1] else boot)
        np.testing.assert_array_equal(o["probs"], np.full((L, 4), 0.25, np.float32))


def _random(rng, S, K, A, maxlen=23, pad=0):
    lengths = rng.randint(1, maxlen + 1, S)
    n = int(lengths.sum())
    rows = n + pad
    h = np.maximum(rng.randn(rows, K), 0).astype(np.float32)
    hb = np.maximum(rng.randn(S, K), 0).astype(np.float32)
    w = (rng.randn(K, A + 1) * 0.05).astype(np.float32)
    b = (rng.randn(A + 1) * 0.1).astype(np.float32)
    actions = rng.randint(0, A, rows).astype(np.int64)
    rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], rows)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int32)
    dones = np.zeros(rows, dtype=np.uint8)
    dones[(offsets + lengths - 1)[rng.rand(S) < 0.4]] = 1
    perm = rng.permutation(S)                                  # the table's slot order is free
    return h, hb, w, b, actions, rewards, dones, offsets[perm], lengths[perm], rows


def _fp64_check(args, o, discount, mode, lam, beta, huber):
    from oracle import a3c as oa
    h, hb, w, b, actions, rewards, dones, offsets, lengths, rows = args
    h64, w64 = h.astype(np.float64), w.astype(np.float64)
    z64 = h64 @ w64 + b
    S, N = len(offsets), w.shape[1]
    n = int(lengths.sum())
    zb = (h.shape[1] + 2) * EPS32 * (np.abs(h64) @ np.abs(w64) + np.abs(b))
    assert (np.abs(o["z"][:n] - z64[:n]) <= zb[:n]).all()
    boot64 = hb.astype(np.float64) @ w64[:, 0] + b[0]
    dz64 = np.zeros((rows, N))
    dzb = np.zeros((rows, 1))
    loss64 = labs = 0.0
    zk = o["z"].astype(np.float64)                             # the loss and dL/dZ in fp64 on the kernel's own outputs
    for s in range(S):
        o0, L = int(offsets[s]), int(lengths[s])
        sl = slice(o0, o0 + L)
        term = bool(dones[o0 + L - 1])
        assert o["boot"][s] == 0 if term else abs(o["boot"][s] - boot64[s]) <= (h.shape[1] + 2) * EPS32 * (
            np.abs(hb[s]).astype(np.float64) @ np.abs(w64[:, 0]) + abs(b[0]))
        # targets and advantages: the oracle on the kernel's own V values, bit for bit
        t, a = oa.segment_targets(o["z"][sl, 0], o["boot"][s], rewards[sl], dones[sl], discount, mode, lam)
        np.testing.assert_array_equal(o["targets"][sl], t.astype(np.float32))
        np.testing.assert_array_equal(o["adv"][sl], a.astype(np.float32))
        t, a = t.astype(np.float32).astype(np.float64), a.astype(np.float32).astype(np.float64)
        v, lg = zk[sl, 0], zk[sl, 1:]
        p = np.exp(lg - lg.max(1, keepdims=True))
        p /= p.sum(1, keepdims=True)
        u = p + np.finfo(np.float32).eps
        su = u.sum(1, keepdims=True)
        ls = np.log(u) - np.log(su)
        H = -(u * ls).sum(1)
        e = v - t
        if huber:
            lv, gv = np.where(np.abs(e) <= 1, 0.5 * e * e, np.abs(e) - 0.5), np.clip(e, -1, 1)
        else:
            lv, gv = e * e, 2 * e
        onehot = np.arange(N - 1)[None, :] == actions[sl][:, None]
        logp = ls[onehot]
        loss64 += (0.5 * lv.mean() - (logp * a).mean() - beta * H.mean()) / S
        labs += (0.5 * lv.mean() + np.abs(logp * a).mean() + beta * np.abs(H).mean()) / S
        c = 1.0 / (S * L)
        g = c * (-a[:, None] * (onehot / u - 1 / su) + beta * ls)
        dz64[sl, 0] = c * 0.5 * gv
        dz64[sl, 1:] = p * (g - (p * g).sum(1, keepdims=True))
        # fp32 softmax, logs and one division per row: within 2^-14 of the row's gradient scale
        dzb[sl, 0] = 2.0 ** -14 * (np.abs(dz64[sl]).max(1) + c * (np.abs(a) + beta * np.abs(ls).max(1)) +
                                   c * np.abs(gv))
        np.testing.assert_allclose(o["probs"][sl], p, rtol=0, atol=1e-6)
    assert not o["targets"][n:].any() and not o["dz"][n:].any() and not o["z"][n:].any()
    dw64, db64 = h64.T @ dz64, dz64.sum(0)
    dh64 = (dz64 @ w64.T) * (h > 0)
    # the reductions add the usual (n + 2) eps sums of absolute terms to the per-row dL/dZ bound
    dzb += 1e-30
    for name, got, want, bound in (
            ("dZ", o["dz"], dz64, np.broadcast_to(dzb, dz64.shape)),
            ("dW", o["dw"], dw64, np.abs(h64).T @ dzb + (rows + 2) * EPS32 * (np.abs(h64).T @ np.abs(dz64))),
            ("db", o["db"], db64, dzb.sum() + (rows + 2) * EPS32 * np.abs(dz64).sum(0)),
            ("dh", o["dh"], dh64, (dzb @ np.ones((1, N)) @ np.abs(w64).T + (N + 2) * EPS32 * np.abs(dz64) @
                                   np.abs(w64).T) * (h > 0))):
        ratio = (np.abs(got - want) / (bound + 1e-30)).max()
        print("%s: observed error / bound = %.3f" % (name, ratio))
        assert ratio <= 1.0, name
    lb = 2.0 ** -14 * labs + (rows + 8) * EPS32 * labs
    print("loss: observed error / bound = %.3f" % (abs(o["loss"][0] - loss64) / lb))
    assert abs(o["loss"][0] - loss64) <= lb


@pytest.mark.parametrize("seed", range(6))
def test_random_segment_tables_against_fp64(seed):
    rng = np.random.RandomState(seed)
    S = [1, 3, 17, 64, 40, 8][seed]
    K = [256, 512][seed % 2]
    A = [1, 2, 6, 18, 18, 6][seed]
    mode = list(MODE)[seed % 3]
    huber, lam, beta = seed % 2, [1.0, 0.96][seed % 2], [0.01, 0.05, 0.0][seed % 3]
    args = _random(rng, S, K, A, pad=[0, 5, 31, 7, 0, 19][seed])
    o = head(*args[:9], 0.99, MODE[mode], lam, beta, huber, rows=args[9])
    _fp64_check(args, o, 0.99, mode, lam, beta, huber)
    assert np.isfinite(o["dh"]).all() and not o["dh"][int(args[8].sum()):].any()


def test_dyadic_probe_is_exact():
    """one action (p = 1: no policy or entropy gradient), small-integer features, dyadic weights, segment lengths and
    counts powers of two: V, dL/dV, dW, db and dh are exact in fp32 and equal the fp64 evaluation"""
    rng = np.random.RandomState(7)
    K, S = 256, 4
    lengths = np.array([1, 2, 4, 1])
    rows = 8
    h = rng.randint(0, 4, (rows, K)).astype(np.float32)
    w = (rng.randint(-4, 5, (K, 2)) / 64.0).astype(np.float32)
    b = np.zeros(2, np.float32)
    rewards = rng.randint(-2, 3, rows).astype(np.float64)
    offsets = np.array([0, 1, 3, 7], np.int32)
    dones = np.ones(rows, np.uint8)
    o = head(h, h[:S], w, b, np.zeros(rows), rewards, dones, offsets, lengths, 0.5, MODE["A_VALUE"], beta=0.0)
    z = h.astype(np.float64) @ w
    np.testing.assert_array_equal(o["z"], z)
    dz = np.zeros((rows, 2))
    for s in range(S):
        for i in range(offsets[s], offsets[s] + lengths[s]):
            dz[i, 0] = (z[i, 0] - np.float64(o["targets"][i])) / (S * lengths[s])
    np.testing.assert_array_equal(o["dz"], dz)
    np.testing.assert_array_equal(o["dw"], h.astype(np.float64).T @ dz)
    np.testing.assert_array_equal(o["db"], dz.sum(0))
    np.testing.assert_array_equal(o["dh"], (dz @ w.astype(np.float64).T) * (h > 0))


def test_repeat_calls_graph_replay_and_planes_give_identical_bits():
    rng = np.random.RandomState(3)
    args = _random(rng, 33, 512, 18, pad=9)
    args = args[:9] + (args[9] + (-args[9]) % 8,)
    a = head(*args[:9], 0.99, 1, 0.96, 0.01, 1, rows=args[9])
    b = head(*args[:9], 0.99, 1, 0.96, 0.01, 1, rows=args[9], planes=True)
    keys = ("z", "dz", "loss", "probs", "targets", "adv", "boot", "dh", "dw", "db")
    for k in keys:
        np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32), err_msg=k)
    t, out, ws, pl = b["_keep"]
    from coach_b200 import _lib as L
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.check(L.load().cb200_actor_critic_head(ctypes.byref(b["_desc"]), L.current_stream()))
    for v in out.values():
        v.fill_(float("nan"))
    pl.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for k in keys:
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
    o = head(*args[:9], 0.99, 0, rows=args[9])
    d = o["_desc"]
    call = lambda: L.check(lib.cb200_actor_critic_head(ctypes.byref(d), L.current_stream()))      # noqa: E731
    for field, bad in (("n_actions", 19), ("n_actions", 0), ("features", 128), ("mode", 3), ("mode", -1),
                       ("segments", 0), ("rows", 0), ("h", None), ("h_boot", None), ("workspace", None),
                       ("seg_lengths", None), ("z", None)):
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
    z = torch.zeros((4, 3), device="cuda")
    act = torch.zeros(4, dtype=torch.int64, device="cuda")
    for envs, A, zp, ap in ((0, 2, z, act), (4, 0, z, act), (4, 19, z, act), (4, 2, None, act), (4, 2, z, None)):
        with pytest.raises(ValueError):
            L.check(lib.cb200_categorical_act(zp.data_ptr() if zp is not None else None, envs, A, None,
                                              ap.data_ptr() if ap is not None else None, None, L.current_stream()))


def test_categorical_act_equals_the_reference_sampler():
    """the fixture's probability vectors planted as logits log(p) (p = 0 as -inf is not representable: -1e30), then
    the recorded choices of the reference's Categorical under the same seeds"""
    from coach_b200 import _lib as L
    from oracle import a3c as oa
    lib = L.load()
    for k in range(int(G["n_cat"])):
        p = G["cat%d_p" % k]
        want = G["cat%d_train" % k]
        E, A = len(want), len(p)
        z = np.zeros((E, A + 1), np.float32)
        z[:, 1:] = np.where(p > 0, np.log(np.maximum(p, 1e-38)), -1e30)
        np.random.seed(int(G["cat%d_seed" % k]))
        u = np.random.random_sample(E)
        zt = torch.from_numpy(z).cuda()
        ut = torch.from_numpy(u).cuda()
        act = torch.zeros(E, dtype=torch.int64, device="cuda")
        probs = torch.zeros((E, A), device="cuda")
        L.check(lib.cb200_categorical_act(zt.data_ptr(), E, A, ut.data_ptr(), act.data_ptr(), probs.data_ptr(),
                                          L.current_stream()))
        pr = probs.cpu().numpy()
        got = act.cpu().numpy()
        assert got.tolist() == [oa.categorical_choice(pr[e], u[e]) for e in range(E)]
        np.testing.assert_allclose(pr[0], p, rtol=0, atol=2e-7)
        if np.array_equal(pr[0], p):                           # the softmax reproduced p exactly: the reference's draws
            assert got.tolist() == want.tolist(), k
        L.check(lib.cb200_categorical_act(zt.data_ptr(), E, A, None, act.data_ptr(), None, L.current_stream()))
        assert (act.cpu().numpy() == np.argmax(pr, axis=1)).all()


# ---- the agent --------------------------------------------------------------------------------------------------------
def _agent(obs, A, E=1, preset="cartpole", mode=None, t_max=None, seed=0, lr=None, huber=False):
    from coach_b200.agents.actor_critic_agent import ActorCriticAgent, PolicyGradientRescaler
    import copy
    if preset == "atari":
        from coach_b200.presets.Atari_A3C import agent_params
    else:
        from coach_b200.presets.CartPole_A3C import agent_params
    ap = copy.deepcopy(agent_params)
    if mode is not None:
        ap.algorithm.policy_gradient_rescaler = PolicyGradientRescaler.A_VALUE if mode == "A_VALUE" else \
            PolicyGradientRescaler.GAE
        ap.algorithm.estimate_state_value_using_gae = mode == "GAE_VALUE"
    if t_max is not None:
        ap.algorithm.num_steps_between_gradient_updates = t_max
    if lr is not None:
        ap.network_wrappers["main"].learning_rate = lr
    ap.network_wrappers["main"].replace_mse_with_huber_loss = huber
    return ActorCriticAgent(ap, observation_shape=obs, num_actions=A, num_envs=E, seed=seed)


def _stream(obs, A, E, steps, seed, p_end=0.15):
    rng = np.random.RandomState(seed)
    mk = (lambda n: rng.randint(0, 256, (n, E) + obs).astype(np.uint8)) if len(obs) == 3 else \
        (lambda n: rng.uniform(-1, 1, (n, E) + obs).astype(np.float32))
    s = mk(steps + 1)
    return dict(states=s[:-1], next_states=s[1:], actions=rng.randint(0, A, (steps, E)),
                rewards=rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], (steps, E)) / 200., dones=rng.rand(steps, E) < p_end)


def _oracle(agent, obs):
    from oracle import nets as on, nstep_q as oq
    nd = agent.net_def
    mk = lambda dt: oq.NStepQNetOracle(obs, agent.num_actions + 1, dt)                 # noqa: E731
    named = nd.store.export_named()
    p = agent.ap.network_wrappers["main"]
    opt32 = on.AdamTF([torch.from_numpy(v) for v in named.values()], p.learning_rate, 0.9, 0.99, 1e-4)
    opt64 = on.AdamTF([torch.from_numpy(v).double() for v in named.values()], p.learning_rate, 0.9, 0.99, 1e-4,
                      dtype=torch.float64)
    return mk(torch.float32), mk(torch.float64), opt32, opt64


def _run_and_check(agent, obs, st, steps):
    """drive observe_batch / train over the stream; at every learn step compare the loss and the new parameters with
    the fp32 / fp64 oracle (1e-5, else no farther from fp64 than twice the fp32 oracle).  Returns the learned
    (step, [(stream, rows)])."""
    from oracle import a3c as oa
    o32, o64, opt32, opt64 = _oracle(agent, obs)
    alg = agent.ap.algorithm
    mode = {0: "A_VALUE", 1: "GAE", 2: "GAE_VALUE"}[agent.mode]
    huber = agent.ap.network_wrappers["main"].replace_mse_with_huber_loss
    learned = []
    for t in range(steps):
        agent.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t], st["dones"][t])
        before = agent.net_def.store.export_named()
        loss = agent.train()
        if not agent.learned_segments:
            continue
        closed = [(e, end - start) for e, start, end in agent.learned_segments]
        learned.append((t, closed))
        segs = []
        for e, L in closed:
            ts = list(range(t - L + 1, t + 1))
            segs.append(dict(states=st["states"][ts, e], next_states=st["next_states"][ts, e],
                             actions=st["actions"][ts, e], rewards=st["rewards"][ts, e],
                             game_overs=st["dones"][ts, e].astype(np.uint8)))
        kw = dict(gae_lambda=alg.gae_lambda, beta=alg.beta_entropy, huber_loss=huber, clip=40.0)
        ref = oa.learn_step(o32, o32.cast(before), opt32, segs, alg.discount, mode, **kw)
        ref64 = oa.learn_step(o64, o64.cast(before), opt64, segs, alg.discount, mode, **kw)
        assert abs(loss - ref["loss"]) <= 1e-5 * max(1.0, abs(ref["loss"])) or \
            abs(loss - ref64["loss"]) <= 2 * abs(ref["loss"] - ref64["loss"]), (loss, ref["loss"], ref64["loss"])
        got = agent.net_def.store.export_named()
        for name in ref["new_params"]:
            want = ref["new_params"][name].numpy()
            try:
                close(got[name], want, name="param " + name)
            except AssertionError as exc:
                w64 = ref64["new_params"][name].numpy()
                e_ours, e_orc = np.abs(got[name] - w64).max(), np.abs(want - w64).max()
                assert e_ours <= 2 * e_orc, "%s; vs fp64: ours %.3e, fp32 oracle %.3e" % (exc, e_ours, e_orc)
    return learned


@pytest.mark.parametrize("preset,obs,A,steps", [("cartpole", (4,), 2, 31), ("atari", (84, 84, 4), 6, 45)],
                         ids=["cartpole", "atari"])
def test_one_stream_follows_the_reference_schedule_and_the_oracle(preset, obs, A, steps):
    from oracle import nstep_q as oq
    torch.manual_seed(0)
    agent = _agent(obs, A, E=1, preset=preset, seed=1)
    st = _stream(obs, A, 1, steps, seed=4, p_end=0.08)
    learned = _run_and_check(agent, obs, st, steps)
    assert len(learned) >= 3
    assert [(t, c) for t, c in learned] == [(t, c) for t, c in oq.lockstep_schedule(st["dones"], agent.t_max) if c]


@pytest.mark.parametrize("E,mode", [(16, "A_VALUE"), (16, "GAE"), (64, "GAE_VALUE"), (64, "A_VALUE")])
def test_many_streams_learn_the_segment_mean(E, mode):
    from oracle import nstep_q as oq
    torch.manual_seed(0)
    obs, A, steps = (4,), 2, 12
    agent = _agent(obs, A, E=E, mode=mode, seed=2, huber=E == 64)
    st = _stream(obs, A, E, steps, seed=5)
    learned = _run_and_check(agent, obs, st, steps)
    assert [(t, sorted(c)) for t, c in learned] == [(t, sorted(c)) for t, c in oq.lockstep_schedule(st["dones"], 5)
                                                     if c]


def test_graph_replay_is_bit_identical_to_eager(monkeypatch):
    obs, A, E, steps = (4,), 2, 60, 20          # every stream cuts at steps 5, 10, ...: 300 rows, a 320-row bucket

    def run(graph):
        monkeypatch.setenv("CB200_A3C_GRAPH", "1" if graph else "0")
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


@pytest.mark.parametrize("preset,obs,A", [("cartpole", (4,), 2), ("atari", (84, 84, 4), 6)])
def test_acting_matches_the_oracle_forward_and_np_random_choice(preset, obs, A):
    from oracle import a3c as oa, nstep_q as oq
    E = 16
    agent = _agent(obs, A, E=E, preset=preset, seed=4)
    rng = np.random.RandomState(0)
    x = rng.randint(0, 256, (E,) + obs).astype(np.uint8) if len(obs) == 3 else rng.randn(E, *obs).astype(np.float32)
    o = oq.NStepQNetOracle(obs, A + 1, torch.float64)
    z = o.forward(o.cast(agent.net_def.store.export_named()), x).numpy()
    p64 = np.exp(z[:, 1:] - z[:, 1:].max(1, keepdims=True))
    p64 /= p64.sum(1, keepdims=True)
    np.random.seed(11)
    actions, probs = agent.choose_actions(x)
    np.random.seed(11)
    u = np.random.random_sample(E)
    close(probs, p64, rtol=1e-5, name="probs")
    assert actions.tolist() == [oa.categorical_choice(probs[e], u[e]) for e in range(E)]
    if all(abs(float(np.sum(probs[e], dtype=np.float64)) - 1) <= 1e-4 for e in range(E)):
        np.random.seed(11)                                     # np.random.choice itself (it checks that p sums to 1)
        assert actions.tolist() == [int(np.random.choice(A, p=probs[e])) for e in range(E)]
    ev, pe = agent.choose_actions(x, evaluation=True)
    np.testing.assert_array_equal(pe, probs)
    assert (ev == np.argmax(probs, axis=1)).all()


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
