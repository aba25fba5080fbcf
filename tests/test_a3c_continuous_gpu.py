"""Actor-Critic (A3C) with continuous actions on the GPU: cb200_actor_critic_gaussian_head at the C ABI (the reference
fixture's targets and advantages bit for bit on whole episodes, random segment tables against an fp64 evaluation, an
exact dyadic probe, repeat-call, graph-replay and operand-plane bits, argument errors), cb200_gaussian_policy_act
against np.random.normal, and the agent (the fp32 / fp64 oracle at E = 1 on the inverted_pendulum and Humanoid shapes,
the segment mean at E = 16, graph replay against eager steps, checkpoint restore)."""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "a3c_continuous.npz")))
EPS32 = 2.0 ** -24
MODE = {"A_VALUE": 0, "GAE": 1, "GAE_VALUE": 2}
LOG_2PI = np.log(2 * np.pi)


def close(got, want, rtol=1e-5, name="", atol=0.0):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    err = np.abs(got - want).max() if got.size else 0.0
    tol = rtol * np.abs(want).max() + atol
    assert err <= tol, "%s: max abs err %.3e > %.3e" % (name, err, tol)


# ---- the head at the C ABI --------------------------------------------------------------------------------------------
def head(h, hb, w, b, actions, rng_, rewards, dones, offsets, lengths, discount, mode, lam=0.96, beta=0.01, huber=0,
         rows=None, planes=False, p_weight=1.0):
    """one cb200_actor_critic_gaussian_head call on host arrays; returns every output as numpy"""
    from coach_b200 import _lib as L
    lib, dev = L.load(), "cuda"
    rows = rows or h.shape[0]
    K, N, S = h.shape[1], w.shape[1], len(offsets)
    D = (N - 1) // 2
    T = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x, dtype=dt)).to(dev)       # noqa: E731
    t = dict(h=T(h, np.float32), hb=T(hb, np.float32), w=T(w, np.float32), b=T(b, np.float32),
             x=T(np.asarray(actions).reshape(rows, D), np.float32), rg=T(rng_, np.float32),
             r=T(rewards, np.float64), d=T(dones, np.uint8), off=T(offsets, np.int32), len=T(lengths, np.int32))
    out = {k: torch.full(s, float("nan"), dtype=torch.float32, device=dev) for k, s in
           (("z", (rows, N)), ("dz", (rows, N)), ("loss", (1,)), ("means", (rows, D)), ("stds", (rows, D)),
            ("targets", (rows,)), ("adv", (rows,)), ("boot", (S,)), ("dh", (rows, K)), ("dw", (K, N)), ("db", (N,)))}
    ws = torch.full((L.acg_workspace_floats(rows, S, K, D),), float("nan"), device=dev)
    d = L.ActorCriticGaussianHeadDesc()
    d.h, d.h_boot, d.w, d.b = (t[k].data_ptr() for k in ("h", "hb", "w", "b"))
    d.actions, d.max_abs_range = t["x"].data_ptr(), t["rg"].data_ptr()
    d.rewards, d.game_overs = t["r"].data_ptr(), t["d"].data_ptr()
    d.seg_offsets, d.seg_lengths, d.segments, d.rows = t["off"].data_ptr(), t["len"].data_ptr(), S, rows
    d.discount, d.gae_lambda, d.mode, d.huber = discount, lam, mode, huber
    d.beta_entropy, d.v_weight, d.p_weight, d.features, d.action_dim = beta, 0.5, p_weight, K, D
    d.z, d.dz, d.loss, d.means, d.stds = (out[k].data_ptr() for k in ("z", "dz", "loss", "means", "stds"))
    d.targets, d.advantages, d.bootstrap = (out[k].data_ptr() for k in ("targets", "adv", "boot"))
    d.dh, d.dw, d.db = (out[k].data_ptr() for k in ("dh", "dw", "db"))
    d.workspace = ws.data_ptr()
    pl = None
    if planes:
        pl = torch.zeros(3 * rows * K, dtype=torch.int16, device=dev)
        d.dh_planes, d.dh_plane_stride = pl.data_ptr(), rows * K
    L.check(lib.cb200_actor_critic_gaussian_head(ctypes.byref(d), L.current_stream()))
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    res["_desc"], res["_keep"] = d, (t, out, ws, pl)
    return res


@pytest.mark.parametrize("mode", list(MODE))
@pytest.mark.parametrize("K", [256, 512])
def test_fixture_targets_and_advantages_bit_for_bit(mode, K):
    """V planted exactly: h = [V | 0], W = e_0 (column 0); whole episodes of 1 to 1000 rows"""
    for c in range(int(G["n_cases"])):
        v, boot, r = G["c%d_values" % c], G["c%d_boot" % c], G["c%d_rewards" % c]
        d, disc, lam = G["c%d_game_overs" % c], float(G["c%d_discount" % c]), float(G["c%d_lambda" % c])
        D, L = int(G["c%d_dim" % c]), len(v)
        h = np.zeros((L, K), np.float32)
        h[:, 0] = v
        hb = np.zeros((1, K), np.float32)
        hb[0, 0] = boot
        w = np.zeros((K, 1 + 2 * D), np.float32)
        w[0, 0] = 1
        o = head(h, hb, w, np.zeros(1 + 2 * D, np.float32), G["c%d_fed_actions" % c], np.ones(D), r, d, [0], [L],
                 disc, MODE[mode], lam)
        np.testing.assert_array_equal(o["z"][:, 0], v)
        for key, got in (("targets", o["targets"]), ("advantages", o["adv"])):
            want = G["c%d_%s_%s" % (c, mode.lower(), key)].astype(np.float32)
            np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32), err_msg="case %d %s" % (c, key))
        assert o["boot"][0] == (0.0 if d[-1] else boot)
        np.testing.assert_array_equal(o["means"], np.zeros((L, D), np.float32))


def _random(rng, S, K, D, maxlen=1000, pad=0):
    lengths = np.minimum(rng.randint(1, maxlen + 1, S), maxlen)
    lengths[0] = maxlen if maxlen >= 1000 else lengths[0]
    n = int(lengths.sum())
    rows = n + pad
    h = np.maximum(rng.randn(rows, K), 0).astype(np.float32)
    hb = np.maximum(rng.randn(S, K), 0).astype(np.float32)
    w = (rng.randn(K, 1 + 2 * D) * 0.05).astype(np.float32)
    b = (rng.randn(1 + 2 * D) * 0.1).astype(np.float32)
    rg = (rng.rand(D) * 3 + 0.5).astype(np.float32)
    actions = (rng.randn(rows, D) * rg).astype(np.float32)
    rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], rows) / 20.
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int32)
    dones = np.zeros(rows, dtype=np.uint8)
    dones[(offsets + lengths - 1)[rng.rand(S) < 0.6]] = 1
    perm = rng.permutation(S)                                  # the table's slot order is free
    return h, hb, w, b, actions, rg, rewards, dones, offsets[perm], lengths[perm], rows


def _softplus_tf(x):
    t = float(np.log(np.float32(EPS32 * 2)) + np.float32(2))
    return np.where(x > -t, x, np.where(x < t, np.exp(x), np.log(np.exp(x) + 1)))


def _fp64_check(args, o, discount, mode, lam, beta, huber):
    from oracle import a3c as oa
    h, hb, w, b, actions, rg, rewards, dones, offsets, lengths, rows = args
    h64, w64 = h.astype(np.float64), w.astype(np.float64)
    z64 = h64 @ w64 + b
    S, N = len(offsets), w.shape[1]
    D = (N - 1) // 2
    n = int(lengths.sum())
    zb = (h.shape[1] + 2) * EPS32 * (np.abs(h64) @ np.abs(w64) + np.abs(b))
    assert (np.abs(o["z"][:n] - z64[:n]) <= zb[:n]).all()
    dz64 = np.zeros((rows, N))
    dzb = np.zeros((rows, 1))
    loss64 = labs = 0.0
    zk = o["z"].astype(np.float64)                             # the loss and dL/dZ in fp64 on the kernel's own outputs
    for s in range(S):
        o0, L = int(offsets[s]), int(lengths[s])
        sl = slice(o0, o0 + L)
        t, a = oa.segment_targets(o["z"][sl, 0], o["boot"][s], rewards[sl], dones[sl], discount, mode, lam)
        np.testing.assert_array_equal(o["targets"][sl], t.astype(np.float32))
        np.testing.assert_array_equal(o["adv"][sl], a.astype(np.float32))
        t, a = t.astype(np.float32).astype(np.float64), a.astype(np.float32).astype(np.float64)
        v, zm, zs = zk[sl, 0], zk[sl, 1:1 + D], zk[sl, 1 + D:]
        th = np.tanh(zm)
        mu = th * rg
        sd = _softplus_tf(zs) + EPS32 * 2
        x = actions[sl].astype(np.float64)
        diff = x - mu
        logp = (-0.5 * (diff / sd) ** 2 - np.log(sd) - 0.5 * LOG_2PI).sum(1)
        H = (0.5 * (1 + LOG_2PI) + np.log(sd)).sum(1)
        e = v - t
        if huber:
            lv, gv = np.where(np.abs(e) <= 1, 0.5 * e * e, np.abs(e) - 0.5), np.clip(e, -1, 1)
        else:
            lv, gv = e * e, 2 * e
        loss64 += (0.5 * lv.mean() - (logp * a).mean() - beta * H.mean()) / S
        labs += (0.5 * lv.mean() + np.abs(logp * a).mean() + beta * np.abs(H).mean()) / S
        c = 1.0 / (S * L)
        cp = -c * a[:, None]
        sig = 1 / (1 + np.exp(-zs))
        dz64[sl, 0] = c * 0.5 * gv
        dz64[sl, 1:1 + D] = cp * diff / sd ** 2 * rg * (1 - th ** 2)
        dz64[sl, 1 + D:] = (cp * (diff ** 2 / sd ** 3 - 1 / sd) - c * beta / sd) * sig
        # fp32 transcendentals and divisions per row: within 2^-14 of the row's gradient scale
        scale = c * (0.5 * np.abs(gv) + (np.abs(a)[:, None] * (np.abs(diff) / sd ** 2 * rg + diff ** 2 / sd ** 3 +
                                                                 1 / sd) + beta / sd).sum(1))
        dzb[sl, 0] = 2.0 ** -14 * scale
        np.testing.assert_allclose(o["means"][sl], mu, rtol=0, atol=2e-6 * rg.max())
        np.testing.assert_allclose(o["stds"][sl], sd, rtol=2e-6, atol=1.2e-7)
    assert not o["targets"][n:].any() and not o["dz"][n:].any() and not o["z"][n:].any()
    dw64, db64 = h64.T @ dz64, dz64.sum(0)
    dh64 = (dz64 @ w64.T) * (h > 0)
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


@pytest.mark.parametrize("seed", range(8))
def test_random_segment_tables_against_fp64(seed):
    rng = np.random.RandomState(seed)
    S = [1, 3, 17, 64, 40, 8, 2, 64][seed]
    K = [256, 512][seed % 2]
    D = [1, 3, 6, 17][seed % 4]
    maxlen = [1000, 300, 60, 20, 50, 1000, 1000, 5][seed]
    mode = list(MODE)[seed % 3]
    huber, lam, beta = seed % 2, [1.0, 0.96][seed % 2], [1e-4, 0.05, 0.0][seed % 3]
    args = _random(rng, S, K, D, maxlen, pad=[0, 5, 31, 7, 0, 19, 64, 3][seed])
    o = head(*args[:10], 0.99, MODE[mode], lam, beta, huber, rows=args[10])
    _fp64_check(args, o, 0.99, mode, lam, beta, huber)
    assert np.isfinite(o["dh"]).all() and not o["dh"][int(args[9].sum()):].any()


def test_dyadic_probe_is_exact():
    """no policy or entropy weight (their dL/dZ are exactly zero), small-integer features, dyadic weights, segment
    lengths and counts powers of two: V, dL/dV, dW, db and dh are exact in fp32 and equal the fp64 evaluation"""
    rng = np.random.RandomState(7)
    K, S, D = 256, 4, 3
    lengths = np.array([1, 2, 4, 1])
    rows = 8
    h = rng.randint(0, 4, (rows, K)).astype(np.float32)
    w = (rng.randint(-4, 5, (K, 1 + 2 * D)) / 64.0).astype(np.float32)
    b = np.zeros(1 + 2 * D, np.float32)
    rewards = rng.randint(-2, 3, rows).astype(np.float64)
    offsets = np.array([0, 1, 3, 7], np.int32)
    dones = np.ones(rows, np.uint8)
    o = head(h, h[:S], w, b, rng.randn(rows, D), np.ones(D), rewards, dones, offsets, lengths, 0.5, MODE["A_VALUE"],
             beta=0.0, p_weight=0.0)
    z = h.astype(np.float64) @ w
    np.testing.assert_array_equal(o["z"], z)
    dz = np.zeros((rows, 1 + 2 * D))
    for s in range(S):
        for i in range(offsets[s], offsets[s] + lengths[s]):
            dz[i, 0] = (z[i, 0] - np.float64(o["targets"][i])) / (S * lengths[s])
    np.testing.assert_array_equal(o["dz"], dz)
    np.testing.assert_array_equal(o["dw"], h.astype(np.float64).T @ dz)
    np.testing.assert_array_equal(o["db"], dz.sum(0))
    np.testing.assert_array_equal(o["dh"], (dz @ w.astype(np.float64).T) * (h > 0))


def test_repeat_calls_graph_replay_and_planes_give_identical_bits():
    rng = np.random.RandomState(3)
    args = _random(rng, 33, 512, 17, 200, pad=9)
    args = args[:10] + (args[10] + (-args[10]) % 8,)
    a = head(*args[:10], 0.99, 1, 0.96, 0.01, 1, rows=args[10])
    b = head(*args[:10], 0.99, 1, 0.96, 0.01, 1, rows=args[10], planes=True)
    keys = ("z", "dz", "loss", "means", "stds", "targets", "adv", "boot", "dh", "dw", "db")
    for k in keys:
        np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32), err_msg=k)
    t, out, ws, pl = b["_keep"]
    from coach_b200 import _lib as L
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L.check(L.load().cb200_actor_critic_gaussian_head(ctypes.byref(b["_desc"]), L.current_stream()))
    for v in out.values():
        v.fill_(float("nan"))
    ws.fill_(float("nan"))
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


def test_optional_outputs_may_be_omitted():
    """targets, advantages, bootstrap, dz, means and stds NULL: the workspace holds them; same loss and gradients"""
    from coach_b200 import _lib as L
    rng = np.random.RandomState(4)
    args = _random(rng, 5, 256, 3, 40)
    a = head(*args[:10], 0.99, 2, rows=args[10])
    d = a["_desc"]
    t, out, ws, pl = a["_keep"]
    for f in ("targets", "advantages", "bootstrap", "dz", "means", "stds", "loss"):
        setattr(d, f, None)
    for k in ("dw", "db", "dh"):
        out[k].fill_(float("nan"))
    L.check(L.load().cb200_actor_critic_gaussian_head(ctypes.byref(d), L.current_stream()))
    torch.cuda.synchronize()
    for k in ("dw", "db", "dh"):
        np.testing.assert_array_equal(out[k].cpu().numpy().view(np.uint32), a[k].view(np.uint32), err_msg=k)


def test_argument_errors():
    from coach_b200 import _lib as L
    lib = L.load()
    rng = np.random.RandomState(1)
    args = _random(rng, 2, 256, 6, 30)
    o = head(*args[:10], 0.99, 0, rows=args[10])
    d = o["_desc"]
    call = lambda: L.check(lib.cb200_actor_critic_gaussian_head(ctypes.byref(d), L.current_stream()))   # noqa: E731
    for field, bad in (("action_dim", 18), ("action_dim", 0), ("features", 128), ("mode", 3), ("mode", -1),
                       ("segments", 0), ("rows", 0), ("h", None), ("h_boot", None), ("workspace", None),
                       ("seg_lengths", None), ("z", None), ("actions", None), ("max_abs_range", None)):
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
    z = torch.zeros((4, 7), device="cuda")
    rg = torch.ones(3, device="cuda")
    act = torch.zeros((4, 3), dtype=torch.float64, device="cuda")
    for envs, D, zp, rp, ap in ((0, 3, z, rg, act), (4, 0, z, rg, act), (4, 18, z, rg, act), (4, 3, None, rg, act),
                                (4, 3, z, None, act), (4, 3, z, rg, None)):
        ptr = lambda x: x.data_ptr() if x is not None else None          # noqa: E731
        with pytest.raises(ValueError):
            L.check(lib.cb200_gaussian_policy_act(ptr(zp), envs, D, ptr(rp), None, ptr(ap), None, None,
                                                  L.current_stream()))


@pytest.mark.parametrize("E,D", [(1, 1), (8, 1), (16, 3), (64, 17)])
def test_gaussian_act_equals_np_random_normal(E, D):
    from coach_b200 import _lib as L
    lib = L.load()
    rng = np.random.RandomState(E + D)
    z = (rng.randn(E, 1 + 2 * D) * 3).astype(np.float32)
    z[0, 1 + D] = -40.0                                        # softplus's exp(x) region
    z[-1, -1] = 30.0                                           # and its identity region
    rg = (rng.rand(D) * 3 + 0.5).astype(np.float32)
    zt, rt = torch.from_numpy(z).cuda(), torch.from_numpy(rg).cuda()
    act = torch.zeros((E, D), dtype=torch.float64, device="cuda")
    means = torch.zeros((E, D), device="cuda")
    stds = torch.zeros((E, D), device="cuda")
    np.random.seed(5)
    n = torch.from_numpy(np.random.standard_normal((E, D))).cuda()
    L.check(lib.cb200_gaussian_policy_act(zt.data_ptr(), E, D, rt.data_ptr(), n.data_ptr(), act.data_ptr(),
                                          means.data_ptr(), stds.data_ptr(), L.current_stream()))
    m, s = means.cpu().numpy(), stds.cpu().numpy()
    np.random.seed(5)
    want = np.array([np.random.normal(m[e], s[e]) for e in range(E)]).reshape(E, D)    # E successive reference calls
    np.testing.assert_array_equal(act.cpu().numpy().view(np.uint64), want.view(np.uint64))
    zd = z.astype(np.float64)
    np.testing.assert_allclose(m, np.tanh(zd[:, 1:1 + D]) * rg, rtol=0, atol=2e-6 * rg.max())
    # log(exp(x) + 1) in fp32 rounds exp(x) + 1 to 2^-24: an absolute error on small stds
    np.testing.assert_allclose(s, _softplus_tf(zd[:, 1 + D:]) + EPS32 * 2, rtol=2e-6, atol=1.2e-7)
    L.check(lib.cb200_gaussian_policy_act(zt.data_ptr(), E, D, rt.data_ptr(), None, act.data_ptr(), None, None,
                                          L.current_stream()))
    np.testing.assert_array_equal(act.cpu().numpy(), m.astype(np.float64))


# ---- the agent --------------------------------------------------------------------------------------------------------
def _agent(obs, D, E=1, mode=None, seed=0, lr=None, huber=False, max_episode_steps=1000):
    from coach_b200.agents.actor_critic_agent import ActorCriticAgent, PolicyGradientRescaler
    from coach_b200.presets.Mujoco_A3C import agent_params
    ap = copy.deepcopy(agent_params)
    if mode is not None:
        ap.algorithm.policy_gradient_rescaler = PolicyGradientRescaler.A_VALUE if mode == "A_VALUE" else \
            PolicyGradientRescaler.GAE
        ap.algorithm.estimate_state_value_using_gae = mode == "GAE_VALUE"
    if lr is not None:
        ap.network_wrappers["main"].learning_rate = lr
    ap.network_wrappers["main"].replace_mse_with_huber_loss = huber
    high = np.full(D, 3.0 if D == 1 else 0.4, np.float32)
    return ActorCriticAgent(ap, observation_shape=obs, action_dim=D, action_low=-high, action_high=high, num_envs=E,
                            seed=seed, max_episode_steps=max_episode_steps)


def _stream(obs, D, E, steps, seed, p_end=0.05, every=None):
    rng = np.random.RandomState(seed)
    s = rng.uniform(-1, 1, (steps + 1, E) + obs).astype(np.float32)
    dones = rng.rand(steps, E) < p_end
    if every is not None:
        dones = np.zeros((steps, E), bool)
        dones[every - 1::every] = True
    return dict(states=s[:-1], next_states=s[1:], actions=rng.randn(steps, E, D) * 0.7,
                rewards=rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], (steps, E)) / 20., dones=dones)


def _run_and_check(agent, obs, st, steps):
    """drive observe_batch / train over the stream; at every learn step compare the loss and the new parameters with
    the fp32 / fp64 oracle (1e-5, else no farther from fp64 than twice the fp32 oracle).  Returns the learned
    (step, [(stream, rows)])."""
    from oracle import a3c_continuous as oc, nets as on, nstep_q as oq
    N = 1 + 2 * agent.action_dim
    o32, o64 = oq.NStepQNetOracle(obs, N, torch.float32), oq.NStepQNetOracle(obs, N, torch.float64)
    named = agent.net_def.store.export_named()
    p = agent.ap.network_wrappers["main"]
    opt32 = on.AdamTF([torch.from_numpy(v) for v in named.values()], p.learning_rate, 0.9, 0.99, 1e-4)
    opt64 = on.AdamTF([torch.from_numpy(v).double() for v in named.values()], p.learning_rate, 0.9, 0.99, 1e-4,
                      dtype=torch.float64)
    alg = agent.ap.algorithm
    mode = {0: "A_VALUE", 1: "GAE", 2: "GAE_VALUE"}[agent.mode]
    rng = agent.max_abs_range.cpu().numpy()
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
        kw = dict(gae_lambda=alg.gae_lambda, beta=alg.beta_entropy,
                  huber_loss=p.replace_mse_with_huber_loss, clip=40.0)
        ref = oc.learn_step(o32, o32.cast(before), opt32, segs, alg.discount, mode, rng, **kw)
        ref64 = oc.learn_step(o64, o64.cast(before), opt64, segs, alg.discount, mode, rng, **kw)
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


@pytest.mark.parametrize("obs,D,mode,steps", [((4,), 1, None, 120), ((376,), 17, "GAE", 90)],
                         ids=["inverted_pendulum", "humanoid"])
def test_one_stream_learns_whole_episodes_like_the_oracle(obs, D, mode, steps):
    from oracle import nstep_q as oq
    torch.manual_seed(0)
    agent = _agent(obs, D, E=1, mode=mode, seed=1, lr=1e-3)
    st = _stream(obs, D, 1, steps, seed=4, p_end=0.06)
    learned = _run_and_check(agent, obs, st, steps)
    assert len(learned) >= 3
    # whole episodes: the cut falls at the episodes' ends only (t_max is 10^7)
    assert [(t, c) for t, c in learned] == [(t, c) for t, c in oq.lockstep_schedule(st["dones"], agent.t_max) if c]


@pytest.mark.parametrize("mode", ["A_VALUE", "GAE_VALUE"])
def test_sixteen_streams_learn_the_segment_mean(mode):
    torch.manual_seed(0)
    obs, D, E, steps = (11,), 3, 16, 40
    agent = _agent(obs, D, E=E, mode=mode, seed=2, lr=1e-3, huber=mode == "GAE_VALUE")
    st = _stream(obs, D, E, steps, seed=5, p_end=0.08)
    learned = _run_and_check(agent, obs, st, steps)
    assert sum(len(c) for _, c in learned) >= 16 and max(len(c) for _, c in learned) >= 2


def test_an_episode_overrunning_max_episode_steps_is_refused():
    obs, D = (4,), 1
    agent = _agent(obs, D, E=2, max_episode_steps=6)
    st = _stream(obs, D, 2, 8, seed=1, p_end=0.0)
    for t in range(6):
        agent.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t], st["dones"][t])
        assert agent.train() == 0
    with pytest.raises(ValueError, match="max_episode_steps"):
        agent.observe_batch(st["states"][6], st["actions"][6], st["rewards"][6], st["next_states"][6], st["dones"][6])


def test_graph_replay_is_bit_identical_to_eager(monkeypatch):
    obs, D, E, steps = (11,), 3, 64, 50          # every stream's episode ends every 10 steps: 640-row buckets

    def run(graph):
        monkeypatch.setenv("CB200_A3C_GRAPH", "1" if graph else "0")
        a = _agent(obs, D, E=E, seed=3, lr=1e-3)
        st = _stream(obs, D, E, steps, seed=6, every=10)
        losses = []
        for t in range(steps):
            a.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t], st["dones"][t])
            losses.append(a.train())
        return a, losses
    g, lg = run(True)
    e, le = run(False)
    assert g.graph_kernel_launches > 0 and e.graph_kernel_launches == 0
    assert lg == le and sum(1 for x in lg if x != 0) == 5
    assert torch.equal(g.net_def.store.theta, e.net_def.store.theta)


def test_acting_and_the_noise_schedule():
    from oracle import a3c_continuous as oc, nstep_q as oq
    from coach_b200.schedules import LinearSchedule
    obs, D, E = (376,), 17, 16
    agent = _agent(obs, D, E=E, seed=4)
    agent.noise_schedule = LinearSchedule(0.5, 0.1, 100)
    x = np.random.RandomState(0).randn(E, *obs).astype(np.float32)
    o = oq.NStepQNetOracle(obs, 1 + 2 * D, torch.float64)
    z = o.forward(o.cast(agent.net_def.store.export_named()), x)
    _, m64, s64, _, _ = oc.gaussian_terms(z, np.zeros((E, D)), agent.max_abs_range.cpu().numpy())
    np.random.seed(11)
    actions, means, stds = agent.choose_actions(x)
    close(means, m64.numpy(), rtol=1e-5, name="means")
    close(stds, s64.numpy(), rtol=1e-5, name="stds")
    np.random.seed(11)
    want = np.array([np.random.normal(means[e], stds[e]) for e in range(E)])
    np.testing.assert_array_equal(actions.view(np.uint64), want.view(np.uint64))
    assert abs(agent.noise_schedule.current_value - (0.5 - E * 0.4 / 100)) < 1e-12
    ev, me, se = agent.choose_actions(x, evaluation=True)
    assert ev.dtype == np.float32
    np.testing.assert_array_equal(ev, means)
    np.testing.assert_array_equal(se, stds)
    assert abs(agent.noise_schedule.current_value - (0.5 - E * 0.4 / 100)) < 1e-12
    assert agent.get_prediction(x).shape == (E, 1 + 2 * D)


def test_checkpoint_restore_continues_identically(tmp_path):
    from coach_b200 import checkpoint
    from coach_b200.schedules import LinearSchedule
    obs, D, E, steps = (4,), 1, 1, 40
    st = _stream(obs, D, E, 2 * steps, seed=8, every=8)
    a = _agent(obs, D, E=E, seed=5, lr=1e-3)
    a.noise_schedule = LinearSchedule(0.5, 0.1, 1000)

    def run(agent, lo, hi):
        out = []
        for t in range(lo, hi):
            agent.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t],
                                st["dones"][t])
            out.append(agent.train())
        return out
    run(a, 0, steps)                                           # 40 steps, episodes of 8: the last step closed one
    a.choose_actions(st["states"][0])
    name = checkpoint.save_checkpoint(a, str(tmp_path), checkpoint_id=1)
    want = run(a, steps, 2 * steps)
    b = _agent(obs, D, E=E, seed=9, lr=1e-3)
    b.noise_schedule = LinearSchedule(0.5, 0.1, 1000)
    checkpoint.restore_checkpoint(b, str(tmp_path), name)
    assert b.noise_schedule.current_value == 0.5 - 0.4 / 1000
    got = run(b, steps, 2 * steps)
    assert got == want
    assert torch.equal(b.net_def.store.theta, a.net_def.store.theta)
    assert b.training_iteration == a.training_iteration
