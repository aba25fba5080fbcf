"""Policy Gradients (REINFORCE) on the GPU: cb200_pg_targets against the reference fixture bit for bit (every rescaler
and length, numpy's pairwise mean / std, the timestep table's snapshots for several episodes closing at one lock-step),
cb200_policy_gradient_head against fp64 on random tables (discrete and continuous), repeat-call / graph-replay / plane
bits and argument errors, cb200_policy_act against numpy's draws, and the agent (the torch oracle at E = 1 across apply
boundaries, E = 16 against a sequential run of the same episodes, checkpoint restore mid-accumulation)."""
import copy
import ctypes
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

G = dict(np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "pg.npz")))
EPS32 = 2.0 ** -24
RESC = {"TOTAL_RETURN": 0, "FUTURE_RETURN": 1, "FUTURE_RETURN_NORMALIZED_BY_EPISODE": 2,
        "FUTURE_RETURN_NORMALIZED_BY_TIMESTEP": 3}


def T(x, dt):
    return torch.as_tensor(np.ascontiguousarray(x, dtype=dt)).cuda()


def lib():
    from coach_b200 import _lib as L
    return L, L.load()


# ---- targets ----------------------------------------------------------------------------------------------------------
def targets(rewards_list, discount, rescaler, table=None, perm=None, rows=None):
    """cb200_nstep_returns + cb200_pg_targets over episodes laid out one after the other (slot order = ``perm`` of the
    episodes, default in order); returns (targets, returns, baselines, stats, table)"""
    L_, lb = lib()
    lengths = np.array([len(r) for r in rewards_list])
    n = int(lengths.sum())
    rows = rows or n
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    r = np.zeros(rows)
    r[:n] = np.concatenate(rewards_list).astype(np.float64)
    st = np.arange(rows, dtype=np.int64)
    en = st + 1
    st[:n] = np.repeat(offsets, lengths)
    en[:n] = np.repeat(offsets + lengths, lengths)
    perm = np.arange(len(lengths)) if perm is None else np.asarray(perm)
    t = dict(r=T(r, np.float64), st=T(st, np.int64), en=T(en, np.int64), off=T(offsets[perm], np.int32),
             len=T(lengths[perm], np.int32))
    ret = torch.zeros(rows, dtype=torch.float64, device="cuda")
    tg = torch.full((rows,), float("nan"), device="cuda")
    base = torch.full((rows,), float("nan"), dtype=torch.float64, device="cuda")
    stats = torch.full((len(lengths), 2), float("nan"), dtype=torch.float64, device="cuda")
    tab = T(table if table is not None else np.zeros((2, 1000)), np.float64)
    L_.check(lb.cb200_nstep_returns(t["r"].data_ptr(), t["st"].data_ptr(), t["en"].data_ptr(), rows, discount, -1,
                                    ret.data_ptr(), L_.current_stream()))
    L_.check(lb.cb200_pg_targets(ret.data_ptr(), t["off"].data_ptr(), t["len"].data_ptr(), len(lengths), rows,
                                 rescaler, tab[0].data_ptr(), tab[1].data_ptr(), tab.shape[1], tg.data_ptr(),
                                 base.data_ptr(), stats.data_ptr(), L_.current_stream()))
    torch.cuda.synchronize()
    return (tg.cpu().numpy(), ret.cpu().numpy(), base.cpu().numpy(), stats.cpu().numpy()[np.argsort(perm)],
            tab.cpu().numpy())


@pytest.mark.parametrize("name", list(RESC))
def test_targets_equal_the_fixture_bit_for_bit(name):
    for c in range(int(G["n_cases"])):
        r, disc = G["c%d_rewards" % c], float(G["c%d_discount" % c])
        tg, ret, _, stats, _ = targets([r], disc, RESC[name])
        np.testing.assert_array_equal(ret.view(np.uint64), G["c%d_returns" % c].view(np.uint64))
        want = G["c%d_%s" % (c, name.lower())].astype(np.float32)
        np.testing.assert_array_equal(tg.view(np.uint32), want.view(np.uint32), err_msg="case %d" % c)
        if name == "FUTURE_RETURN_NORMALIZED_BY_EPISODE":
            R = G["c%d_returns" % c]
            np.testing.assert_array_equal(stats[0], [np.mean(R), np.std(R)])


def test_timestep_table_snapshots_for_episodes_closing_together():
    """the fixture's 12-episode sequence in three calls of 4, 5 and 3 episodes: the table after each call equals the
    reference's table sequence, every row's baseline the oracle's snapshot right after its own episode, and every
    target the reference's"""
    from oracle import pg as op
    table, orc = np.zeros((2, 1000)), op.TimestepTable(1000)
    k = 0
    for size in (4, 5, 3):
        eps = [G["seq%d_rewards" % (k + j)] for j in range(size)]
        tg, ret, base, _, table = targets(eps, 0.99, RESC["FUTURE_RETURN_NORMALIZED_BY_TIMESTEP"], table)
        off = 0
        for j, r in enumerate(eps):
            L = len(r)
            R = op.episode_returns(r, 0.99)
            snap = orc.fold(R)
            np.testing.assert_array_equal(base[off:off + L].view(np.uint64), snap.view(np.uint64))
            np.testing.assert_array_equal(tg[off:off + L], (R - snap).astype(np.float32))
            want = G["seq%d_targets" % (k + j)].astype(np.float32)      # what the reference handed to the network
            np.testing.assert_array_equal(tg[off:off + L].view(np.uint32), want.view(np.uint32))
            off += L
        k += size
        n = len(G["seq%d_mean_table" % (k - 1)])
        np.testing.assert_array_equal(table[0, :n].view(np.uint64), G["seq%d_mean_table" % (k - 1)].view(np.uint64))
        np.testing.assert_array_equal(table[1, :n], G["seq%d_count_table" % (k - 1)])


def test_slot_order_is_the_fold_order():
    from oracle import pg as op
    rng = np.random.RandomState(3)
    eps = [rng.choice([0.0, 1.0, 0.37], L) for L in (5, 9, 3)]
    perm = [2, 0, 1]                                           # slot s holds episode perm[s]
    _, _, base, _, _ = targets(eps, 0.99, 3, perm=perm)
    orc = op.TimestepTable(1000)
    offsets = np.concatenate([[0], np.cumsum([len(e) for e in eps])[:-1]])
    for e in perm:
        snap = orc.fold(op.episode_returns(eps[e], 0.99))
        np.testing.assert_array_equal(base[offsets[e]:offsets[e] + len(eps[e])], snap)


# ---- the head ---------------------------------------------------------------------------------------------------------
def head(h, w, b, tg, actions, offsets, lengths, continuous, rng_=None, beta=0.0, rows=None, planes=False):
    L_, lb = lib()
    rows = rows or h.shape[0]
    K, N, S = h.shape[1], w.shape[1], len(offsets)
    t = dict(h=T(h, np.float32), w=T(w, np.float32), b=T(b, np.float32), tg=T(tg, np.float32),
             off=T(offsets, np.int32), len=T(lengths, np.int32))
    t["a"] = T(actions, np.float32 if continuous else np.int64)
    if continuous:
        t["rg"] = T(rng_, np.float32)
    out = {k: torch.full(s, float("nan"), device="cuda") for k, s in
           (("z", (rows, N)), ("pol", (rows, N)), ("dz", (rows, N)), ("loss", (1,)), ("dh", (rows, K)),
            ("dw", (K, N)), ("db", (N,)))}
    ws = torch.full((rows * (N + 1) + (rows + 63) // 64 * (K * N + N + 1),), float("nan"), device="cuda")
    d = L_.PolicyGradientHeadDesc()
    d.h, d.w, d.b, d.targets = (t[k].data_ptr() for k in ("h", "w", "b", "tg"))
    if continuous:
        d.cont_actions, d.max_abs_range = t["a"].data_ptr(), t["rg"].data_ptr()
    else:
        d.actions = t["a"].data_ptr()
    d.seg_offsets, d.seg_lengths, d.segments, d.rows = t["off"].data_ptr(), t["len"].data_ptr(), S, rows
    d.continuous, d.features, d.n_outputs, d.beta_entropy = int(continuous), K, N, beta
    d.z, d.policy, d.dz, d.loss = (out[k].data_ptr() for k in ("z", "pol", "dz", "loss"))
    d.dh, d.dw, d.db, d.workspace = out["dh"].data_ptr(), out["dw"].data_ptr(), out["db"].data_ptr(), ws.data_ptr()
    pl = None
    if planes:
        pl = torch.zeros(3 * rows * K, dtype=torch.int16, device="cuda")
        d.dh_planes, d.dh_plane_stride = pl.data_ptr(), rows * K
    L_.check(lb.cb200_policy_gradient_head(ctypes.byref(d), L_.current_stream()))
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items()}
    res["_desc"], res["_keep"] = d, (t, out, ws, pl)
    return res


def _random(rng, S, K, N, continuous, maxlen=300, pad=0):
    lengths = rng.randint(1, maxlen + 1, S)
    n = int(lengths.sum())
    rows = n + pad
    h = np.maximum(rng.randn(rows, K), 0).astype(np.float32)
    w = (rng.randn(K, N) * 0.05).astype(np.float32)
    b = (rng.randn(N) * 0.1).astype(np.float32)
    tg = (rng.randn(rows) * 2).astype(np.float32)
    actions = rng.uniform(-3, 3, (rows, N)).astype(np.float32) if continuous else rng.randint(0, N, rows)
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int32)
    perm = rng.permutation(S)
    rg = np.full(N, 3.0, np.float32) if continuous else None
    return h, w, b, tg, actions, offsets[perm], lengths[perm], rows, rg


def _fp64_check(args, o, continuous, beta):
    h, w, b, tg, actions, offsets, lengths, rows, rg = args
    h64, w64 = h.astype(np.float64), w.astype(np.float64)
    z64 = h64 @ w64 + b
    N, n = w.shape[1], int(lengths.sum())
    zb = (h.shape[1] + 2) * EPS32 * (np.abs(h64) @ np.abs(w64) + np.abs(b))
    assert (np.abs(o["z"][:n] - z64[:n]) <= zb[:n]).all()
    zk = o["z"].astype(np.float64)                             # the loss and dL/dZ in fp64 on the kernel's own outputs
    dz64, dzb = np.zeros((rows, N)), np.zeros((rows, 1))
    loss64 = labs = 0.0
    for s in range(len(offsets)):
        o0, L = int(offsets[s]), int(lengths[s])
        sl = slice(o0, o0 + L)
        c, t = 1.0 / L, tg[sl].astype(np.float64)
        if not continuous:
            lg = zk[sl]
            p = np.exp(lg - lg.max(1, keepdims=True))
            p /= p.sum(1, keepdims=True)
            u = p + np.finfo(np.float32).eps
            su = u.sum(1, keepdims=True)
            ls = np.log(u) - np.log(su)
            H = -(u * ls).sum(1)
            onehot = np.arange(N)[None, :] == actions[sl][:, None]
            logp = ls[onehot]
            g = c * (-t[:, None] * (onehot / u - 1 / su) + beta * ls)
            dz64[sl] = p * (g - (p * g).sum(1, keepdims=True))
            dzb[sl, 0] = 2.0 ** -14 * (np.abs(dz64[sl]).max(1) + c * (np.abs(t) + beta * np.abs(ls).max(1)))
            np.testing.assert_allclose(o["pol"][sl], p, rtol=0, atol=1e-6)
        else:
            th = np.tanh(zk[sl])
            mu = th * rg
            diff = actions[sl].astype(np.float64) - mu
            logp = -0.5 * (diff ** 2).sum(1) - 0.5 * N * np.log(2 * np.pi)
            H = np.full(L, 0.5 * N * (1 + np.log(2 * np.pi)))
            dz64[sl] = (-c * t[:, None] * diff) * rg * (1 - th * th)
            dzb[sl, 0] = 2.0 ** -14 * (c * np.abs(t)[:, None] * (np.abs(diff) + rg) * rg).max(1)
            np.testing.assert_allclose(o["pol"][sl], mu, rtol=0, atol=2e-6 * 3)
        loss64 += -(logp * t).mean() - beta * H.mean()
        labs += np.abs(logp * t).mean() + beta * np.abs(H).mean()
    assert not o["dz"][n:].any() and not o["z"][n:].any() and not o["dh"][n:].any()
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


@pytest.mark.parametrize("seed", range(6))
def test_head_against_fp64_on_random_tables(seed):
    rng = np.random.RandomState(seed)
    continuous = seed >= 3
    S = [1, 5, 3, 1, 4, 2][seed]
    K = [256, 512][seed % 2]
    N = [2, 18, 6, 1, 32, 7][seed]
    beta = [0.0, 0.01, 0.05][seed % 3]
    args = _random(rng, S, K, N, continuous, maxlen=[1000, 200, 129, 1000, 64, 300][seed], pad=[0, 5, 31, 7, 0, 19][seed])
    o = head(*args[:7], continuous, args[8], beta, rows=args[7])
    _fp64_check(args, o, continuous, beta)


@pytest.mark.parametrize("continuous", [False, True])
def test_repeat_calls_graph_replay_and_planes_give_identical_bits(continuous):
    rng = np.random.RandomState(5)
    args = _random(rng, 5, 512, 4 if continuous else 18, continuous, pad=9)
    rows = args[7] + (-args[7]) % 8
    a = head(*args[:7], continuous, args[8], 0.01, rows=rows)
    b = head(*args[:7], continuous, args[8], 0.01, rows=rows, planes=True)
    keys = ("z", "pol", "dz", "loss", "dh", "dw", "db")
    for k in keys:
        np.testing.assert_array_equal(a[k].view(np.uint32), b[k].view(np.uint32), err_msg=k)
    t, out, ws, pl = b["_keep"]
    L_, lb = lib()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        L_.check(lb.cb200_policy_gradient_head(ctypes.byref(b["_desc"]), L_.current_stream()))
    for v in out.values():
        v.fill_(float("nan"))
    pl.zero_()
    graph.replay()
    torch.cuda.synchronize()
    for k in keys:
        np.testing.assert_array_equal(out[k].cpu().numpy().view(np.uint32), a[k].view(np.uint32), err_msg=k)
    hi = pl.view(3, -1)[0].cpu().numpy().astype(np.uint16)
    dh = a["dh"].view(np.uint32)
    r, c = np.meshgrid(np.arange(rows), np.arange(512), indexing="ij")
    tiled = ((r // 8) * (512 // 8) + c // 8) * 64 + (r % 8) * 8 + c % 8
    np.testing.assert_array_equal(hi[tiled], (dh >> 16).astype(np.uint16))


def test_argument_errors():
    L_, lb = lib()
    rng = np.random.RandomState(1)
    args = _random(rng, 2, 256, 6, False, maxlen=20)
    o = head(*args[:7], False, None, rows=args[7])
    d = o["_desc"]
    call = lambda: L_.check(lb.cb200_policy_gradient_head(ctypes.byref(d), L_.current_stream()))      # noqa: E731
    for field, bad in (("n_outputs", 19), ("n_outputs", 0), ("features", 128), ("segments", 0), ("rows", 0),
                       ("h", None), ("targets", None), ("workspace", None), ("actions", None), ("z", None)):
        old = getattr(d, field)
        setattr(d, field, bad)
        with pytest.raises(ValueError):
            call()
        setattr(d, field, old)
    d.continuous = 1                                           # continuous without its actions and range
    with pytest.raises(ValueError):
        call()
    d.continuous = 0
    call()
    x = torch.zeros(4, dtype=torch.float64, device="cuda")
    for resc, tab in ((4, x), (-1, x), (3, None)):
        with pytest.raises(ValueError):
            L_.check(lb.cb200_pg_targets(x.data_ptr(), x.data_ptr(), x.data_ptr(), 1, 4, resc,
                                         tab.data_ptr() if tab is not None else None, x.data_ptr(), 4, x.data_ptr(),
                                         None, None, L_.current_stream()))
    z = torch.zeros((4, 3), device="cuda")
    for envs, n, cont in ((0, 2, 0), (4, 19, 0), (4, 33, 1), (4, 0, 0)):
        with pytest.raises(ValueError):
            L_.check(lb.cb200_policy_act(z.data_ptr(), envs, n, cont, z.data_ptr(), None, None, x.data_ptr(), None,
                                         x.data_ptr(), None, L_.current_stream()))


def test_head_beyond_65535_chunks():
    """4,194,340 rows make 65,537 chunks of 64 rows, more than a grid's y dimension holds: the dW pass strides over
    them.  Only the last 100 rows have a nonzero target, so dW, db and the loss come from the chunks past 65,535."""
    L_, lb = lib()
    rows, K, N = 65535 * 64 + 100, 256, 1
    g = torch.Generator(device="cuda").manual_seed(0)
    h = torch.relu(torch.randn((rows, K), device="cuda", generator=g))
    w = torch.randn((K, N), device="cuda", generator=g) * 0.05
    b = torch.zeros(N, device="cuda")
    tg = torch.zeros(rows, device="cuda")
    tg[-100:] = torch.randn(100, device="cuda", generator=g)
    act = torch.rand((rows, N), device="cuda", generator=g) * 6 - 3
    rg = torch.full((N,), 3.0, device="cuda")
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    ln = torch.full((1,), rows, dtype=torch.int32, device="cuda")
    z, dz = torch.empty((rows, N), device="cuda"), torch.empty((rows, N), device="cuda")
    loss, dw, db = torch.empty(1, device="cuda"), torch.empty((K, N), device="cuda"), torch.empty(N, device="cuda")
    ws = torch.empty(rows * (N + 1) + (rows + 63) // 64 * (K * N + N + 1), device="cuda")
    d = L_.PolicyGradientHeadDesc()
    d.h, d.w, d.b, d.targets, d.cont_actions, d.max_abs_range = (x.data_ptr() for x in (h, w, b, tg, act, rg))
    d.seg_offsets, d.seg_lengths, d.segments, d.rows = off.data_ptr(), ln.data_ptr(), 1, rows
    d.continuous, d.features, d.n_outputs = 1, K, N
    d.z, d.dz, d.loss, d.dw, d.db, d.workspace = (x.data_ptr() for x in (z, dz, loss, dw, db, ws))
    L_.check(lb.cb200_policy_gradient_head(ctypes.byref(d), L_.current_stream()))
    torch.cuda.synchronize()
    assert not dz[:-100].any() and dz[-100:].abs().min() > 0
    hl, dzl = h[-100:].double(), dz[-100:].double()
    dw64, db64 = hl.T @ dzl, dzl.sum(0)
    bound = 102 * EPS32 * (hl.abs().T @ dzl.abs()) + 1e-30
    assert ((dw.double() - dw64).abs() <= bound).all()
    assert (db.double() - db64).abs().max() <= 102 * EPS32 * dzl.abs().sum()
    assert float(loss) != 0


# ---- acting -----------------------------------------------------------------------------------------------------------
def test_policy_act_equals_numpys_draws():
    from oracle import a3c as oa, pg as op
    L_, lb = lib()
    rng = np.random.RandomState(2)
    E, A = 64, 5
    z = (rng.randn(E, A) * 2).astype(np.float32)
    u = rng.random_sample(E)
    act = torch.zeros(E, dtype=torch.int64, device="cuda")
    probs = torch.zeros((E, A), device="cuda")
    zt, ut = T(z, np.float32), T(u, np.float64)
    L_.check(lb.cb200_policy_act(zt.data_ptr(), E, A, 0, None, ut.data_ptr(), None, act.data_ptr(), probs.data_ptr(),
                                 None, None, L_.current_stream()))
    pr = probs.cpu().numpy()
    assert act.cpu().numpy().tolist() == [oa.categorical_choice(pr[e], u[e]) for e in range(E)]
    # the same draw as cb200_categorical_act on the actor-critic layout
    z3 = np.concatenate([np.zeros((E, 1), np.float32), z], 1)
    act2 = torch.zeros(E, dtype=torch.int64, device="cuda")
    probs2 = torch.zeros((E, A), device="cuda")
    L_.check(lb.cb200_categorical_act(T(z3, np.float32).data_ptr(), E, A, ut.data_ptr(), act2.data_ptr(),
                                      probs2.data_ptr(), L_.current_stream()))
    assert torch.equal(act, act2) and torch.equal(probs, probs2)
    L_.check(lb.cb200_policy_act(zt.data_ptr(), E, A, 0, None, None, None, act.data_ptr(), None, None, None,
                                 L_.current_stream()))
    assert (act.cpu().numpy() == np.argmax(pr, axis=1)).all()
    # continuous: the fixture's AdditiveNoise draws, means planted as z = atanh(mean / 3)
    means = G["noise_means"]
    n = len(means)
    zc = np.arctanh(means.astype(np.float64) / 3).astype(np.float32)
    np.random.seed(int(G["noise_seed"]))
    normals = np.random.standard_normal((n, 1))
    scale = np.asarray(float(G["noise_value"]) * (G["noise_high"] - G["noise_low"]), dtype=np.float64)
    scale = np.tile(scale, (n, 1))                             # every environment's own scale, [envs, D]
    out = torch.zeros((n, 1), dtype=torch.float64, device="cuda")
    mo = torch.zeros((n, 1), device="cuda")
    zct, nt, sct = T(zc, np.float32), T(normals, np.float64), T(scale, np.float64)
    rgt = T(np.full(1, 3, np.float32), np.float32)
    L_.check(lb.cb200_policy_act(zct.data_ptr(), n, 1, 1, rgt.data_ptr(), nt.data_ptr(), sct.data_ptr(), None, None,
                                 out.data_ptr(), mo.data_ptr(), L_.current_stream()))
    m = mo.cpu().numpy()
    want = op.additive_noise(m[:, 0], float(G["noise_value"]), G["noise_low"], G["noise_high"], normals[:, 0])
    np.testing.assert_array_equal(out.cpu().numpy()[:, 0].view(np.uint64), want.view(np.uint64))
    if np.array_equal(m, means):                               # the tanh reproduced the fixture's means exactly
        np.testing.assert_array_equal(out.cpu().numpy()[:, 0], G["noise_train"][:, 0])
    L_.check(lb.cb200_policy_act(zct.data_ptr(), n, 1, 1, rgt.data_ptr(), None, None, None, None, out.data_ptr(),
                                 None, L_.current_stream()))
    np.testing.assert_array_equal(out.cpu().numpy().astype(np.float32), m)


# ---- the agent --------------------------------------------------------------------------------------------------------
def _agent(continuous=False, E=1, seed=0, rescaler=None, every=None, lr=None, beta=None):
    from coach_b200.agents.policy_gradients_agent import PolicyGradientsAgent, PolicyGradientRescaler
    if continuous:
        from coach_b200.presets import InvertedPendulum_PG as P
        kw = dict(action_dim=P.action_dim, action_low=P.action_low, action_high=P.action_high)
    else:
        from coach_b200.presets import CartPole_PG as P
        kw = dict(num_actions=P.num_actions)
    ap = copy.deepcopy(P.agent_params)
    if rescaler is not None:
        ap.algorithm.policy_gradient_rescaler = PolicyGradientRescaler[rescaler]
    if every is not None:
        ap.algorithm.apply_gradients_every_x_episodes = every
    if lr is not None:
        ap.network_wrappers["main"].learning_rate = lr
    if beta is not None:
        ap.algorithm.beta_entropy = beta
    return PolicyGradientsAgent(ap, observation_shape=P.observation_shape, num_envs=E, seed=seed, **kw)


def _stream(continuous, E, steps, seed, p_end=0.1):
    rng = np.random.RandomState(seed)
    s = rng.uniform(-1, 1, (steps + 1, E, 4)).astype(np.float32)
    acts = rng.uniform(-3, 3, (steps, E, 1)).astype(np.float32) if continuous else rng.randint(0, 2, (steps, E))
    return dict(states=s[:-1], next_states=s[1:], actions=acts,
                rewards=rng.choice([-1.0, 0.0, 1.0, 0.37, 11.0], (steps, E)) / 20., dones=rng.rand(steps, E) < p_end)


def _oracle(agent, dtype=torch.float32):
    from oracle import nets as on, nstep_q as oq, pg as op
    named = agent.net_def.store.export_named()
    p, alg = agent.ap.network_wrappers["main"], agent.ap.algorithm
    net = oq.NStepQNetOracle(agent.observation_shape, agent.num_outputs, dtype)
    opt = on.AdamTF([torch.from_numpy(v).to(dtype) for v in named.values()], p.learning_rate, 0.9, 0.99, 1e-4,
                    dtype=dtype)
    rg = agent.max_abs_range.cpu().numpy() if agent.continuous else None
    return op.Learner(net, net.cast(named), opt, alg.policy_gradient_rescaler.name, alg.discount, agent.every,
                      agent.t_max, agent.continuous, rg, float(alg.beta_entropy))


def _close_params(got, o32, o64, names, lr):
    """within 1e-5 of the fp32 oracle or of fp64, else no farther from fp64 than twice the fp32 oracle; the scale of a
    tensor is its largest magnitude, and at least the learning rate: a parameter that starts at zero (a bias) moves by
    about lr per Adam step"""
    for k in names:
        want, w64 = o32.params[k].numpy(), o64.params[k].numpy()
        tol = 1e-5 * max(np.abs(want).max(), lr)
        if np.abs(got[k] - want).max() > tol and np.abs(got[k] - w64).max() > tol:
            err = np.abs(got[k] - want).max()
            e_ours, e_orc = np.abs(got[k] - w64).max(), np.abs(want - w64).max()
            assert e_ours <= 2 * e_orc, "%s: %.3e > %.3e; vs fp64 ours %.3e, fp32 oracle %.3e" % (k, err, tol, e_ours,
                                                                                                  e_orc)


def _drive(agent, st, steps, sequential, lo_step=0, oracles=None, learned=None):
    """observe / train over the stream's lock-steps [lo_step, steps); after every train() that learned, the fp32 and
    fp64 oracles (new, or ``oracles`` continued) get the same episodes -- as the agent's parts, or one episode per learn
    step (``sequential``) -- and the parameters are compared.  ``learned`` collects (stream, last step, rows) of every
    learned episode.  Returns [(step, [(episodes, applied)])]."""
    o32, o64 = oracles if oracles is not None else (_oracle(agent), _oracle(agent, torch.float64))
    names = list(o32.params.keys())
    log = []
    for t in range(lo_step, steps):
        agent.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t], st["dones"][t])
        loss = agent.train()
        if not agent.learned_segments:
            continue
        eps = []
        for e, start, end in agent.learned_segments:
            ts = list(range(t - (end - start) + 1, t + 1))
            eps.append(dict(states=st["states"][ts, e], actions=st["actions"][ts, e], rewards=st["rewards"][ts, e]))
            if learned is not None:
                learned.append((e, t, end - start))
        log.append((t, list(agent.last_parts)))
        sizes = [1] * len(eps) if sequential else [n for n, _ in agent.last_parts]
        lo = 0
        for n in sizes:
            l32, _ = o32.learn(eps[lo:lo + n])
            l64, _ = o64.learn(eps[lo:lo + n])
            lo += n
        if not sequential:
            assert abs(loss - l32) <= 1e-5 * max(1.0, abs(l32)) or abs(loss - l64) <= 2 * abs(l32 - l64), \
                (loss, l32, l64)
        assert o32.episodes == agent.current_episode
        _close_params(agent.net_def.store.export_named(), o32, o64, names,
                      agent.ap.network_wrappers["main"].learning_rate)
    return log


@pytest.mark.parametrize("continuous,rescaler", [(False, None), (False, "FUTURE_RETURN_NORMALIZED_BY_EPISODE"),
                                                 (True, None), (True, "TOTAL_RETURN")])
def test_one_stream_tracks_the_oracle_across_apply_boundaries(continuous, rescaler):
    torch.manual_seed(0)
    agent = _agent(continuous, E=1, seed=1, rescaler=rescaler, lr=1e-3, beta=0.01 if rescaler else None)
    st = _stream(continuous, 1, 260, seed=4)
    log = _drive(agent, st, 260, sequential=False)
    assert agent.current_episode >= 12
    assert sum(a for _, parts in log for _, a in parts) >= 3   # at least three applies


@pytest.mark.parametrize("continuous", [False, True])
def test_sixteen_streams_equal_a_sequential_run(continuous):
    torch.manual_seed(0)
    agent = _agent(continuous, E=16, seed=2, lr=1e-3)
    st = _stream(continuous, 16, 40, seed=5, p_end=0.12)
    log = _drive(agent, st, 40, sequential=True)
    assert any(len(parts) > 1 for _, parts in log)            # some lock-step was split at a multiple of x


def test_an_episode_reaching_t_max_is_refused():
    agent = _agent(False, E=2, seed=3)
    agent.t_max = 4                                            # the buffers hold 20000 steps; only the check moves
    st = _stream(False, 2, 4, seed=1, p_end=0.0)
    for t in range(3):
        agent.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t], st["dones"][t])
        assert agent.train() == 0
    agent.observe_batch(st["states"][3], st["actions"][3], st["rewards"][3], st["next_states"][3], st["dones"][3])
    theta = agent.net_def.store.theta.clone()
    with pytest.raises(ValueError):
        agent.train()
    assert torch.equal(theta, agent.net_def.store.theta)


def test_graph_replay_is_bit_identical_to_eager(monkeypatch):
    def run(graph):
        monkeypatch.setenv("CB200_PG_GRAPH", "1" if graph else "0")
        a = _agent(False, E=32, seed=3)
        st = _stream(False, 32, 90, seed=6, p_end=0.0)
        st["dones"][[29, 59, 89]] = True                        # 32 episodes of 30 rows close together: parts of up to
        losses = []                                            # 5 episodes, 150 rows in a 160-row bucket
        for t in range(90):
            a.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t], st["dones"][t])
            losses.append(a.train())
        return a, losses
    g, lg = run(True)
    e, le = run(False)
    assert g.graph_kernel_launches > 0 and e.graph_kernel_launches == 0
    assert lg == le
    assert torch.equal(g.net_def.store.theta, e.net_def.store.theta)


@pytest.mark.parametrize("continuous", [False, True])
def test_acting(continuous):
    from oracle import a3c as oa, nstep_q as oq
    E = 16
    agent = _agent(continuous, E=E, seed=4)
    x = np.random.RandomState(0).randn(E, 4).astype(np.float32)
    o = oq.NStepQNetOracle((4,), agent.num_outputs, torch.float64)
    z = o.forward(o.cast(agent.net_def.store.export_named()), x).numpy()
    np.random.seed(11)
    actions, aux = agent.choose_actions(x)
    np.random.seed(11)
    if not continuous:
        u = np.random.random_sample(E)
        p64 = np.exp(z - z.max(1, keepdims=True))
        p64 /= p64.sum(1, keepdims=True)
        np.testing.assert_allclose(aux, p64, rtol=1e-5, atol=1e-7)
        assert actions.tolist() == [oa.categorical_choice(aux[e], u[e]) for e in range(E)]
        ev, _ = agent.choose_actions(x, evaluation=True)
        assert (ev == np.argmax(aux, axis=1)).all()
    else:
        normals = np.random.standard_normal((E, 1))
        np.testing.assert_allclose(aux, np.tanh(z) * 3, rtol=0, atol=1e-5)
        want = aux.astype(np.float64) + np.float64(np.float32(0.1 * 6.0)) * normals
        np.testing.assert_array_equal(actions, want)
        ev, _ = agent.choose_actions(x, evaluation=True)
        assert ev.dtype == np.float32 and np.array_equal(ev, aux)
        # a decaying schedule: environment e's noise is the value after e steps, as E successive get_action calls
        from coach_b200.presets import InvertedPendulum_PG as P
        from coach_b200.schedules import LinearSchedule
        agent.noise_schedule, ref = LinearSchedule(0.3, 0.05, 20), LinearSchedule(0.3, 0.05, 20)
        for _ in range(2):                                     # the second call starts at the 16th value (clipped)
            normals = np.random.RandomState(1).standard_normal((E, 1))
            actions, aux = agent.choose_actions(x, draws=normals)
            scale = []
            for _ in range(E):
                scale.append(np.asarray(ref.current_value * (P.action_high - P.action_low), dtype=np.float64))
                ref.step()
            want = aux.astype(np.float64) + np.stack(scale) * normals
            np.testing.assert_array_equal(actions, want)
            assert len({float(v[0]) for v in scale}) > 1
        assert agent.noise_schedule.current_value == ref.current_value


def test_restore_with_open_episodes_discards_them_and_tracks_the_oracle(tmp_path):
    """E = 4 streams checkpointed with episodes open: after the restore those episodes are neither learned nor counted
    (their rows before the checkpoint are not saved), every episode learned afterwards started after the restore, and
    the parameters, the episode counter and the per-timestep table follow the oracle that saw exactly the learned
    episodes"""
    from coach_b200 import checkpoint
    E, mid, steps = 4, 50, 140
    st = _stream(False, E, steps, seed=9, p_end=0.08)
    a = _agent(False, E=E, seed=6, lr=1e-3)
    o32, o64 = _oracle(a), _oracle(a, torch.float64)
    _drive(a, st, mid, True, oracles=(o32, o64))
    opened = np.nonzero(a.segments.episode_length > 0)[0]
    assert len(opened) >= 2 and a.current_episode >= 4
    name = checkpoint.save_checkpoint(a, str(tmp_path), checkpoint_id=1)
    b = _agent(False, E=E, seed=9, lr=1e-3)
    checkpoint.restore_checkpoint(b, str(tmp_path), name)
    assert torch.equal(b.table, a.table) and b.current_episode == a.current_episode
    learned = []
    _drive(b, st, steps, True, lo_step=mid, oracles=(o32, o64), learned=learned)
    assert all(t - L + 1 >= mid for _, t, L in learned)
    cut = [(e, mid + int(np.argmax(st["dones"][mid:, e]))) for e in opened if st["dones"][mid:, e].any()]
    assert cut and not any((e, t) in {(le, lt) for le, lt, _ in learned} for e, t in cut)
    assert len(learned) >= 8 and o32.episodes == b.current_episode
    tab = b.table.cpu().numpy()
    np.testing.assert_array_equal(tab[0].view(np.uint64), o32.table.mean.view(np.uint64))
    np.testing.assert_array_equal(tab[1], o32.table.count)


def test_checkpoint_mid_accumulation_restores_identically(tmp_path):
    from coach_b200 import checkpoint
    st = _stream(False, 1, 200, seed=8, p_end=0.1)
    a = _agent(False, E=1, seed=5, lr=1e-3)

    def run(agent, lo, hi):
        out = []
        for t in range(lo, hi):
            agent.observe_batch(st["states"][t], st["actions"][t], st["rewards"][t], st["next_states"][t],
                                st["dones"][t])
            out.append(agent.train())
        return out
    mid = 0
    for t in range(200):                                       # stop right after an episode that did not apply
        run(a, t, t + 1)
        if a.learned_segments and a.current_episode % a.every != 0 and a.current_episode >= 7:
            mid = t + 1
            break
    assert mid and a.accumulator.abs().sum() > 0
    name = checkpoint.save_checkpoint(a, str(tmp_path), checkpoint_id=1)
    want = run(a, mid, 200)
    b = _agent(False, E=1, seed=9, lr=1e-3)
    checkpoint.restore_checkpoint(b, str(tmp_path), name)
    got = run(b, mid, 200)
    assert got == want
    assert torch.equal(b.net_def.store.theta, a.net_def.store.theta)
    assert torch.equal(b.table, a.table) and b.current_episode == a.current_episode
