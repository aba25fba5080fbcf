"""Quantile Regression DQN on the GPU.

  cb200_qr_head at the C ABI: the fixture's inputs give the reference's TD targets, midpoints and target actions bit
    for bit; random shapes (B in {1, 32, 512}, A in {1, 2, 6, 18}, N in {1, 2, 50, 200, 1024}, kappa in
    {0, 0.5, 1, 100}) against an fp64 evaluation of the loss and dq within a stated fp32 bound (the observed e / S is
    printed); exact probes on dyadic data; tied rows in the stable order; repeat calls with identical bits; argument
    errors.  cb200_qr_q_values against numpy.
  QuantileRegressionDQNAgent learn steps against oracle/qr_dqn.py (CartPole and Atari shapes, B = 32 and 128), graph
    replay against eager steps, acting, checkpoints and two ranks.
Reads tests/golden/qr_dqn.npz (written from the unmodified reference by oracle/make_golden_qr_dqn.py)."""
import ctypes
import functools
import os
import random
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from oracle import nets as on
from oracle import qr_dqn as oq
from test_learn_gpu import _device_relu_masks, close      # noqa: E402

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qr_dqn.npz")


def _lib():
    from coach_b200 import _lib as L
    return L, L.load()


def head(nxt, onl, actions, rewards, dones, discount, kappa, workspace_fill=0.0):
    """one cb200_qr_head call on host arrays -> dict of host arrays"""
    L, lib = _lib()
    B, A, N = nxt.shape
    dev = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x)).to(device="cuda", dtype=dt)   # noqa: E731
    t = dict(next=dev(nxt, torch.float32), online=dev(onl, torch.float32), actions=dev(actions, torch.int64),
             rewards=dev(rewards, torch.float64), game_overs=dev(dones, torch.uint8))
    out = dict(dq=torch.full((B, A * N), float("nan"), device="cuda"), loss=torch.full((1,), float("nan"), device="cuda"),
               targets=torch.full((B, N), float("nan"), device="cuda"), taus=torch.full((B, N), float("nan"), device="cuda"),
               target_actions=torch.full((B,), -7, dtype=torch.int64, device="cuda"),
               workspace=torch.full((B,), workspace_fill, device="cuda"))
    d = L.QrHeadDesc()
    for k, v in list(t.items()) + list(out.items()):
        setattr(d, k, v.data_ptr())
    d.discount, d.kappa, d.batch, d.n_actions, d.n_atoms = float(discount), float(kappa), B, A, N
    L.check(lib.cb200_qr_head(ctypes.byref(d), L.current_stream()))
    torch.cuda.synchronize()
    res = {k: v.cpu().numpy() for k, v in out.items() if k != "workspace"}
    res["loss"] = res["loss"][0]
    return res


def ref64(theta, targets, taus, kappa):
    """fp64 evaluation of the loss and d loss / d theta from the fp32 feeds, per sample (memory), and the sums of the
    absolute terms the fp32 bounds scale with"""
    B, N = theta.shape
    loss = 0.0
    S_loss = 0.0
    g = np.zeros((B, N))
    S_g = np.zeros((B, N))
    k = float(np.float32(kappa))
    for b in range(B):
        th, t, tau = (x[b].astype(np.float64) for x in (theta, targets, taus))
        e = t[None, :] - th[:, None]
        a = np.abs(e)
        q = np.minimum(a, k)
        h = k * (a - q) + 0.5 * q * q
        w = np.abs(tau[:, None] - (e < 0))
        loss += (w * h).sum()
        S_loss += (w * h).sum()
        wc = w * np.clip(e, -k, k)
        g[b] = -wc.sum(axis=1) / N
        S_g[b] = np.abs(wc).sum(axis=1) / N
    return loss / N, S_loss / N, g, S_g


def _random_inputs(rng, B, A, N, ties=False):
    nxt = (rng.randn(B, A, N) * 2.0).astype(np.float32)
    onl = (rng.randn(B, A, N) * 2.0).astype(np.float32)
    if ties:
        onl = rng.randint(-3, 4, (B, A, N)).astype(np.float32)
    actions = rng.randint(0, A, B).astype(np.int64)
    rewards = rng.choice([-1.0, 0.0, 1.0, 0.37, 1.0 / 3.0, -250.5], B)
    dones = (rng.rand(B) < 0.2).astype(np.uint8)
    return nxt, onl, actions, rewards, dones


def _check_prologue(res, nxt, onl, actions, rewards, dones, discount):
    """targets bit for bit, midpoints bit for bit (stable order), target actions equal unless two actions' Q' lie
    within fp64 rounding of each other"""
    t, ta, tau = oq.qr_targets(nxt, onl, actions, rewards, dones, discount)
    np.testing.assert_array_equal(res["targets"].view(np.uint32), t.astype(np.float32).view(np.uint32))
    np.testing.assert_array_equal(res["taus"].view(np.uint32), tau.astype(np.float32).view(np.uint32))
    q = oq.q_values(nxt)
    for b in np.nonzero(res["target_actions"] != ta)[0]:
        assert abs(q[b, res["target_actions"][b]] - q[b, ta[b]]) <= 1e-12 * np.abs(q[b]).max(), b


# ---- C ABI ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["a2_n50", "a6_n200", "a18_n7", "a2_n1", "a6_n7"])
def test_fixture_targets_midpoints_and_actions_bit_for_bit(tag):
    g = dict(np.load(GOLDEN))
    p = "c_%s_" % tag
    res = head(g[p + "next"], g[p + "online"], g[p + "actions"], g[p + "rewards"], g[p + "dones"],
               float(g[p + "discount"]), 1.0)
    np.testing.assert_array_equal(res["targets"].view(np.uint32), g[p + "targets"].astype(np.float32).view(np.uint32))
    np.testing.assert_array_equal(res["taus"].view(np.uint32), g[p + "output_0_1"].astype(np.float32).view(np.uint32))
    np.testing.assert_array_equal(res["target_actions"], g[p + "target_actions"])


CASES = [(1, 1, 1, 1.0), (1, 2, 1024, 100.0), (1, 6, 200, 0.0), (32, 1, 1024, 1.0), (32, 2, 50, 100.0),
         (32, 6, 200, 1.0), (32, 18, 2, 0.5), (32, 18, 1024, 0.5), (512, 1, 2, 0.0), (512, 6, 200, 1.0),
         (512, 18, 50, 0.5), (512, 2, 1, 100.0)]


@pytest.mark.parametrize("B,A,N,kappa", CASES, ids=["B%d_A%d_N%d_k%g" % c for c in CASES])
def test_head_matches_fp64_within_the_fp32_bound(B, A, N, kappa):
    rng = np.random.RandomState(B * 1000 + A * 10 + N)
    nxt, onl, actions, rewards, dones = _random_inputs(rng, B, A, N)
    res = head(nxt, onl, actions, rewards, dones, 0.99, kappa)
    _check_prologue(res, nxt, onl, actions, rewards, dones, 0.99)
    theta = onl[np.arange(B), actions]
    L, SL, g, Sg = ref64(theta, res["targets"], res["taus"], kappa)
    # every pair term is a handful of fp32 operations on non-negative parts (<= 8u relative); theta_i's j-sum is
    # sequential (N - 1 additions), then the block tree (8 levels), the batch sum (B / 256 + 8) and the division
    err = abs(float(res["loss"]) - L)
    bound = (N + B // 256 + 40) * U32 * SL
    print("B=%d A=%d N=%d kappa=%g: loss e/S = %.3g (bound %.3g)" % (B, A, N, kappa, err / max(SL, 1e-300),
                                                                    bound / max(SL, 1e-300)))
    assert err <= bound, (err, bound)
    dq = res["dq"].reshape(B, A, N)
    got = dq[np.arange(B), actions]
    eg = np.abs(got - g)
    # each product w * clamp(e) is within 3u of its fp64 value (e, w and the product rounded once each); the j-sum
    # runs in fp64 and is rounded to fp32 once
    print("  dq e/S = %.3g" % float((eg / np.maximum(Sg, 1e-300)).max()))
    assert (eg <= 5 * U32 * Sg).all(), float((eg / np.maximum(Sg, 1e-300)).max())
    if kappa == 0.0:
        assert float(res["loss"]) == 0.0 and not np.abs(dq).max()
    mask = np.ones((B, A), dtype=bool)
    mask[np.arange(B), actions] = False
    assert (dq[mask] == 0).all() and not np.signbit(dq[mask]).any()


def test_exact_probes_on_dyadic_data():
    """N = 4 (1/N and every midpoint exact), quantiles in quarters, dyadic rewards, discount 0.5: every fp32 and fp64
    operation of the head is exact, so the loss and dq equal the fp64 evaluation bit for bit"""
    rng = np.random.RandomState(11)
    B, A, N = 64, 3, 4
    nxt = (rng.randint(-16, 17, (B, A, N)) / 4.0).astype(np.float32)
    onl = np.stack([rng.permutation(N) for _ in range(B * A)]).reshape(B, A, N).astype(np.float32) / 2 - 1
    actions = rng.randint(0, A, B).astype(np.int64)
    rewards = rng.choice([-1.0, 0.0, 0.5, 2.25], B)
    dones = (rng.rand(B) < 0.3).astype(np.uint8)
    for kappa in (1.0, 2.0, 0.5):
        res = head(nxt, onl, actions, rewards, dones, 0.5, kappa)
        _check_prologue(res, nxt, onl, actions, rewards, dones, 0.5)
        L, _, g, _ = ref64(onl[np.arange(B), actions], res["targets"], res["taus"], kappa)
        assert float(res["loss"]) == L, (float(res["loss"]), L)
        np.testing.assert_array_equal(res["dq"].reshape(B, A, N)[np.arange(B), actions], g)


def test_tied_rows_follow_the_stable_order():
    rng = np.random.RandomState(5)
    B, A, N = 32, 4, 50
    nxt, onl, actions, rewards, dones = _random_inputs(rng, B, A, N, ties=True)
    res = head(nxt, onl, actions, rewards, dones, 0.99, 1.0)
    rows = onl[np.arange(B), actions]
    assert all(len(np.unique(r)) < N for r in rows)
    _check_prologue(res, nxt, onl, actions, rewards, dones, 0.99)


def test_repeat_calls_give_identical_bits():
    rng = np.random.RandomState(9)
    args = _random_inputs(rng, 512, 6, 200)
    a = head(*args, 0.99, 1.0, workspace_fill=float("nan"))
    b = head(*args, 0.99, 1.0, workspace_fill=-3.0)
    for k in a:
        np.testing.assert_array_equal(np.atleast_1d(a[k]).view(np.uint8), np.atleast_1d(b[k]).view(np.uint8),
                                      err_msg=k)


def test_argument_errors_raise_valueerror():
    L, lib = _lib()
    buf = torch.zeros(4096, dtype=torch.float64, device="cuda")
    p = buf.data_ptr()

    def desc(**kw):
        d = L.QrHeadDesc()
        for f in ("next", "online", "actions", "rewards", "game_overs", "dq", "loss", "workspace"):
            setattr(d, f, p)
        d.discount, d.kappa, d.batch, d.n_actions, d.n_atoms = 0.99, 1.0, 2, 2, 4
        for k, v in kw.items():
            setattr(d, k, v)
        return d
    L.check(lib.cb200_qr_head(ctypes.byref(desc()), L.current_stream()))
    for kw in (dict(n_atoms=0), dict(n_atoms=1025), dict(n_actions=0), dict(n_actions=257), dict(batch=0),
               dict(kappa=-1.0), dict(kappa=float("nan")), dict(next=None), dict(online=None), dict(actions=None),
               dict(rewards=None), dict(game_overs=None), dict(dq=None), dict(loss=None), dict(workspace=None)):
        with pytest.raises(ValueError):
            L.check(lib.cb200_qr_head(ctypes.byref(desc(**kw)), L.current_stream()))
    with pytest.raises(ValueError):
        L.check(lib.cb200_qr_head(None, L.current_stream()))
    for n in (0, 1025):
        with pytest.raises(ValueError):
            L.check(lib.cb200_qr_q_values(p, 4, n, p, L.current_stream()))
    torch.cuda.synchronize()


@pytest.mark.parametrize("N", [1, 7, 200, 1024])
def test_q_values_kernel(N):
    L, lib = _lib()
    x = (np.random.RandomState(N).randn(37, N) * 5).astype(np.float32)
    q = torch.empty(37, dtype=torch.float64, device="cuda")
    xt = torch.from_numpy(x).cuda()
    L.check(lib.cb200_qr_q_values(xt.data_ptr(), 37, N, q.data_ptr(), L.current_stream()))
    np.testing.assert_allclose(q.cpu().numpy(), oq.q_values(x), rtol=1e-13, atol=1e-13)


# ---- the agent --------------------------------------------------------------------------------------------------------
def _agent(obs, A, B, atoms, seed=0):
    from coach_b200.agents.qr_dqn_agent import QuantileRegressionDQNAgent, QuantileRegressionDQNAgentParameters
    from coach_b200.memories.memory import MemoryGranularity
    ap = QuantileRegressionDQNAgentParameters()
    ap.algorithm.atoms = atoms
    ap.memory.max_size = (MemoryGranularity.Transitions, 1024)
    ap.network_wrappers["main"].batch_size = B
    return QuantileRegressionDQNAgent(ap, observation_shape=obs, num_actions=A, seed=seed)


def _data(obs, A, n, seed):
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


@pytest.mark.parametrize("obs,A,N,B", [((4,), 2, 50, 32), ((84, 84, 4), 6, 200, 32), ((84, 84, 4), 6, 200, 128)],
                         ids=["cartpole_N50_B32", "atari_N200_B32", "atari_N200_B128"])
def test_learn_step_matches_oracle(obs, A, N, B):
    torch.manual_seed(0)
    agent = _agent(obs, A, B, N)
    assert agent.head_outputs == A * N and agent.head_desc is None
    agent.memory.store_columns(_data(obs, A, max(256, 2 * B), 5))
    store = agent.net_def.store
    net = agent.networks["main"]
    net.theta_target.copy_(store.theta * 0.9 + 0.01)
    net.target_changed()
    lr, eps = agent.ap.network_wrappers["main"].learning_rate, agent.ap.network_wrappers["main"].optimizer_epsilon
    oracle32 = on.QNetOracle(obs, A * N, False, torch.float32)
    oracle64 = on.QNetOracle(obs, A * N, False, torch.float64)
    for step in range(2):
        online_named = store.export_named()
        target_named = store.export_named(net.theta_target)
        random.seed(20 + step)
        np.random.seed(20 + step)
        batch = agent.sample_batch()
        if step == 0:
            opt32 = on.AdamTF([torch.from_numpy(v) for v in online_named.values()], lr, 0.9, 0.99, eps)
            opt64 = on.AdamTF([torch.from_numpy(v).double() for v in online_named.values()], lr, 0.9, 0.99, eps,
                              dtype=torch.float64)
        loss, losses, gnorm = agent.learn_from_batch(batch)
        torch.cuda.synchronize()
        for k in ("state:observation", "next_state:observation"):
            batch.column(k)
        cols = {k: v.cpu().numpy() for k, v in batch.columns.items()}
        ob = dict(states=cols["state:observation"], next_states=cols["next_state:observation"],
                  actions=cols["action"], rewards=cols["reward"], game_overs=cols["game_over"].astype(bool))
        # the device's own prologue, bit for bit, on its own network outputs
        q_next = net.target_s2.q.cpu().numpy().reshape(B, A, N)
        q_on = net.online_s.q.cpu().numpy().reshape(B, A, N)
        _check_prologue(dict(targets=agent.qr_targets.cpu().numpy(), taus=agent.taus.cpu().numpy(),
                             target_actions=agent.target_actions.cpu().numpy()),
                        q_next, q_on, ob["actions"], ob["rewards"], ob["game_overs"], 0.99)
        masks = _device_relu_masks(agent)
        k32, k64 = dict(masks=masks, tol=1e-5), dict(masks=masks, tol=1e-5)
        ref = oq.qr_learn_step(oracle32, oracle32.cast(online_named), oracle32.cast(target_named), opt32, ob, 0.99, A, N,
                               kink=k32, sort_quantiles=q_on)
        ref64 = oq.qr_learn_step(oracle64, oracle64.cast(online_named), oracle64.cast(target_named), opt64, ob, 0.99, A,
                                 N, kink=k64, sort_quantiles=q_on)
        assert k32.get("hard", 0) == 0 and k64.get("hard", 0) == 0, "ReLU masks differ away from the kink"
        np.testing.assert_array_equal(agent.target_actions.cpu().numpy(), ref["target_actions"])
        close(agent.qr_targets.cpu().numpy(), ref["targets"], name="TD targets", atol=1e-6)
        close(loss, ref["loss"], name="loss")
        close(net.online_s.dq.cpu().numpy(), ref["dq"], name="dq", atol=1e-8)
        close(gnorm, ref["grad_norm"], name="grad_norm", rtol=2e-5)
        got_grads = store.export_named(store.grad)
        for name in ref["grads"]:
            want = ref["grads"][name].numpy()
            e_ours = np.abs(got_grads[name] - ref64["grads"][name].numpy()).max()
            e_orc = np.abs(want - ref64["grads"][name].numpy()).max()
            try:
                close(got_grads[name], want, name="grad " + name)
            except AssertionError as exc:
                # ill-conditioned weight-gradient sums: not farther from the fp64 evaluation than the fp32 oracle is
                assert e_ours <= 1.5 * e_orc, "%s; vs fp64: ours %.3e, fp32 oracle %.3e" % (exc, e_ours, e_orc)
            assert e_ours <= 4 * e_orc + 2e-6 * (np.abs(want).max() + 1e-30), (name, e_ours, e_orc)
        got_params = store.export_named()
        for name in ref["new_params"]:
            want = ref["new_params"][name].numpy()
            try:
                close(got_params[name], want, name="param " + name)
            except AssertionError as exc:
                # d dq_i / d theta is about 1/2 here (a C51 logit's is p (1 - p)), and QR's Adam epsilon (0.01 / 32)
                # keeps the first update linear in small gradients: the rounding of the forward passes reaches the
                # parameters undamped.  Not farther from fp64 than the weight-gradient clause above allows.
                w64 = ref64["new_params"][name].numpy()
                e_ours, e_orc = np.abs(got_params[name] - w64).max(), np.abs(want - w64).max()
                assert e_ours <= 4 * e_orc, "%s; vs fp64: ours %.3e, fp32 oracle %.3e" % (exc, e_ours, e_orc)


def test_graph_replay_matches_eager(monkeypatch):
    results = []
    for graph in (0, 1):
        monkeypatch.setenv("CB200_DQN_GRAPH", str(graph))
        torch.manual_seed(0)
        agent = _agent((84, 84, 4), 6, 128, 200)
        assert agent.use_graph == bool(graph)
        agent.memory.store_columns(_data((84, 84, 4), 6, 512, 3))
        losses = []
        for step in range(6):                       # 2 eager steps, capture, 3 replays
            random.seed(20 + step)
            np.random.seed(20 + step)
            agent.total_steps_counter += 4
            losses.append(agent.train() if step % 2 else agent.learn_from_batch(agent.sample_batch())[0])
        torch.cuda.synchronize()
        if graph:
            assert agent._graphs is not None and agent.graph_kernel_launches > 0
        results.append((losses, agent.net_def.store.theta.clone(), agent.networks["main"].online_s.dq.clone()))
    assert results[0][0] == results[1][0]
    assert torch.equal(results[0][1], results[1][1])
    assert torch.equal(results[0][2], results[1][2])


def test_acting_q_values():
    """get_all_q_values_for_states = the mean quantile per action in fp64 (np.dot with ones(N) / N)"""
    agent = _agent((4,), 3, 32, 50)
    x = np.random.RandomState(1).uniform(-1, 1, (16, 4)).astype(np.float32)
    q = agent.get_all_q_values_for_states(x).cpu().numpy()
    quantiles = agent._acting[16][1].q.cpu().numpy().reshape(16, 3, 50)
    np.testing.assert_allclose(q, oq.q_values(quantiles), rtol=1e-13, atol=1e-13)


def test_checkpoint_restore_continues_bit_identically(tmp_path):
    from coach_b200 import checkpoint
    obs, A, B = (4,), 2, 32
    a = _agent(obs, A, B, 50, seed=1)
    a.memory.store_columns(_data(obs, A, 300, 2))

    def steps(agent, n, seed):
        out = []
        for k in range(n):
            random.seed(seed + k)
            np.random.seed(seed + k)
            out.append(agent.learn_from_batch(agent.sample_batch())[:2])
        return out
    steps(a, 3, 10)
    a.networks["main"].update_target_network(1.0)
    steps(a, 1, 30)
    name = checkpoint.save_checkpoint(a, str(tmp_path), checkpoint_id=1)
    want = steps(a, 3, 40)
    b = _agent(obs, A, B, 50, seed=9)
    checkpoint.restore_checkpoint(b, str(tmp_path), name)
    got = steps(b, 3, 40)
    assert got == want
    assert torch.equal(b.net_def.store.theta, a.net_def.store.theta)
    assert torch.equal(b.taus, a.taus)


# ---- two ranks (gloo, both on cuda:0: the pattern of tests/test_naf_gpu.py) -------------------------------------------
def _run_ranked(data_seed):
    ag = _agent((4,), 2, 32, 50, seed=5)
    ag.memory.store_columns(_data((4,), 2, 600, data_seed))
    losses = []
    for step in range(4):
        random.seed(20 + step)
        np.random.seed(20 + step)
        losses.append(ag.learn_from_batch(ag.sample_batch())[0])
    torch.cuda.synchronize()
    return losses, ag.net_def.store.theta.cpu().numpy()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, port, shard_by_rank, out_q):
    os.environ.update(RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                      CB200_GRAPH_COLLECTIVES="0")          # gloo collectives cannot be captured into a CUDA graph
    try:
        from coach_b200 import parallel
        assert parallel.init_from_env(backend="gloo") == (rank, 2)
        out_q.put((rank, _run_ranked(3 + rank if shard_by_rank else 3)))
        torch.distributed.destroy_process_group()
    except BaseException as exc:
        out_q.put((rank, "rank %d failed: %r" % (rank, exc)))
        raise


@functools.lru_cache(maxsize=None)
def _one_rank():
    return _run_ranked(3)


@pytest.mark.parametrize("shard_by_rank", [False, True])
def test_two_ranks(shard_by_rank):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, shard_by_rank, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = dict(q.get(timeout=600) for _ in procs)
        for r in range(2):
            assert not isinstance(res[r], str), res[r]
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.pid is not None:
                if p.is_alive():
                    p.terminate()
                p.join(timeout=30)
    (l0, t0), (l1, t1) = res[0], res[1]
    assert np.array_equal(t0, t1), "the ranks' parameters diverged"
    if shard_by_rank:
        assert not np.array_equal(t0, _one_rank()[1]), "rank 0 trained as if alone: no gradient exchange"
    else:
        # g + g and the 1/2 rescale are exact: identical shards reproduce one rank bit for bit
        assert l0 == l1 == _one_rank()[0] and np.array_equal(t0, _one_rank()[1])
