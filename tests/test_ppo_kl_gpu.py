"""PPO (KL penalty) on the GPU: cb200_ppo_kl_head and cb200_ppo_gaussian_act at the C ABI against fp64 references, and
the agent's critic step, actor step, training phase (eager and CUDA-graph replay), KL coefficient updates, acting and
checkpoint round trip against oracle/ppo.py.

Head bound: every output within 1e-4 of its fp64 magnitude -- for a gradient element or the KL, the sum of the absolute
values of the terms it adds up (fp32 sums of up to 4096 rows of up to 32 dimensions, and a likelihood ratio whose
exponent is a difference of two sums of up to 32 squares plus the log-normaliser).  Agent bound: the error
against fp64 at most 2x the fp32 oracle's own deviation from fp64, plus a floor of 2e-6 of the tensor's scale."""

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import ppo as op     # noqa: E402  (checker only)

EPS = 1e-15


def _lib():
    from coach_b200 import _lib as L
    return L, L.load()


def _case(rng, B, A, spread):
    """inputs of one head call; spread scales how far the new policy is from the old one"""
    mu = rng.randn(B, A).astype(np.float32)
    old_mu = (mu + spread * rng.randn(B, A)).astype(np.float32)
    logstd = (rng.randn(A) * 0.3).astype(np.float32)
    old_logstd = (logstd + spread * rng.randn(A)).astype(np.float32)
    actions = (mu + np.exp(logstd) * rng.randn(B, A)).astype(np.float32)
    adv = rng.randn(B).astype(np.float32)
    return dict(mu=mu, logstd=logstd, actions=actions, old_mu=old_mu, old_logstd=old_logstd, adv=adv)


def _magnitudes(c, kl_coef, cutoff, hp, use_kl, beta):
    """fp64 sums of the absolute row terms of every output (the scale a fp32 sum's error is relative to)"""
    d = {k: v.astype(np.float64) for k, v in c.items()}
    B, A = d["mu"].shape
    s, so = np.exp(d["logstd"]) + EPS, np.exp(d["old_logstd"]) + EPS
    z, zo, dm = (d["actions"] - d["mu"]) / s, (d["actions"] - d["old_mu"]) / so, (d["mu"] - d["old_mu"]) / s
    logp = -0.5 * (z * z).sum(1) - np.log(s).sum()
    logpo = -0.5 * (zo * zo).sum(1) - np.log(so).sum()
    ratio = np.exp(logp - logpo)
    rs = so / s
    kl = (0.5 * (rs * rs + dm * dm - 1) - np.log(rs)).sum(1)
    kl_abs = (0.5 * (rs * rs + dm * dm + 1) + np.abs(np.log(rs))).sum(1)      # the terms the fp32 sum cancels
    f = (kl_coef + 2 * hp * max(0.0, kl.mean() - cutoff)) if use_kl else 0.0
    dlogp = np.abs(d["adv"] * ratio)[:, None] / B
    m_mu = (dlogp * np.abs(z) + f / B * np.abs(dm)) / s
    m_ls = (dlogp * (z * z + 1) + f / B * (1 + rs * rs + dm * dm)).sum(0) + abs(beta)
    surr = np.abs(d["adv"] * ratio).mean()
    ent = 0.5 * A * (1 + np.log(2 * np.pi)) + np.abs(np.log(s)).sum()
    m_sc = np.array([surr + abs(beta) * ent + f * kl_abs.mean() + kl_coef, kl_abs.mean(), ent, ratio.mean(), surr])
    return m_mu, m_ls, m_sc, kl.mean()


def _run(c, kl_coef_dev, cutoff, hp, use_kl, beta, outs=None):
    L, lib = _lib()
    t = {k: torch.from_numpy(v).cuda() for k, v in c.items()}
    B, A = c["mu"].shape
    if outs is None:
        outs = (torch.full((B, A), np.nan, device="cuda"), torch.full((A,), np.nan, device="cuda"),
                torch.full((5,), np.nan, device="cuda"))
    rc = lib.cb200_ppo_kl_head(t["mu"].data_ptr(), t["logstd"].data_ptr(), t["actions"].data_ptr(),
                               t["old_mu"].data_ptr(), t["old_logstd"].data_ptr(), t["adv"].data_ptr(), B, A,
                               kl_coef_dev.data_ptr() if kl_coef_dev is not None else None, cutoff, hp, int(use_kl),
                               beta, outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(),
                               L.current_stream())
    L.check(rc)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in outs], t


def _check_head(c, got, kl_coef, cutoff, hp, use_kl, beta):
    g_mu, g_ls, sc = op.kl_head(c["mu"], c["logstd"], c["actions"], c["old_mu"], c["old_logstd"], c["adv"], kl_coef,
                                cutoff, hp, use_kl, beta)
    m_mu, m_ls, m_sc, klbar = _magnitudes(c, kl_coef, cutoff, hp, use_kl, beta)
    for name, x, ref, mag in (("d_mu", got[0], g_mu, m_mu), ("d_logstd", got[1], g_ls, m_ls),
                              ("scalars", got[2], sc, m_sc)):
        err = np.abs(x.astype(np.float64) - ref)
        assert np.all(err <= 1e-4 * mag + 1e-30), (name, float((err / (mag + 1e-30)).max()))
    return klbar


@pytest.mark.parametrize("A", [1, 3, 6, 17, 32])
@pytest.mark.parametrize("B", [1, 128, 1000, 4096])
def test_kl_head_against_fp64(A, B):
    rng = np.random.RandomState(A * 10007 + B)
    c = _case(rng, B, A, 0.1)
    k = torch.tensor([0.7], device="cuda")
    got, _ = _run(c, k, 0.02, 1000.0, True, 0.01)
    _check_head(c, got, 0.7, 0.02, 1000.0, True, 0.01)


@pytest.mark.parametrize("spread,use_kl,side", [(0.02, True, "below"), (0.3, True, "above"), (0.3, False, "above")])
def test_kl_head_around_the_cutoff_and_without_the_penalty(spread, use_kl, side):
    rng = np.random.RandomState(7)
    c = _case(rng, 512, 6, spread)
    cutoff = 0.02
    got, _ = _run(c, torch.tensor([0.2], device="cuda") if use_kl else None, cutoff, 1000.0, use_kl, 0.0)
    klbar = _check_head(c, got, 0.2, cutoff, 1000.0, use_kl, 0.0)
    assert (klbar > 1.5 * cutoff) if side == "above" else (klbar < 0.5 * cutoff)
    if not use_kl:
        # the KL is still reported; the loss is the surrogate alone
        assert got[2][0] == got[2][4]


def test_kl_head_reads_the_device_coefficient_in_a_graph_and_repeats_bits():
    L, lib = _lib()
    rng = np.random.RandomState(11)
    c = _case(rng, 1000, 6, 0.3)
    B, A = c["mu"].shape
    k = torch.tensor([0.2], device="cuda")
    outs = (torch.zeros((B, A), device="cuda"), torch.zeros(A, device="cuda"), torch.zeros(5, device="cuda"))
    first, t = _run(c, k, 0.02, 1000.0, True, 0.01, outs)
    again, _ = _run(c, k, 0.02, 1000.0, True, 0.01, outs)
    for x, y in zip(first, again):
        np.testing.assert_array_equal(x.view(np.uint32), y.view(np.uint32))
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.cuda.graph(g):
        L.check(lib.cb200_ppo_kl_head(t["mu"].data_ptr(), t["logstd"].data_ptr(), t["actions"].data_ptr(),
                                      t["old_mu"].data_ptr(), t["old_logstd"].data_ptr(), t["adv"].data_ptr(), B, A,
                                      k.data_ptr(), 0.02, 1000.0, 1, 0.01, outs[0].data_ptr(), outs[1].data_ptr(),
                                      outs[2].data_ptr(), L.current_stream()))
    g.replay()
    torch.cuda.synchronize()
    for x, y in zip(first, outs):
        np.testing.assert_array_equal(x.view(np.uint32), y.cpu().numpy().view(np.uint32))
    k.fill_(3.0)                                   # a coefficient update between replays
    g.replay()
    torch.cuda.synchronize()
    got = [o.cpu().numpy() for o in outs]
    _check_head(c, got, 3.0, 0.02, 1000.0, True, 0.01)
    assert not np.array_equal(got[1], first[1])


def test_kl_head_and_act_argument_errors():
    L, lib = _lib()
    x = torch.zeros(64, device="cuda")
    p = x.data_ptr()
    bad = [dict(B=0), dict(A=0), dict(A=33), dict(mu=None), dict(d_mu=None), dict(d_logstd=None), dict(k=None)]
    for b in bad:
        a = dict(mu=p, B=4, A=2, k=None if b.get("k", 1) is None else p, d_mu=p, d_logstd=p)
        a.update(b)
        rc = lib.cb200_ppo_kl_head(a["mu"], p, p, p, p, p, a["B"], a["A"], a["k"], 0.02, 1000.0, 1, 0.0, a["d_mu"],
                                   a["d_logstd"], None, L.current_stream())
        assert rc == -1, b
    assert lib.cb200_ppo_gaussian_act(p, p, 0, 2, None, None, None, L.current_stream()) == -1
    assert lib.cb200_ppo_gaussian_act(p, p, 4, 33, None, None, None, L.current_stream()) == -1
    assert lib.cb200_ppo_gaussian_act(p, p, 4, 2, p, None, None, L.current_stream()) == -1
    with pytest.raises(ValueError):
        L.check(lib.cb200_ppo_kl_head(None, p, p, p, p, p, 4, 2, p, 0.02, 1000.0, 1, 0.0, p, p, None,
                                      L.current_stream()))
    # the library and torch stay usable
    _run(_case(np.random.RandomState(1), 8, 2, 0.1), torch.tensor([1.0], device="cuda"), 0.02, 1000.0, True, 0.0)
    assert float((x + 1).sum()) == 64.0


# ---- agent ---------------------------------------------------------------------------------------------------------------
def _agent(D=17, A=6, graph=True, seed=0, playing=256, hp=1000.0, target=0.01, k0=1.0, beta=0.01, rescaler="GAE"):
    from coach_b200.agents.actor_critic_agent import PolicyGradientRescaler
    from coach_b200.agents.ppo_agent import PPOAgent, PPOAgentParameters
    from coach_b200.base_parameters import Dense
    from coach_b200.memories.memory import MemoryGranularity
    ap = PPOAgentParameters()
    for n in ("actor", "critic"):
        ap.network_wrappers[n].input_embedders_parameters['observation'].scheme = [Dense(64)]
        ap.network_wrappers[n].middleware_parameters.scheme = [Dense(64)]
        ap.network_wrappers[n].learning_rate = 1e-3
    ap.memory.max_size = (MemoryGranularity.Transitions, 4096)
    ap.algorithm.num_consecutive_playing_steps.num_steps = playing
    ap.algorithm.high_kl_penalty_coefficient = hp
    ap.algorithm.target_kl_divergence = target
    ap.algorithm.initial_kl_coefficient = k0
    ap.algorithm.beta_entropy = beta
    ap.algorithm.policy_gradient_rescaler = getattr(PolicyGradientRescaler, rescaler)
    return PPOAgent(ap, observation_dim=D, action_dim=A, action_low=-2.0, action_high=2.0, seed=seed,
                    use_cuda_graph=graph)


def _rollout(rng, n, D, A, ep_len):
    s = rng.randn(n, D).astype(np.float32)
    a = rng.randn(n, A).astype(np.float32)
    r = rng.randn(n)
    done = np.zeros(n, np.uint8)
    done[ep_len - 1::ep_len] = 1
    done[-1] = 1
    return s, a, r, done


def _returns(r, done, discount=0.99):
    out, acc = np.zeros_like(r), 0.0
    for i in range(len(r) - 1, -1, -1):
        acc = r[i] + (0.0 if done[i] else discount * acc)
        out[i] = acc
    return out


def _within(got, f32, f64, name):
    e_ours = np.abs(got.astype(np.float64) - f64).max()
    e_orc = np.abs(f32.astype(np.float64) - f64).max()
    assert e_ours <= 2 * e_orc + 2e-6 * (np.abs(f64).max() + 1e-30), (name, e_ours, e_orc)


def test_critic_and_actor_steps_match_the_oracle():
    ag = _agent(graph=False)
    rng = np.random.RandomState(3)
    B, D, A = ag.B, ag.D, ag.A
    sa = ag.actor.store
    sa.theta.add_(torch.randn(sa.size, device="cuda") * 0.02)              # the new policy differs from the old
    sa.view(sa.theta, ag.logstd_name).copy_(torch.tensor(rng.randn(A).astype(np.float32) * 0.3))
    states, actions = rng.randn(B, D).astype(np.float32), rng.randn(B, A).astype(np.float32)
    adv, targets = rng.randn(B).astype(np.float32), rng.randn(B).astype(np.float32)
    cols = ag._training_columns(B)
    for k, v in dict(states=states, actions=actions, advantages=adv, targets=targets[:, None]).items():
        cols[k].copy_(torch.from_numpy(v))
    c_named, a_named = ag.critic.store.export_named(), sa.export_named()
    a_old = sa.export_named(ag.actor.target)
    lr, b1, b2, eps = 1e-3, 0.9, 0.99, 1e-4
    ref = {dt: op.critic_step(c_named, op.make_adam(c_named, lr, b1, b2, eps, dt), states, targets, dt)
           for dt in (torch.float32, torch.float64)}
    ag.cursor.zero_()
    ag._critic_kernels()
    torch.cuda.synchronize()
    got = ag.critic.store.export_named(ag.critic.store.grad)
    for n in got:
        _within(got[n], ref[torch.float32]["grads"][n], ref[torch.float64]["grads"][n], "critic grad " + n)
    got = ag.critic.store.export_named()
    for n in got:
        _within(got[n], ref[torch.float32]["new_params"][n], ref[torch.float64]["new_params"][n], "critic " + n)
    kw = dict(kl_coef=1.0, kl_cutoff=0.02, high_kl_penalty=1000.0, use_kl=True, beta_entropy=0.01)
    ref = {dt: op.actor_step(a_named, a_old, op.make_adam(a_named, lr, b1, b2, eps, dt), states, actions, adv,
                             dtype=dt, **kw) for dt in (torch.float32, torch.float64)}
    cols["old_mu"].copy_(torch.from_numpy(ref[torch.float32]["old_mu"]))
    ag.cursor.zero_()
    ag._actor_kernels()
    torch.cuda.synchronize()
    got = sa.export_named(sa.grad)
    for n in got:
        _within(got[n], ref[torch.float32]["grads"][n], ref[torch.float64]["grads"][n], "actor grad " + n)
    got = sa.export_named()
    for n in got:
        _within(got[n], ref[torch.float32]["new_params"][n], ref[torch.float64]["new_params"][n], "actor " + n)
    np.testing.assert_allclose(ag.scalars[1].item(), ref[torch.float64]["kl"], rtol=1e-4)
    assert int(ag.cursor.item()) == B


def _phase_tensors(rng, n, D, A, ep_len):
    s, a, r, done = _rollout(rng, n, D, A, ep_len)
    ret = _returns(r, done)
    dev = lambda x: torch.from_numpy(x).cuda()      # noqa: E731
    return (s, a, r, done, ret), (dev(s), dev(a), dev(r), dev(done), dev(ret))


def _oracle_phase(c_named, a_named, host, lam=0.96, k=1.0, hp=1000.0, target=0.01, beta=0.01, rescaler="GAE",
                  dtype=torch.float32, B=128):
    s, a, r, done, ret = host
    lr, b1, b2, eps = 1e-3, 0.9, 0.99, 1e-4
    v = op.values(c_named, s)                                       # fp32 V(s), as the agent computes it
    adv = op.fill_advantages(r, v, done.astype(bool), ret, 0.99, lam, rescaler)
    plan = op.minibatches(len(r), B, 256)
    opt = op.make_adam(c_named, lr, b1, b2, eps, dtype)
    cur = dict(c_named)
    for lo, hi in plan:
        cur = op.critic_step(cur, opt, s[lo:hi], ret[lo:hi].astype(np.float32), dtype)["new_params"]
    critic = cur
    opt = op.make_adam(a_named, lr, b1, b2, eps, dtype)
    cur, old = dict(a_named), dict(a_named)
    for epoch in range(10):
        kls = []
        for lo, hi in plan:
            out = op.actor_step(cur, old, opt, s[lo:hi], a[lo:hi], adv[lo:hi].astype(np.float32), k, 2 * target, hp,
                                True, beta, dtype)
            kls.append(out["kl"])
            cur = out["new_params"]
    return critic, cur, float(np.mean(kls))


@pytest.mark.parametrize("rescaler", ["GAE", "A_VALUE"])
def test_training_phase_eager_and_graph_agree_and_match_the_oracle(rescaler):
    rng = np.random.RandomState(5)
    host, devs = _phase_tensors(rng, 300, 17, 6, 70)
    agents = [_agent(graph=g, rescaler=rescaler) for g in (False, True)]
    c0, a0 = agents[0].critic.store.export_named(), agents[0].actor.store.export_named()
    kls = [ag.train_phase(*devs) for ag in agents]
    torch.cuda.synchronize()
    for st in ("critic", "actor"):
        x, y = (getattr(ag, st).store.theta.cpu().numpy() for ag in agents)
        np.testing.assert_array_equal(x.view(np.uint32), y.view(np.uint32))
    assert kls[0] == kls[1]
    assert agents[1]._actor_step.graph is not None and agents[1]._actor_step.launches > 0
    ref = {dt: _oracle_phase(c0, a0, host, rescaler=rescaler, dtype=dt) for dt in (torch.float32, torch.float64)}
    for i, st in enumerate(("critic", "actor")):
        got = getattr(agents[1], st).store.export_named()
        for n in got:
            _within(got[n], ref[torch.float32][i][n], ref[torch.float64][i][n], st + " " + n)
    np.testing.assert_allclose(kls[1], ref[torch.float64][2], rtol=1e-3)


@pytest.mark.parametrize("direction", ["up", "down"])
def test_kl_coefficient_updates(direction):
    """the high-KL penalty off, so the target does not change the training; the target is then placed so that the
    oracle's KL mean sits 20 % beyond 1.3 x target (up) or 20 % below 0.7 x target (down)"""
    rng = np.random.RandomState(9)
    host, devs = _phase_tensors(rng, 256, 11, 3, 64)
    probe = _agent(D=11, A=3, hp=0.0, k0=0.5)
    c0, a0 = probe.critic.store.export_named(), probe.actor.store.export_named()
    m = _oracle_phase(c0, a0, host, k=0.5, hp=0.0, dtype=torch.float64)[2]
    target = m / (1.3 * 1.2) if direction == "up" else m / (0.7 * 0.8)
    ag = _agent(D=11, A=3, hp=0.0, k0=0.5, target=target)
    s, a, r, done, _ = host
    ag.memory.store_columns({"state:observation": s, "next_state:observation": s, "action": a, "reward": r,
                             "game_over": done})
    ag.total_steps_counter = 256
    ag.train()
    np.testing.assert_allclose(ag.last_kl_mean, m, rtol=0.05)
    want = op.update_kl_coefficient(np.float32(0.5), m, target)
    assert ag.kl_coefficient == want and float(ag.kl_coef.item()) == float(want)
    assert (want > 0.5) == (direction == "up")
    assert ag.memory.num_transitions() == 0 and ag.training_iteration == 1


def test_too_few_rows_is_refused():
    rng = np.random.RandomState(2)
    _, devs = _phase_tensors(rng, 127, 17, 6, 50)
    ag = _agent()
    theta = ag.actor.store.theta.clone()
    with pytest.raises(ValueError, match="fewer than one minibatch"):
        ag.train_phase(*devs)
    assert torch.equal(theta, ag.actor.store.theta)


def test_acting_bits_against_numpy():
    ag = _agent(D=5, A=3)
    sa = ag.actor.store
    sa.view(sa.theta, ag.logstd_name).copy_(torch.tensor([0.3, -0.2, 0.05]))
    rng = np.random.RandomState(4)
    s = rng.randn(7, 5).astype(np.float32)
    n = rng.randn(7, 3)
    v0 = float(ag.noise_schedule.current_value)
    acts, means, stds = ag.choose_actions(s, normals=n)
    assert acts.dtype == np.float64
    np.testing.assert_array_equal(acts.view(np.uint64), op.normal_action(means, stds, n).view(np.uint64))
    ls = sa.view(sa.theta, ag.logstd_name).cpu().numpy()
    np.testing.assert_allclose(stds, np.exp(ls.astype(np.float64))[None].repeat(7, 0), rtol=2e-7)
    ev, means2, _ = ag.choose_actions(s, evaluation=True)
    np.testing.assert_array_equal(ev, means)
    np.testing.assert_array_equal(means2, means)
    a_named = sa.export_named()
    want = op.mlp([torch.from_numpy(v) for v in list(a_named.values())[0:6]], torch.from_numpy(s), op.ACTS).numpy()
    np.testing.assert_allclose(means, want, rtol=1e-5, atol=1e-6)
    assert ag.noise_schedule.current_value == v0      # LinearSchedule(0.1, 0.1, ...) stays; it was stepped 7 times


def test_checkpoint_restore_then_next_phase_is_bit_identical(tmp_path):
    from coach_b200 import checkpoint
    rng = np.random.RandomState(8)
    _, devs1 = _phase_tensors(rng, 256, 17, 6, 64)
    _, devs2 = _phase_tensors(rng, 384, 17, 6, 96)
    a = _agent()
    a.update_kl_coefficient(a.train_phase(*devs1))
    a.noise_schedule.step()
    name = checkpoint.save_checkpoint(a, str(tmp_path))
    b = _agent(seed=123)                       # different weights until restored
    checkpoint.restore_checkpoint(b, str(tmp_path), name)
    assert b.kl_coefficient == a.kl_coefficient and float(b.kl_coef.item()) == float(a.kl_coefficient)
    assert b.noise_schedule.current_value == a.noise_schedule.current_value
    ka, kb = a.train_phase(*devs2), b.train_phase(*devs2)
    torch.cuda.synchronize()
    assert ka == kb
    for st in ("critic", "actor"):
        for buf in ("theta", "m", "v"):
            x, y = (getattr(getattr(ag, st).store, buf).cpu().numpy() for ag in (a, b))
            np.testing.assert_array_equal(x.view(np.uint32), y.view(np.uint32))
        np.testing.assert_array_equal(getattr(a, st).adam_state.cpu().numpy(), getattr(b, st).adam_state.cpu().numpy())
