"""CPU checks of tests/policy_ref.py: pinned to the reference agents' restatements (oracle/actor_critic.py,
oracle/sac.py, oracle/rl_math.py) and the fixtures, hand-worked cases, the bounds against exact and fp32-emulated
evaluations, and one plausible kernel bug per tolerance shown to fall outside it."""
import math
import os
from fractions import Fraction

import numpy as np
import pytest
import torch

import policy_cases as pc
import policy_ref as pr
from oracle import actor_critic as oac
from oracle import rl_math as orm
from oracle import sac as osac

F32, F64 = np.float32, np.float64
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


# ---- fp32 emulations of the kernels (the mutation hooks are the bugs named in the tests) -------------------------------
def ppo_emulate(mu, ls, a, omu, ols, adv, eps, beta, flip_min=False, clip_grad_passes=False):
    B, A = mu.shape
    sig = (np.exp(ls) + F32(1e-15)).astype(F32)
    osig = (np.exp(ols) + F32(1e-15)).astype(F32)
    z, zo = ((a - mu) / sig).astype(F32), ((a - omu) / osig).astype(F32)
    c = F32(0.5) * F32(A) * F32(pr.LOG2PI)
    lp = -F32(0.5) * (z * z).sum(1, dtype=F32) - np.log(sig).sum(dtype=F32) - c
    lpo = -F32(0.5) * (zo * zo).sum(1, dtype=F32) - np.log(osig).sum(dtype=F32) - c
    r = np.exp(lp - lpo).astype(F32)
    lo, hi = (F32(x) for x in pr.ppo_clip_range(eps))
    cl = np.minimum(np.maximum(r, lo), hi)
    s1, s2 = r * adv, cl * adv
    first = (s1 >= s2) if flip_min else (s1 <= s2)
    inside = np.ones(B, bool) if clip_grad_passes else (r >= lo) & (r <= hi)
    ds = np.where(first | inside, adv, F32(0))
    dlogp = -(F32(1) / F32(B)) * ds * r
    g = ((sig - F32(1e-15)) / sig).astype(F32)
    dmu = (dlogp[:, None] * z / sig).astype(F32)
    dls = ((dlogp[:, None] * (z * z - 1) * g).sum(0, dtype=F32) - F32(beta) * g).astype(F32)
    ent = F32(0.5) * F32(A) * (F32(1) + F32(pr.LOG2PI)) + np.log(sig).sum(dtype=F32)
    rs, dm = osig / sig, (mu - omu) / sig
    kl = (F32(0.5) * (rs * rs + dm * dm - 1) - np.log(rs)).sum(1, dtype=F32)
    sc = np.array([-np.minimum(s1, s2).sum(dtype=F32) / F32(B) - F32(beta) * ent, kl.sum(dtype=F32) / F32(B), ent,
                   r.sum(dtype=F32) / F32(B), cl.sum(dtype=F32) / F32(B)], F32)
    return dmu, dls, sc


def sac_grad_emulate(head, e2, e3, dq, open_mask=False):
    B, A = e2.shape
    mu, lsr = head[:, :A], head[:, A:]
    ls = np.clip(lsr, F32(-20), F32(2))
    inr = ((lsr > -20) & (lsr < 2)) if open_mask else ((lsr >= -20) & (lsr <= 2))
    sig = np.exp(ls).astype(F32)
    t2 = np.tanh(mu + sig * e2).astype(F32)
    gp = (F32(-2) * t2 * (F32(1) - t2 * t2)) / (F32(1) - t2 * t2 + F32(1e-6))
    ib = F32(1) / F32(B)
    t3 = np.tanh(mu + sig * e3).astype(F32)
    w = dq * (F32(1) - t3 * t3)
    d_mu = ib * -gp - w
    d_ls = (ib * (F32(-1) - gp * sig * e2) - w * sig * e3) * inr.astype(F32)
    return np.concatenate([d_mu, d_ls], 1).astype(F32)


def gae_emulate(r, v, done, disc, lam, threads=pr.BLOCK_GAE, warp_bug=False, drop_done=False):
    """the kernel's scan in fp64: chunk folds, a reverse warp scan, warp carries, the chunk replay"""
    n = len(r)
    nd = np.zeros(n) + 1.0 if drop_done else 1.0 - np.asarray(done, bool)
    vn = np.append(np.asarray(v, F64)[1:], 0.0)
    delta = r + disc * nd * vn - np.asarray(v, F64)
    gl = disc * lam
    per = -(-n // threads)
    f = []
    for tid in range(threads):
        a, b = 1.0, 0.0
        for t in range(min(n, (tid + 1) * per) - 1, tid * per - 1, -1):
            a, b = gl * nd[t] * a, gl * nd[t] * b + delta[t]
        f.append((a, b))
    comp = lambda L, R: (L[0] * R[0], L[0] * R[1] + L[1])          # noqa: E731
    s = [None] * threads
    for w in range(threads // 32):                                  # inclusive reverse scan inside each warp
        acc = (1.0, 0.0)
        for lane in range(31, -1, -1):
            acc = comp(f[w * 32 + lane], acc)
            s[w * 32 + lane] = acc
    wt = [s[w * 32] for w in range(threads // 32)]
    adv = np.empty(n)
    for tid in range(threads):
        w, lane = divmod(tid, 32)
        later = (1.0, 0.0)
        for k in range(threads // 32 - 1, w, -1):
            if warp_bug and k == w + 1:
                continue
            later = comp(wt[k], later)
        ex = s[tid + 1] if lane < 31 else (1.0, 0.0)
        y = comp(ex, later)[1]
        for t in range(min(n, (tid + 1) * per) - 1, tid * per - 1, -1):
            y = delta[t] + gl * nd[t] * y
            adv[t] = y
    return adv


# ---- pins ---------------------------------------------------------------------------------------------------------------
def test_ppo_pinned_to_oracle():
    """logp against oracle.actor_critic.ppo_logp; the policy loss and its gradients against ppo_losses with an identity
    policy network (mu = tanh(tanh(s)) inverted on the input), all in fp64"""
    A, B, eps, beta = 4, 32, 0.2, 0.01
    mu, ls, act, omu, ols, adv = pc.ppo_inputs(A, B, eps, seed=11)
    mu = (np.tanh(mu) * 0.7).astype(F32)                             # |mu| < tanh(1) for the identity network
    ref = pr.ppo_reference(mu, ls, act, omu, ols, adv, eps, beta)
    t = lambda x: torch.tensor(np.asarray(x, F64))                   # noqa: E731
    np.testing.assert_allclose(ref["logp"], oac.ppo_logp(t(mu), t(ls), t(act)).numpy(), rtol=1e-13)
    eye = torch.eye(A, dtype=torch.float64)
    zero = torch.zeros(A, dtype=torch.float64)
    p = [eye.clone().requires_grad_(True) if k % 2 == 0 else zero.clone().requires_grad_(True) for k in range(6)]
    v = [torch.zeros(A, 1, dtype=torch.float64), torch.zeros(1, dtype=torch.float64)] * 3
    v[0], v[2] = torch.zeros(A, A, dtype=torch.float64), torch.zeros(A, A, dtype=torch.float64)
    v[1], v[3] = zero, zero
    lst = t(ls).requires_grad_(True)
    states = torch.atanh(torch.atanh(t(mu)))
    _, _, pl, ex = oac.ppo_losses(v, p, lst, t(omu), t(ols), states, t(act), t(adv), torch.zeros(B, dtype=torch.float64),
                                  eps, float(F32(beta)))
    g_b2, g_ls = torch.autograd.grad(pl, [p[5], lst])
    lo, hi = pr.ppo_clip_range(eps)
    assert abs(float(pl.detach()) - ref["scalars"][0]) < 1e-6        # the oracle clips at 1 -+ eps in fp64, the kernel in fp32
    assert not ((np.abs(ref["ratio"] - lo) < 1e-6) | (np.abs(ref["ratio"] - hi) < 1e-6)).any()
    np.testing.assert_allclose(g_b2.numpy(), ref["d_mu"].sum(0), rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(g_ls.numpy(), ref["d_logstd"], rtol=1e-10, atol=1e-13)
    np.testing.assert_allclose(float(ex["entropy"]), ref["scalars"][2], rtol=1e-14)
    np.testing.assert_allclose(ex["ratio"].detach().numpy(), ref["ratio"], rtol=1e-12)


def test_ppo_hand_worked():
    """A = 1, B = 2, logstd = 0: sample 0 has z = 1, z_old = 0.5, ratio e^-0.375 < 0.8 and a positive advantage (the
    unclipped side is smaller: the gradient passes); sample 1 has ratio 1 and advantage -2"""
    mu = np.zeros((2, 1), F32)
    act = np.array([[1.0], [-1.0]], F32)
    omu = np.array([[0.5], [0.0]], F32)
    z0 = np.zeros(1, F32)
    adv = np.array([1.0, -2.0], F32)
    ref = pr.ppo_reference(mu, z0, act, omu, z0, adv, 0.2, 0.0)
    r0 = math.exp(-0.375)
    np.testing.assert_allclose(ref["ratio"], [r0, 1.0], rtol=1e-15)
    np.testing.assert_allclose(ref["d_mu"][:, 0], [-0.5 * r0 * 1.0, -0.5 * (-2.0) * 1.0 * -1.0], rtol=1e-14)
    np.testing.assert_allclose(ref["scalars"][0], -(r0 - 2.0) / 2, rtol=1e-14)
    # d logp / d logstd = z^2 - 1 (sigma = 1): sample 0 contributes -(1/2) r0 (1 - 1) = 0, sample 1 -(1/2)(-2)(1 - 1)
    np.testing.assert_allclose(ref["d_logstd"], [0.0], atol=1e-14)        # sigma = 1 + 1e-15 in fp64
    # the ratio above the range with a positive advantage: clipped, no gradient
    ref = pr.ppo_reference(np.array([[0.5], [0.0]], F32), z0, np.zeros((2, 1), F32), np.array([[1.0], [0.0]], F32), z0,
                           np.array([1.0, 1.0], F32), 0.2, 0.0)
    assert ref["ratio"][0] == pytest.approx(math.exp(0.375)) and not ref["pass_"][0]
    assert ref["d_mu"][0, 0] == 0.0
    np.testing.assert_allclose(ref["scalars"][4], (float(F32(1.2)) + 1.0) / 2, rtol=1e-15)


def test_sac_pinned_to_oracle():
    """sample and log-prob against oracle.sac.policy_sample with an identity network (relu(x + 100) - 100)"""
    A, B = 5, 64
    head, eps = pc.sac_inputs(A, B, seed=2)
    head[:, A:] = np.maximum(head[:, A:], -30)                       # the identity network needs x > -100
    head[:, :A] = np.clip(head[:, :A], -3, 3)                        # and shifts mu by ~1e-14: no saturated tanh
    eye = torch.eye(2 * A, dtype=torch.float64)
    c = torch.full((2 * A,), 100.0, dtype=torch.float64)
    p = [eye, c, eye, torch.zeros(2 * A, dtype=torch.float64), eye, -c]
    act, logp = osac.policy_sample(p, torch.tensor(head.astype(F64)), torch.tensor(eps.astype(F64)))
    ref = pr.sac_sample_reference(head, eps)
    np.testing.assert_allclose(ref["act"], act.numpy(), rtol=1e-12, atol=1e-13)
    # the oracle's (u - mu) / sigma cancels in fp64 where sigma = e^-20; the reference uses eps itself
    np.testing.assert_allclose(ref["logp"], logp.numpy(), rtol=1e-7, atol=1e-7)


def test_rl_math_pinned_to_fixtures():
    fx = np.load(os.path.join(GOLDEN, "rl_math.npz"))
    for k in range(len(fx["gae_lens"])):
        r, v = fx["gae_r_%d" % k], fx["gae_v_%d" % k]
        done = np.zeros(len(r), np.uint8)
        done[-1] = 1
        ref = pr.gae_reference(r, v[:-1].astype(F32), done, 0.99, 0.95)
        vv = v[:-1].astype(F32).astype(F64)                          # the device reads fp32 values
        a_fx, _ = orm.gae(r, np.append(vv, 0.0), 0.99, 0.95)
        assert (np.abs(ref["adv"] - a_fx) <= ref["b_adv"]).all()
        if np.array_equal(v[:-1].astype(F32).astype(F64), v[:-1]):
            assert (np.abs(ref["adv"] - fx["gae_adv_%d" % k]) <= ref["b_adv"]).all()
    for k in range(int(fx["nstep_cases"])):
        r = fx["nstep_r_%d" % k]
        assert np.array_equal(pr.nstep_returns(r, [len(r)], 0.99, int(fx["nstep_n_%d" % k])), fx["nstep_out_%d" % k])
    rs = orm.RunningStats([17])
    s, q, count = np.zeros(17), np.full(17, 1e-2), 1e-2
    for k in range(3):
        x = fx["rs_push%d" % k]
        rs.push(x)
        s, q = s + x.astype(F64).sum(0), q + np.square(x.astype(F64)).sum(0)
        count += x.shape[0]
        m, sd = pr.stats_finalize(rs.sum, rs.sum_squares, rs.count, 1e-2)
        assert np.array_equal(m, rs.mean) and np.array_equal(sd, rs.std)
        np.testing.assert_allclose(m, fx["rs_means"][k], rtol=1e-12, atol=1e-13)
        np.testing.assert_allclose(sd, fx["rs_stds"][k], rtol=1e-11)
    o32, o64 = pr.stats_normalize(fx["rs_query"], rs.mean, rs.std, -5.0, 5.0)
    assert np.array_equal(o64, rs.normalize(fx["rs_query"].astype(F32).astype(F64)))


def test_fill_advantages_pinned():
    """gae_reference over several episodes and a trailing unfinished segment against oracle.ppo_fill_advantages, and
    standardize_reference against its standardisation"""
    rng = np.random.RandomState(4)
    n = 3000
    r, v = rng.randn(n), rng.randn(n).astype(F32)
    done = (rng.rand(n) < 0.02).astype(np.uint8)
    done[-5:] = 0
    ref = pr.gae_reference(r, v, done, 0.99, 0.95)
    o_adv, o_tgt, o_nv = orm.ppo_fill_advantages(r, v, done.astype(bool), 0.99, 0.95)
    nv = ref["n_valid"]
    assert nv == o_nv
    assert (np.abs(ref["tgt"][:nv] - o_tgt[:nv]) <= ref["b_tgt"][:nv]).all()
    out, m, sd, b_out, b_m, b_sd = pr.standardize_reference(ref["adv"], nv)
    assert (np.abs(out[:nv] - o_adv[:nv]) <= b_out[:nv] + 1e-13).all() and np.isnan(out[nv:]).all()


def test_td_targets_and_smoothing_pinned_to_fixture():
    fx = np.load(os.path.join(GOLDEN, "agent_prologues.npz"))
    lo, hi = (float(x) for x in fx["td3_space"])
    sm = pr.td3_smooth(fx["td3_next_actions"], fx["td3_noise"], 0.5, lo, hi)
    assert np.array_equal(sm, np.asarray(fx["td3_smoothed_actions"]).astype(F32))


# ---- bounds against exact and emulated evaluations ----------------------------------------------------------------------
@pytest.mark.parametrize("A,B", [(1, 2), (6, 64), (32, 257)])
def test_ppo_bounds_hold_for_fp32_emulation(A, B):
    for eps, beta in ((0.1, 0.0), (0.2, 0.01)):
        inp = pc.ppo_inputs(A, B, eps, seed=A + B)
        pr.ppo_check(*ppo_emulate(*inp, eps, beta), pr.ppo_reference(*inp, eps, beta), "emulated")


def test_sac_bounds_hold_for_fp32_emulation():
    A, B = 6, 300
    head, e3 = pc.sac_inputs(A, B, seed=9)
    rng = np.random.RandomState(1)
    e2, dq = rng.randn(B, A).astype(F32), rng.randn(B, A).astype(F32)
    g = pr.sac_grad_reference(head, e2, e3, dq)
    assert (np.abs(sac_grad_emulate(head, e2, e3, dq) - g["d"]) <= g["b"]).all()


def test_gae_bound_holds_exactly():
    """a small rollout in exact rational arithmetic: the fp64 reference and the emulated scan (32 threads so that
    chunks, warps and carries all take part) are within the bound"""
    rng = np.random.RandomState(0)
    n = 200
    r, v = rng.randn(n), rng.randn(n).astype(F32)
    done = pc.gae_dones(n, "random", rng)
    ref = pr.gae_reference(r, v, done, 0.99, 0.95)
    g, gl = Fraction(0.99), Fraction(0.99) * Fraction(0.95)
    y, exact = Fraction(0), [None] * n
    for t in range(n - 1, -1, -1):
        nd = 0 if done[t] else 1
        vn = Fraction(float(v[t + 1])) if t + 1 < n else Fraction(0)
        y = Fraction(r[t]) + g * nd * vn - Fraction(float(v[t])) + gl * nd * y
        exact[t] = y
    exact = np.array([float(e) for e in exact])
    assert (np.abs(ref["adv"] - exact) <= ref["b_adv"]).all()
    emu = gae_emulate(r, v, done, float(Fraction(0.99)), 0.95, threads=64)
    assert (np.abs(emu - exact) <= ref["b_adv"]).all()


# ---- mutations: each named bug falls outside its tolerance --------------------------------------------------------------
def test_mutation_ppo_flipped_minimum_rule():
    """s1 >= s2 instead of s1 <= s2: samples above the range with a negative advantage lose their gradient"""
    inp = pc.ppo_inputs(6, 64, 0.2, seed=1)
    ref = pr.ppo_reference(*inp, 0.2, 0.0)
    with pytest.raises(AssertionError):
        pr.ppo_check(*ppo_emulate(*inp, 0.2, 0.0, flip_min=True), ref, "mutant")


def test_mutation_ppo_clip_gradient_always_passes():
    inp = pc.ppo_inputs(6, 64, 0.2, seed=1)
    ref = pr.ppo_reference(*inp, 0.2, 0.0)
    with pytest.raises(AssertionError, match="clipped sample"):
        pr.ppo_check(*ppo_emulate(*inp, 0.2, 0.0, clip_grad_passes=True), ref, "mutant")


def test_mutation_sac_open_in_range_mask():
    """a log-sigma mask open at the ends zeroes d log-sigma at exactly -20 and 2"""
    A, B = 6, 300
    head, e3 = pc.sac_inputs(A, B, seed=9)
    rng = np.random.RandomState(1)
    e2, dq = rng.randn(B, A).astype(F32), rng.randn(B, A).astype(F32)
    g = pr.sac_grad_reference(head, e2, e3, dq)
    bad = np.abs(sac_grad_emulate(head, e2, e3, dq, open_mask=True) - g["d"]) > g["b"]
    assert bad.any()


@pytest.mark.parametrize("bug", ["warp_bug", "drop_done"])
def test_mutation_gae(bug):
    """a carry taken past the next warp, or the (1 - done) factor dropped, leaves the bound"""
    rng = np.random.RandomState(3)
    n = 5000
    r, v = rng.randn(n), rng.randn(n).astype(F32)
    done = pc.gae_dones(n, "random", rng)
    ref = pr.gae_reference(r, v, done, 0.99, 0.95)
    good = gae_emulate(r, v, done, 0.99, 0.95, threads=128)
    assert (np.abs(good - ref["adv"]) <= ref["b_adv"]).all()
    mutant = gae_emulate(r, v, done, 0.99, 0.95, threads=128, **{bug: True})
    assert (np.abs(mutant - ref["adv"]) > ref["b_adv"]).any()


def test_mutation_td_targets_fp32_discount():
    """an fp32 discount on the done-aware path changes the bits of some targets"""
    rng = np.random.RandomState(0)
    B = 4096
    r, done, q = rng.randn(B), (rng.rand(B) < 0.2).astype(np.uint8), (rng.randn(B) * 30).astype(F32)
    want = pr.ac_td_targets(r, done, q, 0.99, 0, None)
    mutant = (r + (1.0 - done) * float(F32(0.99)) * q.astype(F64)).astype(F32)
    assert (mutant != want).any()


def test_mutation_finalize_fused_multiply_add():
    """count * mean^2 fused into the subtraction (one rounding) changes the std of a large-mean / small-variance
    column: what the explicit rounding in stats_finalize_kernel prevents"""
    rng = np.random.RandomState(0)
    diffs = 0
    for trial in range(20):
        x = (rng.randn(100000) * 0.3 + 1e3).astype(F32).astype(F64)
        s, q, count = x.sum(), (x * x).sum(), float(len(x))
        m, sd = pr.stats_finalize(np.array([s]), np.array([q]), count, 1e-2)
        fused = float(Fraction(q) - Fraction(count) * Fraction(float(m[0] * m[0])))
        sd_fma = math.sqrt(max(fused / max(count - 1, 1), 1e-2))
        diffs += sd_fma != sd[0]
    assert diffs > 0


def test_mutation_clip_drops_nan():
    """fmin(fmax(v, lo), hi) maps NaN to a bound; np.clip keeps it"""
    x = np.array([[np.nan, 1.0]], F32)
    o32, o64 = pr.stats_normalize(x, np.zeros(2), np.ones(2), -5.0, 5.0)
    assert np.isnan(o64[0, 0]) and np.isnan(o32[0, 0])
    assert not np.isnan(np.fmin(np.fmax(o64[0, 0], -5.0), 5.0))
    y = pr.ac_td_targets([0.0], [0], np.array([np.nan], F32), 0.99, 0, (-1.0, 1.0))
    assert np.isnan(y[0])


def test_min_seed_ties_and_signed_zero():
    q1 = np.array([1.0, 2.0, 0.0, -0.0, 3.0], F32)
    q2 = np.array([1.0, 1.0, -0.0, 0.0, 4.0], F32)
    d1, d2, qm = pr.sac_min_seed(q1, q2)
    s = F32(1) / F32(5)
    assert list(d1) == [s, 0, s, s, s] and list(d2) == [0, s, 0, 0, 0]
    assert np.array_equal(qm.view(np.uint32), q1[[0, 0, 2, 3, 4]].view(np.uint32)[[0, 0, 2, 3, 4]] * 0 +
                          np.array([q1[0], q2[1], q1[2], q1[3], q1[4]], F32).view(np.uint32))
    assert np.array_equal(pr.min2(q1, q2).view(np.uint32), qm.view(np.uint32))
