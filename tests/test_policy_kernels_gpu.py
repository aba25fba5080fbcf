"""The continuous-control head kernels and the rollout recurrences at the C ABI against tests/policy_ref.py, at the
shapes and edges of tests/policy_cases.py:

  (a) cb200_ppo_continuous_head: every regime of the clipped surrogate, all five scalars, d_mu and d_logstd within
      their fp64 bounds; an exact probe; repeat calls give the same bits;
  (b) cb200_sac_policy_sample / _grad: the log-sigma clip at and one ulp beyond its ends, saturated tanh, NULL outputs;
  (c) cb200_sac_min_seed, cb200_min2, cb200_sub, cb200_f64_to_f32, cb200_ac_td_targets, cb200_td3_smooth_actions,
      cb200_nstep_returns, cb200_running_stats_finalize / _normalize: bit for bit across block edges;
  (d) cb200_gae_scan, cb200_standardize, cb200_running_stats_push: within fp64 bounds, done flags on chunk and warp
      edges, n_valid exact;
  (e) the contract: argument errors write nothing, launch counts, and a final check that every regime ran."""
import ctypes

import numpy as np
import pytest
import torch

import policy_cases as pc
import policy_ref as pr
from abi_util import Outs, _dev, _lib, _ptr, assert_bits

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
RAN = set()


ALIVE = []                                   # device inputs of the call being made (see d())


def call(name, *args):
    """one call through the C ABI; every entry point here is one launch"""
    L, lib = _lib()
    c0 = lib.cb200_launch_count()
    L.check(getattr(lib, name)(*(args + (L.current_stream(),))))
    assert lib.cb200_launch_count() - c0 == 1, "%s: launch count" % name
    torch.cuda.synchronize()
    del ALIVE[:]


def d(x):
    """a device copy of x that stays allocated until the next call() returns, so that `_ptr(d(x))` can be passed
    inline (the caching allocator would otherwise hand its memory to the next input)"""
    t = _dev(np.ascontiguousarray(x))
    ALIVE.append(t)
    return t


# ---- (a) PPO ------------------------------------------------------------------------------------------------------------
def run_ppo(mu, ls, act, omu, ols, adv, eps, beta):
    B, A = mu.shape
    o = Outs()
    args = [d(x) for x in (mu, ls, act, omu, ols, adv)]
    p_dmu, p_dls, p_sc = o.add("d_mu", (B, A)), o.add("d_logstd", (A,)), o.add("scalars", (5,))
    call("cb200_ppo_continuous_head", *[_ptr(t) for t in args], B, A, eps, beta, p_dmu, p_dls, p_sc)
    return o.numpy()


@pytest.mark.parametrize("A", pc.PPO_A)
@pytest.mark.parametrize("B", pc.PPO_B)
def test_ppo_head(A, B):
    for eps, beta in ((0.1, 0.0), (0.2, 0.01)) if B != 1000 else [(e, b) for e in pc.PPO_EPS for b in pc.PPO_BETA]:
        inp = pc.ppo_inputs(A, B, eps, seed=A * 1000 + B)
        ref = pr.ppo_reference(*inp, eps, beta)
        lo, hi = pr.ppo_clip_range(eps)
        for reg in pc.ppo_regime(ref["ratio"], inp[5], lo, hi):
            RAN.add(("ppo", reg))
        if ref["either"].any():
            RAN.add(("ppo", "edge"))
        got = run_ppo(*inp, eps, beta)
        pr_name = "ppo A=%d B=%d eps=%g beta=%g" % (A, B, eps, beta)
        pr.ppo_check(got["d_mu"], got["d_logstd"], got["scalars"], ref, pr_name)
        again = run_ppo(*inp, eps, beta)
        for k in got:
            assert_bits(again[k], got[k], "%s repeat %s" % (pr_name, k))


def test_ppo_edge_samples():
    """ratios placed on the fp32 clip bounds (logstd = old logstd, mu moved along one component so that the fp64
    ratio is 1 -+ eps up to rounding): either branch is accepted there, every other check holds"""
    A, B, eps = 3, 64, 0.2
    mu, _, act, omu, ols, adv = pc.ppo_inputs(A, B, eps, seed=7)
    lo, hi = pr.ppo_clip_range(eps)
    osig = np.exp(ols.astype(F64)) + pr.PPO_EPS
    a64, om64 = act.astype(F64), omu.astype(F64)
    zo2 = ((a64[:, 0] - om64[:, 0]) / osig[0]) ** 2
    target = np.where(np.arange(B) % 2 == 0, lo, hi)
    mu = omu.copy()
    mu[:, 0] = (a64[:, 0] - np.sign(a64[:, 0] - om64[:, 0]) * osig[0] * np.sqrt(zo2 - 2 * np.log(target))).astype(F32)
    ref = pr.ppo_reference(mu, ols, act, omu, ols, adv, eps, 0.0)
    assert ref["either"].sum() >= B // 2
    RAN.add(("ppo", "edge"))
    got = run_ppo(mu, ols, act, omu, ols, adv, eps, 0.0)
    pr.ppo_check(got["d_mu"], got["d_logstd"], got["scalars"], ref, "ppo edge")


@pytest.mark.parametrize("A,B", [(1, 1), (6, 64), (32, 256), (17, 1024)])
def test_ppo_exact_probe(A, B):
    mu, ls, act, omu, ols, adv = pc.ppo_exact_inputs(A, B, seed=A + B)
    got = run_ppo(mu, ls, act, omu, ols, adv, 0.2, 0.0)
    RAN.add(("ppo", "exact"))
    z = (act.astype(F64) - mu)
    dlogp = -adv.astype(F64) / B
    assert_bits(got["d_mu"], (dlogp[:, None] * z).astype(F32), "ppo exact d_mu")
    assert_bits(got["d_logstd"], (dlogp[:, None] * (z * z - 1)).sum(0).astype(F32), "ppo exact d_logstd")
    sc = got["scalars"]
    assert sc[0] == F32(-adv.astype(F64).sum() / B), sc
    assert sc[1] == 0 and sc[3] == 1 and sc[4] == 1, sc


# ---- (b) SAC ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("A", pc.SAC_A)
@pytest.mark.parametrize("B", pc.SAC_B)
def test_sac_policy_sample_and_grad(A, B):
    head, eps = pc.sac_inputs(A, B, seed=A * 100 + B)
    ref = pr.sac_sample_reference(head, eps)
    o = Outs()
    p_raw, p_act, p_lp = o.add("raw", (B, A)), o.add("act", (B, A)), o.add("logp", (B,))
    dh, de = d(head), d(eps)
    call("cb200_sac_policy_sample", _ptr(dh), _ptr(de), B, A, p_raw, p_act, p_lp)
    got = o.numpy()
    for k in ("raw", "act", "logp"):
        err = np.abs(got[k].astype(F64) - ref[k])
        assert (err <= ref["b_" + k]).all(), "sac %s A=%d B=%d: worst %g" % (
            k, A, B, (err / np.maximum(ref["b_" + k], 1e-300)).max())
    lsr = head[:, A:]
    for name, m in (("ls_low", lsr == -20), ("ls_high", lsr == 2), ("ls_low_out", lsr < -20),
                    ("ls_high_out", lsr > 2), ("ls_inside", (lsr > -20) & (lsr < 2)),
                    ("saturated", np.abs(ref["raw"]) > 9)):
        if m.any():
            RAN.add(("sac", name))
    rng = np.random.RandomState(B)
    e2, e3 = rng.randn(B, A).astype(F32), eps
    dq = rng.randn(B, A).astype(F32)
    gr = pr.sac_grad_reference(head, e2, e3, dq)
    o = Outs()
    p = o.add("dz", (B, 2 * A))
    call("cb200_sac_policy_grad", _ptr(dh), _ptr(d(e2)), _ptr(d(e3)), _ptr(d(dq)), B, A, p)
    dz = o.numpy()["dz"]
    err = np.abs(dz.astype(F64) - gr["d"])
    assert (err <= gr["b"]).all(), "sac grad A=%d B=%d: worst %g at %s" % (
        A, B, (err / np.maximum(gr["b"], 1e-300)).max(), np.unravel_index(np.argmax(err - gr["b"]), err.shape))
    assert (dz[:, A:][~gr["in_range"]] == 0).all()


def test_sac_sample_null_outputs():
    """every combination of NULL outputs: the given outputs are the bits of the full call, nothing else is written"""
    A, B = 6, 257
    head, eps = pc.sac_inputs(A, B, seed=3)
    dh, de = d(head), d(eps)
    shapes = (("raw", (B, A)), ("act", (B, A)), ("logp", (B,)))
    full = None
    for mask in (7, 0, 1, 2, 3, 4, 5, 6):
        o = Outs()
        ptrs = [o.add(k, sh) if mask >> i & 1 else None for i, (k, sh) in enumerate(shapes)]
        call("cb200_sac_policy_sample", _ptr(dh), _ptr(de), B, A, *ptrs)
        got = o.numpy()                        # checks the canaries after every given output
        if full is None:
            full = got
        for k, v in got.items():
            assert_bits(v, full[k], "sac sample %s, output mask %d" % (k, mask))
    RAN.add(("sac", "null_outputs"))


def test_sac_grad_exact_out_of_range():
    """eps = 0 and log sigma outside [-20, 2]: d log-sigma is exactly +-0, d mu is the reference's"""
    A, B = 4, 300
    rng = np.random.RandomState(5)
    head = np.concatenate([rng.uniform(-1, 1, (B, A)), np.where(rng.rand(B, A) < 0.5, -25.0, 3.5)], 1).astype(F32)
    z = np.zeros((B, A), F32)
    dq = rng.randn(B, A).astype(F32)
    o = Outs()
    p = o.add("dz", (B, 2 * A))
    call("cb200_sac_policy_grad", _ptr(d(head)), _ptr(d(z)), _ptr(d(z)), _ptr(d(dq)), B, A, p)
    dz = o.numpy()["dz"]
    assert (dz[:, A:] == 0).all()
    RAN.add(("sac", "exact_out_of_range"))


# ---- (c) bit-exact glue -------------------------------------------------------------------------------------------------
def _pairs(n, rng):
    a = rng.randn(n).astype(F32)
    b = rng.randn(n).astype(F32)
    k = np.arange(n)
    b[k % 7 == 0] = a[k % 7 == 0]                    # ties
    a[k % 11 == 1], b[k % 11 == 1] = F32(0.0), F32(-0.0)
    a[k % 11 == 2], b[k % 11 == 2] = F32(-0.0), F32(0.0)
    return a, b


@pytest.mark.parametrize("n", pc.FLAT_N)
def test_min_sub_seed_bits(n):
    rng = np.random.RandomState(n)
    a, b = _pairs(n, rng)
    da, db = d(a), d(b)
    o = Outs()
    p_min, p_sub = o.add("min", (n,)), o.add("sub", (n,))
    p1, p2, pq = o.add("d1", (n,)), o.add("d2", (n,)), o.add("qmin", (n,))
    call("cb200_min2", _ptr(da), _ptr(db), n, p_min)
    call("cb200_sub", _ptr(da), _ptr(db), n, p_sub)
    call("cb200_sac_min_seed", _ptr(da), _ptr(db), n, p1, p2, pq)
    got = o.numpy()
    assert_bits(got["min"], pr.min2(a, b), "min2")
    assert_bits(got["sub"], a - b, "sub")
    w1, w2, wq = pr.sac_min_seed(a, b)
    assert_bits(got["d1"], w1, "seed d1")
    assert_bits(got["d2"], w2, "seed d2")
    assert_bits(got["qmin"], wq, "seed qmin")
    for mask in range(7):                           # NULL outputs: the given ones are the same bits
        o2 = Outs()
        ptrs = [o2.add(k, (n,)) if mask >> i & 1 else None for i, k in enumerate(("d1", "d2", "qmin"))]
        call("cb200_sac_min_seed", _ptr(da), _ptr(db), n, *ptrs)
        for k, v in o2.numpy().items():
            assert_bits(v, got[k], "seed %s mask %d" % (k, mask))
    RAN.update({("glue", "ties"), ("glue", "signed_zero")})


@pytest.mark.parametrize("n", [21, 257, 65537])
def test_f64_to_f32_bits(n):
    rng = np.random.RandomState(n)
    x = rng.randn(n) * 10.0 ** rng.randint(-45, 39, n)
    sp = pc.f32_specials()
    x[:len(sp) if n >= len(sp) else n] = sp[:n]
    o = Outs()
    p = o.add("y", (n,))
    call("cb200_f64_to_f32", _ptr(d(x)), n, p)
    with np.errstate(over="ignore"):
        want = x.astype(F32)
    y = o.numpy()["y"]
    nan = np.isnan(want)
    assert np.isnan(y[nan]).all()
    assert_bits(y[~nan], want[~nan], "f64_to_f32")
    RAN.update({("glue", "overflow"), ("glue", "subnormal"), ("glue", "ties_even")})


@pytest.mark.parametrize("ld_q", [1, 2, 5])
@pytest.mark.parametrize("B", [1, 255, 257, 65537])
def test_ac_td_targets_bits(ld_q, B):
    rng = np.random.RandomState(B * 10 + ld_q)
    r = rng.randn(B) * 3
    done = (rng.rand(B) < 0.3).astype(np.uint8)
    q = (rng.randn(B, ld_q) * 20).astype(F32)
    q[::97, 0] = np.nan
    dr, dd, dq = d(r), d(done), d(q)
    for ignore_done in (0, 1):
        for clip in (None, (-15.0, 10.0)):
            o = Outs()
            p = o.add("y", (B,))
            call("cb200_ac_td_targets", _ptr(dr), _ptr(dd), _ptr(dq), ld_q, B, 0.99, ignore_done,
                 int(clip is not None), *(clip or (0.0, 0.0)), p)
            y = o.numpy()["y"]
            want = pr.ac_td_targets(r, done, q[:, 0], 0.99, ignore_done, clip)
            nan = np.isnan(want)
            assert np.isnan(y[nan]).all(), "a NaN q_next must give a NaN target (clip=%s)" % (clip,)
            assert_bits(y[~nan], want[~nan], "td targets ld_q=%d ignore=%d clip=%s" % (ld_q, ignore_done, clip))
            RAN.update({("td", "ld%d" % ld_q), ("td", "nan")})
            if clip:
                RAN.add(("td", "clip"))
            if ignore_done:
                RAN.add(("td", "ignore_done"))


@pytest.mark.parametrize("n", [1, 255, 257, 65537])
def test_td3_smooth_bits(n):
    rng = np.random.RandomState(n)
    a = rng.uniform(-1.2, 1.2, n).astype(F32)
    a[::5] = np.where(np.arange(len(a[::5])) % 2 == 0, F32(1), F32(-1))     # on the bounds
    a[3::97] = np.nan
    noise = rng.randn(n) * 0.4
    noise[1::13] = np.where(np.arange(len(noise[1::13])) % 2 == 0, 0.5, -0.5)
    da = d(a)
    call("cb200_td3_smooth_actions", _ptr(da), _ptr(d(noise)), n, 0.5, -1.0, 1.0)
    got = da.cpu().numpy()
    want = pr.td3_smooth(a, noise, 0.5, -1.0, 1.0)
    nan = np.isnan(want)
    assert np.isnan(got[nan]).all()
    assert_bits(got[~nan], want[~nan], "td3 smooth")


@pytest.mark.parametrize("n_step", [1, 3, -1, 400])
@pytest.mark.parametrize("discount", [0.0, 0.99, 1.0])
def test_nstep_returns_bits(n_step, discount):
    rng = np.random.RandomState(abs(n_step))
    lens = [1, 5, 1, 300, 17, 1, 260]
    n = sum(lens)
    r = rng.randn(n)
    starts = np.repeat(np.cumsum([0] + lens[:-1]), lens).astype(np.int64)
    ends = np.repeat(np.cumsum(lens), lens).astype(np.int64)
    o = Outs(); p = o.add("out", (n,), torch.float64)                                  # noqa: E702
    call("cb200_nstep_returns", _ptr(d(r)), _ptr(d(starts)), _ptr(d(ends)), n, discount, n_step, p)
    assert_bits(o.numpy()["out"], pr.nstep_returns(r, lens, discount, n_step), "nstep")
    RAN.update({("nstep", "len1"), ("nstep", {1: "n1", 3: "n3", -1: "to_end", 400: "beyond"}[n_step]),
                ("nstep", {0.0: "d0", 1.0: "d1", 0.99: "n3"}[discount])})


# ---- (d) running statistics ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 255, 256, 257, 131072])
@pytest.mark.parametrize("cols", [1, 17, 300])
def test_running_stats(rows, cols):
    if rows * cols > 131072 * 17:
        rows = 4096
    rng = np.random.RandomState(rows + cols)
    loc = rng.uniform(-3, 3, cols)
    loc[0] = 1e3                                    # large mean, small variance
    scale = np.full(cols, 2.0)
    scale[0] = 0.3
    if cols > 1:
        scale[1] = 0.0                              # a constant column hits the epsilon floor
    x1 = (rng.randn(rows, cols) * scale + loc).astype(F32)
    x2 = (rng.randn(rows, cols) * scale + loc).astype(F32)
    eps = 1e-2
    s0, q0 = np.zeros(cols), np.full(cols, eps)
    ds, dq = d(s0), d(q0)
    call("cb200_running_stats_push", _ptr(d(x1)), rows, cols, _ptr(ds), _ptr(dq))
    s1, q1, bs1, bq1 = pr.push_reference(x1, s0, q0)
    assert (np.abs(ds.cpu().numpy() - s1) <= bs1).all() and (np.abs(dq.cpu().numpy() - q1) <= bq1).all()
    g1s, g1q = ds.cpu().numpy(), dq.cpu().numpy()
    call("cb200_running_stats_push", _ptr(d(x2)), rows, cols, _ptr(ds), _ptr(dq))
    s2, q2, bs2, bq2 = pr.push_reference(x2, g1s, g1q)
    assert (np.abs(ds.cpu().numpy() - s2) <= bs2).all() and (np.abs(dq.cpu().numpy() - q2) <= bq2).all()
    RAN.add(("stats", "two_pushes"))
    gs, gq = ds.cpu().numpy(), dq.cpu().numpy()
    for count in (eps + 2 * rows, 0.5, 1.0):
        o = Outs()
        pm, psd = o.add("mean", (cols,), torch.float64), o.add("std", (cols,), torch.float64)
        call("cb200_running_stats_finalize", _ptr(ds), _ptr(dq), count, eps, cols, pm, psd)
        got = o.numpy()
        wm, wsd = pr.stats_finalize(gs, gq, count, eps)
        assert_bits(got["mean"], wm, "finalize mean count=%g" % count)
        assert_bits(got["std"], wsd, "finalize std count=%g" % count)
        if count <= 1:
            RAN.add(("stats", "count_le_1"))
    RAN.add(("stats", "large_mean"))
    if (wsd == np.sqrt(eps)).any():
        RAN.add(("stats", "eps_floor"))
    # normalize with the count = 2 rows statistics, a NaN observation, both outputs and each alone
    wm, wsd = pr.stats_finalize(gs, gq, eps + 2 * rows, eps)
    xq = x2.copy()
    xq.flat[::7] = np.nan
    w32, w64 = pr.stats_normalize(xq, wm, wsd, -5.0, 5.0)
    dx, dm_, dsd = d(xq), d(wm), d(wsd)
    for which in (3, 1, 2):
        o = Outs()
        p32 = o.add("o32", (rows, cols)) if which & 1 else None
        p64 = o.add("o64", (rows, cols), torch.float64) if which & 2 else None
        call("cb200_running_stats_normalize", _ptr(dx), rows, cols, _ptr(dm_), _ptr(dsd), -5.0, 5.0, p32, p64)
        got = o.numpy()
        for k, w in (("o32", w32), ("o64", w64)):
            if k in got:
                nan = np.isnan(w)
                assert np.isnan(got[k][nan]).all(), "normalize: a NaN observation must stay NaN"
                assert_bits(got[k][~nan], w[~nan], "normalize %s" % k)
    RAN.add(("stats", "nan"))


# ---- (d) GAE and standardize --------------------------------------------------------------------------------------------
GAE_PATTERNS = {"random": None, "chunk_edges": ("chunk_first", "chunk_last"), "warp_edges": ("warp_first", "warp_last"),
                "all": ("all_done",), "none": ("none_done",), "first_only": ("first_only",)}


def run_gae(r, v, done, disc, lam, with_nvalid=True):
    n = len(r)
    o = Outs()
    pa, pt = o.add("adv", (n,), torch.float64), o.add("tgt", (n,), torch.float64)
    pn = o.add("nv", (1,), torch.int64) if with_nvalid else None
    call("cb200_gae_scan", _ptr(d(r)), _ptr(d(v)), _ptr(d(done)), n, disc, lam, pa, pt, pn)
    return o.numpy()


@pytest.mark.parametrize("n", pc.GAE_N)
def test_gae_scan(n):
    rng = np.random.RandomState(n % 100003)
    r = rng.randn(n)
    v = rng.randn(n).astype(F32)
    pats = list(GAE_PATTERNS) if n < 2 ** 21 else ["random", "warp_edges", "none"]
    for pat in pats:
        done = pc.gae_dones(n, pat, rng)
        for disc, lam in pc.GAE_GL if n < 2 ** 21 or pat == "random" else [(0.99, 0.95)]:
            ref = pr.gae_reference(r, v, done, disc, lam)
            got = run_gae(r, v, done, disc, lam)
            assert int(got["nv"][0]) == ref["n_valid"], (pat, got["nv"], ref["n_valid"])
            for k in ("adv", "tgt"):
                err = np.abs(got[k] - ref[k])
                assert (err <= ref["b_" + k]).all(), "gae %s n=%d %s gl=%g: worst %g" % (
                    k, n, pat, disc * lam, (err / np.maximum(ref["b_" + k], 1e-300)).max())
            for name in GAE_PATTERNS[pat] or ():
                RAN.add(("gae", name))
            RAN.add(("gae", "gl0" if lam == 0 else "gl1" if disc * lam == 1 else "random"))
    got = run_gae(r, v, done, 0.99, 0.95, with_nvalid=False)     # n_valid = NULL is accepted
    assert "nv" not in got


@pytest.mark.parametrize("n", pc.STD_N)
def test_standardize(n):
    rng = np.random.RandomState(n)
    x = rng.randn(n) * 3 + 2
    variants = [(None, "null"), (0, "zero"), (1, "one"), (n - 1, "n-1"), (n, "n"), (n + 5, "clamped")]
    for nv, name in variants:
        dx = d(x)
        dnv = None if nv is None else d(np.array([nv], np.int64))
        o = Outs()
        pms = o.add("ms", (2,), torch.float64)
        call("cb200_standardize", _ptr(dx), n, _ptr(dnv), pms)
        got = dx.cpu().numpy()
        ms = o.numpy()["ms"]
        want, m, sd, b_out, b_m, b_sd = pr.standardize_reference(x, nv)
        nan = np.isnan(want)
        assert np.isnan(got[nan]).all(), "standardize %s: NaN expected" % name
        assert (np.abs(got[~nan] - want[~nan]) <= b_out[~nan]).all(), "standardize %s n=%d" % (name, n)
        assert abs(ms[0] - m) <= b_m and (abs(ms[1] - sd) <= b_sd or (np.isnan(b_sd))), (name, ms, m, sd)
        RAN.add(("std", name))


# ---- (e) contract -------------------------------------------------------------------------------------------------------
def test_argument_errors_write_nothing():
    L, lib = _lib()
    o = Outs()
    f = d(np.ones(64, F32))
    f64 = d(np.ones(64, F64))
    u8 = d(np.zeros(64, np.uint8))
    i64 = d(np.zeros(64, np.int64))
    p32, p64 = o.add("f", (64,)), o.add("g", (64,), torch.float64)
    pf, pd, pu, pi = _ptr(f), _ptr(f64), _ptr(u8), _ptr(i64)
    s = L.current_stream()
    bad = [
        ("cb200_ppo_continuous_head", (pf, pf, pf, pf, pf, pf, 4, 0, 0.2, 0.0, p32, p32, p32, s)),
        ("cb200_ppo_continuous_head", (pf, pf, pf, pf, pf, pf, 1, 33, 0.2, 0.0, p32, p32, p32, s)),
        ("cb200_ppo_continuous_head", (pf, pf, pf, pf, pf, pf, 0, 2, 0.2, 0.0, p32, p32, p32, s)),
        ("cb200_ppo_continuous_head", (pf, pf, pf, pf, pf, None, 4, 2, 0.2, 0.0, p32, p32, p32, s)),
        ("cb200_sac_policy_sample", (pf, pf, 0, 2, p32, p32, p32, s)),
        ("cb200_sac_policy_sample", (pf, pf, 4, 0, p32, p32, p32, s)),
        ("cb200_sac_policy_sample", (None, pf, 4, 2, p32, p32, p32, s)),
        ("cb200_sac_policy_grad", (pf, pf, pf, pf, 0, 2, p32, s)),
        ("cb200_sac_policy_grad", (pf, pf, pf, None, 4, 2, p32, s)),
        ("cb200_sac_min_seed", (pf, pf, 0, p32, p32, p32, s)),
        ("cb200_sac_min_seed", (None, pf, 4, p32, p32, p32, s)),
        ("cb200_min2", (pf, pf, 0, p32, s)),
        ("cb200_sub", (pf, None, 4, p32, s)),
        ("cb200_f64_to_f32", (pd, 0, p32, s)),
        ("cb200_ac_td_targets", (pd, pu, pf, 0, 4, 0.99, 0, 0, 0.0, 0.0, p32, s)),
        ("cb200_ac_td_targets", (pd, pu, pf, 1, 0, 0.99, 0, 0, 0.0, 0.0, p32, s)),
        ("cb200_td3_smooth_actions", (None, pd, 4, 0.5, -1.0, 1.0, s)),
        ("cb200_gae_scan", (pd, pf, pu, 0, 0.99, 0.95, p64, p64, None, s)),
        ("cb200_gae_scan", (pd, pf, None, 4, 0.99, 0.95, p64, p64, None, s)),
        ("cb200_standardize", (p64, 0, None, None, s)),
        ("cb200_nstep_returns", (pd, pi, pi, 4, 0.99, 0, p64, s)),
        ("cb200_nstep_returns", (pd, pi, pi, 4, 0.99, -2, p64, s)),
        ("cb200_nstep_returns", (pd, pi, pi, 0, 0.99, 1, p64, s)),
        ("cb200_running_stats_push", (pf, 0, 4, p64, p64, s)),
        ("cb200_running_stats_finalize", (pd, pd, 0.0, 1e-2, 4, p64, p64, s)),
        ("cb200_running_stats_finalize", (pd, pd, 1.0, 1e-2, 0, p64, p64, s)),
        ("cb200_running_stats_normalize", (pf, 4, 4, pd, pd, -5.0, 5.0, None, None, s)),
        ("cb200_running_stats_normalize", (pf, 4, 4, None, pd, -5.0, 5.0, p32, None, s)),
    ]
    c0 = lib.cb200_launch_count()
    for name, args in bad:
        rc = getattr(lib, name)(*args)
        assert rc == -1, "%s%s returned %d" % (name, args[:-1], rc)
    assert lib.cb200_launch_count() == c0
    got = o.numpy()
    canary = np.array(0x7FA5A5A5, np.uint32)
    assert (got["f"].view(np.uint32) == canary).all(), "an argument error wrote an output"
    assert (got["g"].view(np.uint64) == np.array(0x7FF4A5A5A5A5A5A5, np.uint64)).all()


def test_every_policy_regime_was_run():
    missing = sorted(pc.REGIMES - RAN)
    assert not missing, "regimes never reached: %s" % missing
