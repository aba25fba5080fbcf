"""Shapes, inputs and regimes of the policy-head and recurrence kernel tests (tests/test_policy_kernels_gpu.py).
Every regime named in REGIMES must be reached by some case: the suite's last test checks it."""
import math

import numpy as np

import policy_ref as pr

F32, F64 = np.float32, np.float64

PPO_A = [1, 2, 6, 17, 31, 32]
PPO_B = [1, 7, 64, 255, 256, 257, 1000]
PPO_BETA = [0.0, 0.01]
PPO_EPS = [0.1, 0.2]
SAC_A = [1, 6, 17, 64]
SAC_B = [1, 255, 256, 257, 4097]
FLAT_N = [1, 255, 256, 257, 4097, 65537]
GAE_N = [1, 2, 31, 32, 33, 1023, 1024, 1025, 2047, 2049, 32 * 1024 - 1, 32 * 1024 + 1, 2 ** 21]
GAE_GL = [(0.99, 0.0), (0.99, 0.95), (1.0, 1.0)]
STD_N = [1, 2, 1000, 1024, 1025, 65537, 2 ** 21]

# PPO samples: inside the clip range, or the ratio above / below it with a positive / negative advantage
PPO_REGIMES = ["inside", "above_pos", "above_neg", "below_pos", "below_neg"]
REGIMES = set(
    [("ppo", r) for r in PPO_REGIMES] + [("ppo", "exact"), ("ppo", "edge")]
    + [("sac", r) for r in ("ls_low", "ls_high", "ls_low_out", "ls_high_out", "ls_inside", "saturated")]
    + [("sac", "null_outputs"), ("sac", "exact_out_of_range")]
    + [("gae", r) for r in ("chunk_first", "chunk_last", "warp_first", "warp_last", "all_done", "none_done",
                            "first_only", "gl0", "gl1")]
    + [("std", r) for r in ("null", "zero", "one", "n-1", "n", "clamped")]
    + [("nstep", r) for r in ("n1", "n3", "to_end", "beyond", "len1", "d0", "d1")]
    + [("td", r) for r in ("ld1", "ld2", "ld5", "clip", "ignore_done", "nan")]
    + [("stats", r) for r in ("large_mean", "count_le_1", "eps_floor", "nan", "two_pushes")]
    + [("glue", r) for r in ("ties", "signed_zero", "overflow", "subnormal", "ties_even")])


def ppo_regime(ratio, adv, lo, hi):
    """regime names of every sample from its fp64 ratio"""
    out = np.where((ratio >= lo) & (ratio <= hi), "inside", "")
    out = np.where(ratio > hi, np.where(adv > 0, "above_pos", "above_neg"), out)
    out = np.where(ratio < lo, np.where(adv > 0, "below_pos", "below_neg"), out)
    return out


def ppo_inputs(A, B, clip_eps, seed):
    """(mu, logstd, actions, old_mu, old_logstd, adv): the ratio of sample i is steered into regime i mod 5 by moving
    mu along the first action component; the log-stds differ from the old ones, so every term of the head is live.
    Target ratios keep at least clip_eps / 2 away from the clip bounds."""
    rng = np.random.RandomState(seed)
    old_ls = (rng.uniform(-0.7, 0.3, A)).astype(F32)
    ls = (old_ls + rng.uniform(-0.02, 0.02, A)).astype(F32)
    old_mu = rng.uniform(-1, 1, (B, A)).astype(F32)
    sig, osig = np.exp(ls.astype(F64)), np.exp(old_ls.astype(F64))
    d = rng.uniform(-1.0, 1.0, (B, A)) * osig
    d[:, 0] = np.where(rng.rand(B) < 0.5, -1, 1) * rng.uniform(3.0, 4.0, B) * osig[0]
    actions = (old_mu + d).astype(F32)
    adv = rng.uniform(0.1, 2.0, B) * np.where(rng.rand(B) < 0.5, -1, 1)
    target = np.empty(B)
    e = clip_eps
    for i in range(B):
        k = i % 5
        if k == 0:
            target[i] = rng.uniform(1 - e / 2, 1 + e / 2)
        elif k in (1, 2):
            target[i] = rng.uniform(1 + 1.5 * e, 2.5)
        else:
            target[i] = rng.uniform(0.3, 1 - 1.5 * e)
        if k in (1, 3):
            adv[i] = abs(adv[i])
        elif k in (2, 4):
            adv[i] = -abs(adv[i])
    # log ratio = base + component 0's quadratic term; solve for mu[:, 0] in fp64
    a64, om64 = actions.astype(F64), old_mu.astype(F64)
    zo2 = ((a64 - om64) / osig) ** 2
    base = -0.5 * (((a64[:, 1:] - om64[:, 1:]) / sig[1:]) ** 2).sum(1) + 0.5 * zo2[:, 1:].sum(1) \
        - np.log(sig).sum() + np.log(osig).sum()
    rhs = sig[0] ** 2 * (zo2[:, 0] - 2.0 * (np.log(target) - base))
    assert (rhs > 0).all()
    dd = np.sign(a64[:, 0] - om64[:, 0]) * np.sqrt(rhs)     # a - mu on component 0
    mu = old_mu.copy()
    mu[:, 0] = (a64[:, 0] - dd).astype(F32)
    return mu, ls, actions, old_mu, old_ls, adv.astype(F32)


def ppo_exact_inputs(A, B, seed):
    """logstd = old logstd = 0, mu = old mu, dyadic a - mu and advantages, B a power of two: the ratio is exactly 1,
    the KL 0, the mean (clipped) ratio 1, and d_mu, d_logstd are exact"""
    rng = np.random.RandomState(seed)
    mu = (rng.randint(-64, 64, (B, A)) / 16.0).astype(F32)
    actions = (mu + rng.randint(-32, 33, (B, A)) / 8.0).astype(F32)
    adv = (rng.randint(-16, 17, B) / 4.0).astype(F32)
    z = np.zeros(A, F32)
    return mu, z, actions, mu.copy(), z.copy(), adv


def sac_inputs(A, B, seed):
    """head [B, 2A], eps [B, A]: raw log sigma exactly at -20 and 2, one ulp outside each, well outside, and inside;
    some |u| up to about 12 (tanh saturates in fp32)"""
    rng = np.random.RandomState(seed)
    mu = rng.uniform(-1.5, 1.5, (B, A)).astype(F32)
    specials = np.array([-20.0, 2.0, np.nextafter(F32(-20), F32(-30)), np.nextafter(F32(2), F32(3)), -35.0, 6.0],
                        F32)
    lsr = rng.uniform(-3.0, 1.0, (B, A)).astype(F32)
    pick = rng.rand(B, A) < 0.4
    lsr[pick] = specials[rng.randint(0, len(specials), pick.sum())]
    eps = rng.randn(B, A).astype(F32)
    sat = rng.rand(B, A) < 0.1
    mu[sat] = (np.where(rng.rand(sat.sum()) < 0.5, -1, 1) * rng.uniform(9.0, 12.0, sat.sum())).astype(F32)
    eps[sat] = F32(0.0)
    return np.concatenate([mu, lsr], 1), eps


def gae_dones(n, pattern, rng):
    """done flags of one case; patterns place them on thread-chunk and warp edges of the 1024-thread scan"""
    per = -(-n // pr.BLOCK_GAE)
    d = np.zeros(n, np.uint8)
    if pattern == "random":
        d[rng.rand(n) < 0.05] = 1
        d[-1] = 1
    elif pattern == "chunk_edges":
        d[0::per] = 1                         # the first element of every chunk
        d[per - 1::per] = 1                   # the last element of every chunk
    elif pattern == "warp_edges":
        d[0::32 * per] = 1
        d[32 * per - 1::32 * per] = 1
        d[min(n - 1, 7 * 32 * per + 3)] = 1
    elif pattern == "all":
        d[:] = 1
    elif pattern == "first_only":
        d[0] = 1
    elif pattern != "none":
        raise ValueError(pattern)
    return d


def spread64(rng, n, scale=1.0):
    return rng.randn(n) * scale


def f32_specials():
    """values where a cast or a min goes wrong: the fp32 overflow threshold, subnormals, ties to even"""
    big = float(np.finfo(F32).max)
    half_ulp = 2.0 ** (127 - 24)
    sub = 2.0 ** -149
    return np.array([big, big + half_ulp * 0.99, big + half_ulp, -(big + half_ulp), 1e39, -np.inf, np.inf, np.nan,
                     sub, sub / 2, sub * 0.51, sub * 1.5, sub * 2.5, 2.0 ** -126 * (1 - 2.0 ** -24), 1.0 + 2.0 ** -24,
                     1.0 + 3 * 2.0 ** -24, 1.0 + 2.0 ** -24 + 2.0 ** -50, -0.0, 0.0, 1e-46, math.pi], F64)
