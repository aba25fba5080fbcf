"""Host references of the continuous-control head kernels and the rollout recurrences of include/coach_b200.h:
cb200_ppo_continuous_head, cb200_sac_policy_sample / _grad / _min_seed, cb200_min2, cb200_sub, cb200_f64_to_f32,
cb200_ac_td_targets, cb200_td3_smooth_actions, cb200_gae_scan, cb200_standardize, cb200_nstep_returns and
cb200_running_stats_push / _finalize / _normalize.  numpy (+ torch CPU for the gradients), importable without CUDA.

Two kinds of expectation:

* exact, where the header promises the reference's bits: the TD targets, the smoothed TD3 actions, the n-step returns,
  min / sub / casts, the SAC min seeds, the running-stats finalize (given sum, sumsq and count) and normalize.  These are
  the numpy expressions of oracle/rl_math.py, evaluated as numpy evaluates them;
* an fp64 evaluation plus a per-element bound, elsewhere.  Gradients come from torch fp64 autograd through
  torch.where, written with the reference's tie rules (tf.minimum sends the gradient to its first argument when
  x <= y, tf.clip_by_value passes it on the closed interval), not from the kernels' hand-derived formulas.  Each bound
  is built like head_ref.py's gamma_n S: S sums the absolute values of the terms of an output, and n counts the
  roundings and function errors on the longest path to it.  Where expf / logf / tanhf take part, their error is the
  maximum the CUDA Math API documents for sm_90 without fast math (CUDA C++ Programming Guide, "Mathematical
  Functions", single precision): expf 2 ulp, logf 1 ulp, tanhf 2 ulp.  An error of k ulp is at most 2 k u relative
  (u = 2^-24).  The error is then carried through each element's own condition number: the squash term
  log(1 - t^2 + 1e-6) and its derivative by about 1 / (1 - t^2 + 1e-6), the PPO ratio by |logp| + |logp_old|, the GAE
  scan by the number of affine compositions on the path.

tests/test_policy_ref_host.py pins this module to oracle/ and the fixtures, checks the bounds against high-precision
evaluations, and shows that plausible kernel bugs fall outside them.
"""
import math

import numpy as np
import torch

F32, F64 = np.float32, np.float64
U32 = 2.0 ** -24
U64 = 2.0 ** -53
ULP_EXPF, ULP_LOGF, ULP_TANHF = 2, 1, 2
LOG2PI = math.log(2.0 * math.pi)
PPO_EPS = float(F32(1e-15))                # `eps` of the PPO head, an fp32 constant of the graph
SAC_EPS = float(F32(1e-6))                 # squash-correction epsilon of the SAC head, fp32 in the graph
SAC_LS_MIN, SAC_LS_MAX = -20.0, 2.0
BLOCK_PPO, BLOCK_FLAT, BLOCK_GAE, BLOCK_STD, BLOCK_PUSH = 256, 256, 1024, 1024, 256


def gamma(n, u=U32):
    n = np.asarray(n, dtype=F64)
    return n * u / (1.0 - n * u)


def ulp_rel(k):
    """relative error of a result within k ulp"""
    return 2.0 * k * U32


def reduce_terms(n, threads):
    """additions on the longest path of the kernels' block sums: ceil(n / threads) strided terms per thread, then a
    tree over the threads"""
    return -(-int(n) // threads) + int(math.log2(threads))


def clip_where(x, lo, hi):
    """tf.clip_by_value: the gradient passes on the closed interval [lo, hi]"""
    return torch.where(x < lo, torch.full_like(x, lo), torch.where(x > hi, torch.full_like(x, hi), x))


def min_where(x, y):
    """tf.minimum's gradient rule: the first argument where x <= y"""
    return torch.where(x <= y, x, y)


# ---- PPO, continuous actions --------------------------------------------------------------------------------------------
def ppo_clip_range(clip_eps):
    """1 -+ clip_eps as the fp32 graph (and the kernel) rounds them"""
    e = F32(clip_eps)
    return float(F32(1) - e), float(F32(1) + e)


def ppo_reference(mu, logstd, actions, old_mu, old_logstd, adv, clip_eps, beta):
    """fp64 PPO head (heads/ppo_head.py) with torch autograd and the reference's tie rules, plus the bounds of the fp32
    kernel.  Returns a dict:
      ratio [B], pass_ [B] (the surrogate's gradient reaches the ratio: s1 <= s2, or the ratio lies in [lo, hi]),
      scalars [5] = (loss, KL(old||new), entropy, mean ratio, mean clipped ratio), d_mu [B, A], d_logstd [A];
      b_* the bounds of the same names, and either [B]: samples whose fp64 ratio lies within its bound of 1 -+ eps,
      whose branch the kernel may take either way."""
    t = lambda x: torch.tensor(np.asarray(x, F64))          # noqa: E731
    mu_t, ls_t = t(mu).requires_grad_(True), t(logstd).requires_grad_(True)
    a, omu, ols, adv_t = t(actions), t(old_mu), t(old_logstd), t(adv)
    B, A = mu_t.shape
    lo, hi = ppo_clip_range(clip_eps)
    beta = float(F32(beta))

    def logp_of(m, ls):
        sig = torch.exp(ls) + PPO_EPS
        z = (a - m) / sig
        return -0.5 * (z * z).sum(1) - torch.log(sig).sum() - 0.5 * A * LOG2PI, z, sig

    logp, z, sig = logp_of(mu_t, ls_t)
    logp_old, zo, osig = logp_of(omu, ols)
    ratio = torch.exp(logp - logp_old)
    cl = clip_where(ratio, lo, hi)
    surr = min_where(ratio * adv_t, cl * adv_t)
    entropy = 0.5 * A * (1.0 + LOG2PI) + torch.log(sig).sum()
    loss = -surr.mean() - beta * entropy
    d_mu, d_ls = torch.autograd.grad(loss, [mu_t, ls_t], retain_graph=True)
    d_mu_pass = torch.autograd.grad(-(ratio * adv_t).mean(), mu_t)[0]     # the branch where the gradient passes
    with torch.no_grad():
        rs = osig / sig
        dm = (mu_t - omu) / sig
        kl = (0.5 * (rs * rs + dm * dm - 1.0) - torch.log(rs)).sum(1)
        r, c = ratio, cl
        pass_ = (r * adv_t <= c * adv_t) | ((r >= lo) & (r <= hi))
    n = lambda x: x.detach().numpy()                          # noqa: E731
    r, c, z, zo, sig, osig, rs, dm = n(r), n(c), n(z), n(zo), n(sig), n(osig), n(rs), n(dm)
    out = dict(ratio=r, pass_=n(pass_), d_mu=n(d_mu), d_mu_pass=n(d_mu_pass), d_logstd=n(d_ls), logp=n(logp),
               logp_old=n(logp_old),
               scalars=np.array([float(x.detach()) for x in (loss, kl.mean(), entropy, ratio.mean(), cl.mean())]))
    # --- bounds.  sigma = expf(ls) + eps: 2 ulp + 1 rounding; z = (a - mu) / sigma: 2 more roundings; logp sums A
    # squares and A logs (logf: 1 ulp, plus sigma's relative error as an absolute error) in fp32
    e_sig = ulp_rel(ULP_EXPF) + U32
    e_z = e_sig + 2 * U32
    log_sig, log_osig = np.log(sig), np.log(osig)
    const = 0.5 * A * LOG2PI

    def err_logp(zz, lsig):
        s = 0.5 * zz.sum(1) + np.abs(lsig).sum() + const
        return gamma(A + 4) * s + (zz * e_z).sum(1) + (e_sig + ulp_rel(ULP_LOGF) * np.abs(lsig)).sum()

    e_delta = err_logp(z * z, log_sig) + err_logp(zo * zo, log_osig) + U32 * np.abs(out["logp"] - out["logp_old"])
    e_ratio = np.expm1(e_delta + ulp_rel(ULP_EXPF))          # relative error of the ratio (the condition |logp|+|logp_old|)
    b_ratio = r * e_ratio
    either = (np.abs(r - lo) <= b_ratio) | (np.abs(r - hi) <= b_ratio)
    aa = np.abs(np.asarray(adv, F64))
    # d_mu = -(1/B) adv ratio z / sigma
    b_dmu = np.abs(out["d_mu_pass"]) * (e_ratio[:, None] + e_z + e_sig + gamma(5))
    # d_logstd_j = sum_i -(1/B) adv_i ratio_i (z_ij^2 - 1) exp(ls_j) / sigma_j  -  beta exp(ls_j) / sigma_j; an
    # edge sample may contribute its term or not
    n_red = reduce_terms(B, BLOCK_PPO)
    t_ls = (aa * r / B)[:, None] * (z * z + 1.0)
    live = (out["pass_"] | either)[:, None]
    b_dls = (t_ls * live * (e_ratio[:, None] + 2 * e_z + 2 * e_sig + gamma(7))).sum(0) + \
        gamma(n_red) * (t_ls * live).sum(0) + (t_ls * either[:, None]).sum(0) * (1 + e_ratio.max()) + \
        abs(beta) * (2 * e_sig + gamma(4)) + U32 * np.abs(out["d_logstd"])
    # scalars
    s_ent = 0.5 * A * (1 + LOG2PI) + np.abs(log_sig).sum()
    b_ent = gamma(A + 3) * s_ent + (e_sig + ulp_rel(ULP_LOGF) * np.abs(log_sig)).sum()
    m = aa * np.maximum(r, c)
    b_loss = ((m * (e_ratio + U32)).sum() + gamma(n_red + 2) * (m * (1 + e_ratio)).sum()) / B + \
        abs(beta) * (b_ent + gamma(2) * s_ent) + U32 * abs(out["scalars"][0])
    s_kl = (0.5 * (rs * rs + dm * dm + 1.0) + np.abs(np.log(rs))).sum(1)
    e_kl = ((rs * rs + dm * dm) * (2 * e_z + 2 * e_sig + 2 * U32) + 2 * e_sig + U32).sum(1) + gamma(A + 4) * s_kl
    b_kl = (e_kl.sum() + gamma(n_red + 2) * (np.abs(n(kl)) + e_kl).sum()) / B
    b_mr = ((r * e_ratio).sum() + gamma(n_red + 2) * (r * (1 + e_ratio)).sum()) / B
    b_mcr = ((c * e_ratio).sum() + gamma(n_red + 2) * (c * (1 + e_ratio)).sum()) / B
    out.update(b_ratio=b_ratio, either=either, b_d_mu=b_dmu, b_d_logstd=b_dls,
               b_scalars=np.array([b_loss, b_kl, b_ent, b_mr, b_mcr]))
    return out


def ppo_check(got_dmu, got_dls, got_scalars, ref, name="ppo"):
    """the kernel's outputs against ppo_reference: a sample whose branch is fixed is checked on it (the d_mu row of a
    clipped sample is exactly 0); an edge sample's row may match the pass branch or be exactly 0"""
    d = np.abs(np.asarray(got_dmu, F64) - ref["d_mu_pass"])
    either, pas = ref["either"], ref["pass_"]
    clipped = ~pas & ~either
    assert (got_dmu[clipped] == 0).all(), "%s: d_mu of a clipped sample is not exactly 0" % name
    inb = d <= ref["b_d_mu"]
    fixed = pas & ~either
    assert inb[fixed].all(), "%s: d_mu out of bound at %s" % (name, np.argwhere(~inb & fixed[:, None])[:3])
    assert (inb[either].all(1) | (got_dmu[either] == 0).all(1)).all(), "%s: d_mu of an edge sample" % name
    dls = np.abs(np.asarray(got_dls, F64) - ref["d_logstd"])
    assert (dls <= ref["b_d_logstd"]).all(), "%s: d_logstd out of bound: %s > %s" % (name, dls, ref["b_d_logstd"])
    ds = np.abs(np.asarray(got_scalars, F64) - ref["scalars"])
    assert (ds <= ref["b_scalars"]).all(), "%s: scalars out of bound: %s > %s" % (name, ds, ref["b_scalars"])


# ---- SAC policy head ----------------------------------------------------------------------------------------------------
def _tanh_err(t, err_u):
    """tanhf of an argument with absolute error err_u: the derivative 1 - t^2 times err_u, plus 2 ulp"""
    return (1.0 - t * t) * err_u + ulp_rel(ULP_TANHF) * np.abs(t)


def sac_sample_reference(head, eps):
    """fp64 SACPolicyHead sample (heads/sac_head.py): raw u, action tanh(u), logp; and their bounds b_raw, b_act,
    b_logp.  head [B, 2A] = [mu | raw log sigma], eps [B, A]."""
    h, e = np.asarray(head, F64), np.asarray(eps, F64)
    A = e.shape[1]
    mu, lsr = h[:, :A], h[:, A:]
    ls = np.clip(lsr, SAC_LS_MIN, SAC_LS_MAX)
    sig = np.exp(ls)
    u = mu + sig * e
    t = np.tanh(u)
    w = 1.0 - t * t + SAC_EPS
    terms = -0.5 * e * e - ls - 0.5 * LOG2PI - np.log(w)
    # u = mu + expf(ls) * eps: 2 ulp of sigma, the product and the sum
    err_u = np.abs(sig * e) * (ulp_rel(ULP_EXPF) + U32) + U32 * (np.abs(u) + np.abs(sig * e))
    err_t = _tanh_err(t, err_u)
    # w = 1 - t^2 + 1e-6: t's error through 2|t|, three roundings; log w: 1 ulp plus w's relative error, which the
    # squash term amplifies by 1 / w
    err_w = 2 * np.abs(t) * err_t + U32 * (t * t + np.abs(1 - t * t) + w)
    rel_w = np.minimum(err_w / w, 0.999999)
    err_term = -np.log1p(-rel_w) + ulp_rel(ULP_LOGF) * np.abs(np.log(w)) + \
        gamma(3) * (0.5 * e * e + np.abs(ls) + 0.5 * LOG2PI)
    b_logp = err_term.sum(1) + gamma(A + 1) * np.abs(terms).sum(1)
    return dict(raw=u, act=t, logp=terms.sum(1), b_raw=err_u, b_act=err_t, b_logp=b_logp, in_range=(
        (lsr >= SAC_LS_MIN) & (lsr <= SAC_LS_MAX)))


def sac_grad64(head, eps_lp, eps_q, dq_da):
    """d/d head of  mean_b logp(eps_lp) - sum_b <dq_da_b, tanh(mu + sigma eps_q)_b>  with torch fp64 autograd, the
    log-sigma clip through clip_where (closed interval)"""
    h = torch.tensor(np.asarray(head, F64), requires_grad=True)
    e2, e3, dq = (torch.tensor(np.asarray(x, F64)) for x in (eps_lp, eps_q, dq_da))
    B, A = e2.shape
    mu, ls = h[:, :A], clip_where(h[:, A:], SAC_LS_MIN, SAC_LS_MAX)
    u2 = mu + torch.exp(ls) * e2
    # the Gaussian term of the reparameterised sample, (u2 - mu) / sigma = eps exactly: written with eps, since
    # u2 - mu cancels in fp64 when |mu| >> sigma
    logp = (-0.5 * e2 * e2 - ls - 0.5 * LOG2PI).sum(1) - torch.log(1 - torch.tanh(u2) ** 2 + SAC_EPS).sum(1)
    a3 = torch.tanh(mu + torch.exp(ls) * e3)
    obj = logp.mean() - (dq * a3).sum()
    return torch.autograd.grad(obj, h)[0].numpy()


def sac_grad_reference(head, eps_lp, eps_q, dq_da):
    """sac_grad64 and the per-element bound of the fp32 kernel, b [B, 2A]; in_range [B, A]"""
    h = np.asarray(head, F64)
    e2, e3, dq = (np.asarray(x, F64) for x in (eps_lp, eps_q, dq_da))
    B, A = e2.shape
    mu, lsr = h[:, :A], h[:, A:]
    ls = np.clip(lsr, SAC_LS_MIN, SAC_LS_MAX)
    sig = np.exp(ls)
    inv_b = 1.0 / B
    e_sig = ulp_rel(ULP_EXPF)

    def branch(e):
        u = mu + sig * e
        t = np.tanh(u)
        err_u = np.abs(sig * e) * (e_sig + U32) + U32 * (np.abs(u) + np.abs(sig * e))
        return t, _tanh_err(t, err_u)

    t2, et2 = branch(e2)
    t3, et3 = branch(e3)
    w0 = 1.0 - t2 * t2
    w = w0 + SAC_EPS
    gp = -2.0 * t2 * w0 / w                                   # d/du log(1 - t^2 + eps)
    dgp_dt = -2.0 * w0 / w + 4.0 * t2 * t2 * SAC_EPS / (w * w)
    dgp_dw0 = -2.0 * t2 * SAC_EPS / (w * w)
    err_gp = np.abs(dgp_dt) * et2 + np.abs(dgp_dw0) * U32 * (t2 * t2 + np.abs(w0)) + gamma(4) * np.abs(gp)
    w3 = 1.0 - t3 * t3
    err_w3 = 2 * np.abs(t3) * et3 + U32 * (t3 * t3 + np.abs(w3))
    b_mu = inv_b * (err_gp + gamma(2) * np.abs(gp)) + np.abs(dq) * err_w3 + \
        gamma(2) * (inv_b * np.abs(gp) + np.abs(dq * w3))
    se2, se3 = np.abs(sig * e2), np.abs(sig * e3)
    b_ls = inv_b * (se2 * err_gp + np.abs(gp) * se2 * (e_sig + gamma(3)) + U32) + \
        se3 * (np.abs(dq) * err_w3 + np.abs(dq * w3) * (e_sig + gamma(3))) + \
        gamma(3) * (inv_b * (1.0 + np.abs(gp) * se2) + np.abs(dq * w3) * se3)
    in_range = (lsr >= SAC_LS_MIN) & (lsr <= SAC_LS_MAX)
    return dict(d=sac_grad64(head, eps_lp, eps_q, dq_da), b=np.concatenate([b_mu, b_ls], 1), in_range=in_range)


def sac_min_seed(q1, q2):
    """(d1, d2, qmin): the seed float32(1) / float32(B) goes to q1 where q1 <= q2 (tf.minimum's gradient), else to q2;
    qmin = q2 where q2 < q1, else q1 (std::min, what tf.minimum evaluates)"""
    q1, q2 = np.asarray(q1, F32), np.asarray(q2, F32)
    s = F32(1) / F32(len(q1))
    first = q1 <= q2
    z = F32(0)
    return np.where(first, s, z).astype(F32), np.where(first, z, s).astype(F32), np.where(q2 < q1, q2, q1)


def min2(a, b):
    """tf.minimum's value (std::min): b where b < a, else a"""
    a, b = np.asarray(a, F32), np.asarray(b, F32)
    return np.where(b < a, b, a)


# ---- bit-exact glue -----------------------------------------------------------------------------------------------------
def ac_td_targets(rewards, game_overs, q_next, discount, ignore_done, clip):
    """the numpy expression of the reference (oracle/rl_math.py), rounded once to fp32 as the train op's placeholder
    does; q_next [B] fp32"""
    from oracle import rl_math as orm
    y = orm.ac_td_targets(rewards, game_overs, np.asarray(q_next, F32), discount, clip=clip,
                          use_non_zero_discount_for_terminal_states=bool(ignore_done))
    return y.reshape(-1).astype(F32)


def td3_smooth(actions, noise, noise_clip, lo, hi):
    from oracle import rl_math as orm
    return orm.td3_smooth_actions(np.asarray(actions, F32), noise, noise_clip, lo, hi).astype(F32)


def nstep_returns(rewards, lens, discount, n_step):
    """Episode.update_discounted_rewards per episode, episodes back to back"""
    from oracle import rl_math as orm
    out, o = [], 0
    for L in lens:
        out.append(orm.n_step_returns(rewards[o:o + L], discount, n_step))
        o += L
    return np.concatenate(out)


def stats_finalize(s, q, count, epsilon):
    """NumpySharedRunningStats.push's mean / std expression given sum, sumsq and count"""
    mean = s / count
    std = np.sqrt(np.maximum((q - count * np.square(mean)) / np.maximum(count - 1, 1), epsilon))
    return mean, std


def stats_normalize(x, mean, std, lo, hi):
    """(fp32, fp64) of np.clip((x - mean) / (std + 1e-15), lo, hi)"""
    v = np.clip((np.asarray(x, F32).astype(F64) - mean) / (std + 1e-15), lo, hi)
    return v.astype(F32), v


# ---- fp64 recurrences with bounds ---------------------------------------------------------------------------------------
def gae_reference(rewards, values, dones, discount, lam):
    """one reverse recurrence over the whole rollout, A_t = delta_t + gl (1 - d_t) A_{t+1}, delta_t = r_t +
    discount (1 - d_t) V_{t+1} - V_t (V_n = 0): what fill_advantages computes episode by episode.  Returns adv, tgt,
    n_valid and the bounds b_adv, b_tgt.  The kernel reaches A_t through a chunk of ceil(n / 1024) steps, 5 shuffle
    levels, up to 31 warp carries and the exclusive shift: k affine compositions of two fp64 roundings each, applied
    to S_t, the same recurrence on the absolute values of the terms."""
    r = np.asarray(rewards, F64)
    v = np.asarray(values, F32).astype(F64)
    nd = 1.0 - np.asarray(dones, bool)
    n = len(r)
    gl = discount * lam
    vnext = np.append(v[1:], 0.0)
    delta = r + discount * nd * vnext - v
    s_delta = np.abs(r) + discount * nd * np.abs(vnext) + np.abs(v)
    c = (gl * nd).tolist()
    dl, sd = delta.tolist(), s_delta.tolist()
    adv, S = [0.0] * n, [0.0] * n
    y = s = 0.0
    for i in range(n - 1, -1, -1):
        y = dl[i] + c[i] * y
        s = sd[i] + c[i] * s
        adv[i], S[i] = y, s
    adv, S = np.array(adv), np.array(S)
    k = -(-n // BLOCK_GAE) + 5 + 31 + 2
    b_adv = gamma(2 * k + 4, U64) * S
    last = np.flatnonzero(np.asarray(dones, bool))
    n_valid = int(last[-1]) + 1 if len(last) else 0
    tgt = adv + v
    return dict(adv=adv, tgt=tgt, n_valid=n_valid, b_adv=b_adv, b_tgt=b_adv + U64 * (np.abs(tgt) + S + np.abs(v)))


def standardize_reference(x, n_valid):
    """(out, mean, std, b_out, b_mean, b_std): exact-rounded mean and population std of x[:nv] (math.fsum), nv =
    min(n, n_valid) (n_valid None: n); out[nv:] is NaN.  nv = 0: mean 0, std 1.  The kernel sums ceil(nv / 1024)
    strided terms per thread and then a 10-level tree."""
    x = np.asarray(x, F64)
    n = len(x)
    nv = n if n_valid is None else max(0, min(n, int(n_valid)))
    out = np.full(n, np.nan)
    if nv == 0:
        return out, 0.0, 1.0, np.zeros(n), 0.0, 0.0
    xv = x[:nv]
    mean = math.fsum(xv) / nv
    d = xv - mean
    ss = math.fsum(d * d)
    std = math.sqrt(ss / nv)
    k = reduce_terms(nv, BLOCK_STD)
    b_mean = gamma(k + 1, U64) * math.fsum(np.abs(xv)) / nv
    e_ss = gamma(k + 3, U64) * (ss + nv * b_mean ** 2) + nv * b_mean ** 2 + 2 * nv * U64 * abs(mean) * b_mean
    rel_std = (0.5 * e_ss / ss + gamma(2, U64)) if ss > 0 else np.inf
    b_std = std * rel_std if ss > 0 else 0.0
    with np.errstate(invalid="ignore", divide="ignore"):
        out[:nv] = d / std
        b_out = np.zeros(n)
        b_out[:nv] = np.abs(out[:nv]) * (rel_std + gamma(2, U64)) + b_mean / std
    return out, mean, std, b_out, b_mean, b_std


def push_reference(x, sum0, sumsq0):
    """column sums of x and x^2 added to sum0 / sumsq0 (exact-rounded, math.fsum), and their bounds: each thread
    sums ceil(rows / 256) rows, an 8-level tree, one add to the running sum.  x^2 of an fp32 value is exact in fp64."""
    x = np.asarray(x, F32).astype(F64)
    rows, cols = x.shape
    s = np.array([math.fsum(np.append(x[:, j], sum0[j])) for j in range(cols)])
    q = np.array([math.fsum(np.append(x[:, j] ** 2, sumsq0[j])) for j in range(cols)])
    k = gamma(reduce_terms(rows, BLOCK_PUSH) + 1, U64)
    return s, q, k * (np.abs(x).sum(0) + np.abs(sum0)), k * ((x * x).sum(0) + np.abs(sumsq0))
