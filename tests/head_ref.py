"""Host references of the fused Q heads of include/coach_b200.h: cb200_dqn_head_fused (DQN / DDQN, MMC, PAL, persistent
PAL), cb200_ensemble_head_fused (Bootstrapped DQN) and cb200_c51_head (categorical).  numpy only, importable without
CUDA.

Every head has two evaluations:

* an fp32 emulation of the header's contract.  Where the header promises bits (the TD targets and td_err given the Q
  values, dL/dQ given Q and the targets, the C51 projection given the probabilities, the ensemble's fp32 rescale of the
  feature gradient) it takes the kernel's rounding steps one by one.  Elsewhere (dot products, batch sums) it sums in the
  kernel's order in fp32 (an FMA is emulated through an exact fp64 product, so up to a double rounding): its error is
  the yardstick the kernel's error is measured against;
* an fp64 evaluation, together with S, the sum of the absolute values of the terms of every output, for the bound
  |got - fp64| <= gamma_n S, gamma_n = n u / (1 - n u), u = 2^-24.

tests/test_head_ref_host.py pins this module to the reference agents' restatements (oracle/) and fixtures.
"""
import numpy as np

F32, F64 = np.float32, np.float64
U32 = 2.0 ** -24
TINY32 = 2.0 ** -126            # absolute floor for fp32 underflow (a softmax term e^-160 flushes to 0)

TARGET_DQN, TARGET_MMC, TARGET_PAL, TARGET_PAL_PERSISTENT = 0, 1, 2, 3
RULE_NAMES = {TARGET_DQN: "dqn", TARGET_MMC: "mmc", TARGET_PAL: "pal", TARGET_PAL_PERSISTENT: "pal_persistent"}
HEAD_ROWS, HEAD_WARPS = 2, 8     # rows per warp, warps per block of the DQN / ensemble head kernels


def gamma(n):
    n = np.asarray(n, dtype=F64)
    return n * U32 / (1.0 - n * U32)


def fma32(a, b, c):
    """fp32 fused multiply-add through an exact fp64 product (the fp64 add can round once more than an FMA)"""
    return (np.asarray(a, F64) * np.asarray(b, F64) + np.asarray(c, F64)).astype(F32)


# ---- Q values --------------------------------------------------------------------------------------------------------
def head_q32(h, w, bias):
    """head_dot: lane l accumulates features l + 32 j (j ascending) with FMAs, an xor butterfly folds the 32 lanes, then
    the bias is added.  h [B, K], w [K, A], bias [A] (fp32) -> [B, A] fp32"""
    B, K = h.shape
    A = w.shape[1]
    kpl = K // 32
    hl = np.asarray(h, F32).reshape(B, kpl, 32)
    wl = np.asarray(w, F32).reshape(kpl, 32, A)
    s = np.zeros((B, 32, A), F32)
    for j in range(kpl):
        s = fma32(hl[:, j, :, None], wl[None, j], s)
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        s = s + s[:, lanes ^ o]
    return s[:, 0] + np.asarray(bias, F32)


def head_q64(h, w, bias):
    """(fp64 Q, S) of h w + bias"""
    h64, w64, b64 = (np.asarray(x, F64) for x in (h, w, bias))
    return h64 @ w64 + b64, np.abs(h64) @ np.abs(w64) + np.abs(b64)


def dot_terms(K):
    """accumulation length of head_dot: K / 32 FMAs per lane, 5 butterfly adds, the bias"""
    return K // 32 + 6


# ---- TD targets ------------------------------------------------------------------------------------------------------
def rule_targets(rule, q_online, q_next, q_select, actions, rewards, game_overs, discount, q_target_s=None,
                 returns=None, alpha=0.0, rho=0.0):
    """The header's target contract, bit for bit given the fp32 Q values.  a* = first argmax of q_select (q_next when
    q_select is None: DQN); y = r + ((1 - done) discount) q_next[a*] in fp64; the rule's fp32 target replaces Q(s, a).
    A row whose action is outside [0, A) keeps Q(s) and gets td_err 0.  Returns (targets fp32 [B, A], td_err fp64 [B],
    a* [B])."""
    qo = np.asarray(q_online, F32)
    qn = np.asarray(q_next, F32)
    B, A = qo.shape
    rows = np.arange(B)
    sel = np.argmax(np.asarray(q_next if q_select is None else q_select, F32), axis=1)
    q_best = qn[rows, sel]
    not_done = 1.0 - np.asarray(game_overs, F64)
    y = np.asarray(rewards, F64) + (not_done * discount) * q_best.astype(F64)
    act = np.asarray(actions, np.int64)
    ok = (act >= 0) & (act < A)
    a = np.where(ok, act, 0)
    if rule == TARGET_DQN:
        ty = y.astype(F32)
        td = np.abs(y - qo[rows, a].astype(F64))
    elif rule == TARGET_MMC:
        R = np.asarray(returns, F64)
        ty = ((1.0 - rho) * y + rho * R).astype(F32)
        td = np.abs(ty.astype(F64) - qo[rows, a].astype(F64))
    else:
        qt = np.asarray(q_target_s, F32)
        R = np.asarray(returns, F64)
        adv = qt.max(axis=1) - qt[rows, a]                                    # fp32 array arithmetic
        nadv = qn.max(axis=1) - q_best
        m = np.where((rule == TARGET_PAL_PERSISTENT) & (nadv < adv), nadv, adv)
        t1 = y.astype(F32) - F32(alpha) * m
        t2 = F32(1.0 - rho) * t1
        ty = (t2.astype(F64) + rho * R).astype(F32)
        td = np.abs(ty.astype(F64) - qo[rows, a].astype(F64))
    targets = qo.copy()
    targets[rows[ok], a[ok]] = ty[ok]
    return targets, np.where(ok, td, 0.0), sel


# ---- loss and dL/dQ --------------------------------------------------------------------------------------------------
def loss_grad32(q_online, targets, weights, huber, B):
    """head_loss_grad: e = Q - target (fp32); Huber (delta 1) or squared error; dq = (w * (1 / B)) * l'(e), bit-exact
    (no additions, so nothing for the compiler to contract).  Returns (dq fp32 [B, A], row losses fp32 [B])"""
    qo, tg = np.asarray(q_online, F32), np.asarray(targets, F32)
    e = qo - tg
    if huber:
        ae = np.abs(e)
        qq = np.minimum(ae, F32(1))
        l = fma32(F32(0.5) * qq, qq, ae - qq)
        g = np.where(ae <= 1, e, np.where(e > 0, F32(1), F32(-1))).astype(F32)
    else:
        l = e * e
        g = F32(2) * e
    w = np.ones(qo.shape[0], F32) if weights is None else np.asarray(weights, F32)
    inv_b = F32(1) / F32(B)
    dq = (w * inv_b)[:, None] * g
    row = np.zeros(qo.shape[0], F32)
    for a in range(qo.shape[1]):
        row = row + l[:, a]
    return dq, row


def loss64(q_online, targets, weights, huber, B):
    """fp64 loss mean_b(w_b sum_a l(e)) of the given fp32 Q and targets -> (loss, S)"""
    e = np.asarray(q_online, F64) - np.asarray(targets, F64)
    ae = np.abs(e)
    l = np.where(ae <= 1, 0.5 * e * e, ae - 0.5) if huber else e * e
    w = np.ones(e.shape[0]) if weights is None else np.asarray(weights, F64)
    terms = w[:, None] * l / B
    return terms.sum(), np.abs(terms).sum()


def dq64(q_online, targets, weights, huber, B):
    e = np.asarray(q_online, F64) - np.asarray(targets, F64)
    g = np.clip(e, -1.0, 1.0) if huber else 2.0 * e
    w = np.ones(e.shape[0]) if weights is None else np.asarray(weights, F64)
    return w[:, None] * g / B


# ---- backward ----------------------------------------------------------------------------------------------------------
def _fold_partials32(parts):
    """dqn_head_reduce_kernel: 8 strided sums over the per-warp partials (q = w, w + 8, ...), folded in order"""
    P = parts.shape[0]
    pad = (-P) % HEAD_WARPS
    if pad:
        parts = np.concatenate([parts, np.zeros((pad,) + parts.shape[1:], F32)])
    parts = parts.reshape((-1, HEAD_WARPS) + parts.shape[1:])
    s = np.zeros(parts.shape[1:], F32)
    for q in range(parts.shape[0]):
        s = s + parts[q]
    out = s[0]
    for k in range(1, HEAD_WARPS):
        out = out + s[k]
    return out


def _row_pairs(x):
    """[B, ...] -> [warps, HEAD_ROWS, ...] with zero rows after the last one"""
    B = x.shape[0]
    pad = (-B) % HEAD_ROWS
    if pad:
        x = np.concatenate([x, np.zeros((pad,) + x.shape[1:], x.dtype)])
    return x.reshape((-1, HEAD_ROWS) + x.shape[1:])


def backward32(h, w, dq, row_loss, weights, B):
    """the head's backward pass in the kernel's order: per warp, dW += h dq by FMA and db += dq over its two rows, the
    loss partial w * row by FMA; the partials folded by the reduction; dh = (FMA chain over a of dq_a W[k, a]) masked
    with h > 0.  Returns dict(dw [K, A], db [A], loss, dh [B, K]) in fp32"""
    h, w, dq = np.asarray(h, F32), np.asarray(w, F32), np.asarray(dq, F32)
    K, A = w.shape
    hp, dp = _row_pairs(h), _row_pairs(dq)
    wt = np.ones(h.shape[0], F32) if weights is None else np.asarray(weights, F32)
    lp, wp = _row_pairs(np.asarray(row_loss, F32)), _row_pairs(wt)
    acc_w = np.zeros((hp.shape[0], K, A), F32)
    acc_b = np.zeros((hp.shape[0], A), F32)
    acc_l = np.zeros(hp.shape[0], F32)
    for rr in range(HEAD_ROWS):
        acc_w = fma32(hp[:, rr, :, None], dp[:, rr, None, :], acc_w)
        acc_b = acc_b + dp[:, rr]
        acc_l = fma32(wp[:, rr], lp[:, rr], acc_l)
    s = np.zeros((h.shape[0], K), F32)
    for a in range(A):
        s = fma32(dq[:, a, None], w[None, :, a], s)
    return dict(dw=_fold_partials32(acc_w), db=_fold_partials32(acc_b),
                loss=_fold_partials32(acc_l) * (F32(1) / F32(B)), dh=np.where(h > 0, s, F32(0)))


def backward64(h, w, dq):
    """fp64 dW = h^T dq, db = sum_b dq, dh = (dq W^T) [h > 0] of the given fp32 dq, each with S"""
    h64, w64, d64 = (np.asarray(x, F64) for x in (h, w, dq))
    mask = h64 > 0
    return dict(dw=(h64.T @ d64, np.abs(h64).T @ np.abs(d64)), db=(d64.sum(0), np.abs(d64).sum(0)),
                dh=(np.where(mask, d64 @ w64.T, 0.0), np.where(mask, np.abs(d64) @ np.abs(w64).T, 0.0)))


def dqn_head(rule, h_next, h_online, h_select, w_target, b_target, w_online, b_online, actions, rewards, game_overs,
             discount, weights=None, huber=True, h_target_s=None, returns=None, alpha=0.0, rho=0.0):
    """cb200_dqn_head_fused, fp32 emulation: every output of the descriptor (q_target_s only for PAL)"""
    B = h_online.shape[0]
    qn = head_q32(h_next, w_target, b_target)
    qo = head_q32(h_online, w_online, b_online)
    qs = head_q32(h_select, w_online, b_online) if h_select is not None else None
    qt = head_q32(h_target_s, w_target, b_target) if rule >= TARGET_PAL else None
    targets, td, sel = rule_targets(rule, qo, qn, qs, actions, rewards, game_overs, discount, qt, returns, alpha, rho)
    dq, row = loss_grad32(qo, targets, weights, huber, B)
    out = dict(q_online=qo, q_next=qn, q_select=qs, q_target_s=qt, targets=targets, td_err=td, dq=dq, sel=sel)
    out.update(backward32(h_online, w_online, dq, row, weights, B))
    return out


# ---- ensemble head ---------------------------------------------------------------------------------------------------
def ensemble_targets(q_online, q_next, q_select, actions, rewards, game_overs, masks, discount, H):
    """per head h (columns [h A, (h + 1) A)): the double-DQN target where masks[:, h] != 0, the online prediction
    elsewhere.  Returns (targets fp32 [B, H A], a* [B, H])"""
    qo = np.asarray(q_online, F32)
    A = qo.shape[1] // H
    targets = qo.copy()
    sels = []
    for h in range(H):
        c = slice(h * A, (h + 1) * A)
        t, _, sel = rule_targets(TARGET_DQN, qo[:, c], q_next[:, c], q_select[:, c], actions, rewards, game_overs,
                                 discount)
        use = np.asarray(masks)[:, h] != 0
        targets[use, c] = t[use]
        sels.append(sel)
    return targets, np.stack(sels, 1)


def ensemble_head(h_next, h_online, h_select, w_target, b_target, w_online, b_online, actions, rewards, game_overs,
                  masks, discount, H, huber=True, rescale=1.0):
    """cb200_ensemble_head_fused, fp32 emulation.  Per head the loss mean_b(sum_a l) and its partials like the DQN head;
    the losses summed in head order; dh = fp32(rescale * (sum over heads, in order, of each head's FMA chain)) masked
    with h > 0 -- the rescale in fp32 before the plane split.  dw [K, H A] / db [H A] in the kernel's layout."""
    B, K = h_online.shape
    A = w_online.shape[1] // H
    qn = head_q32(h_next, w_target, b_target)          # column by column: one head_dot per (head, action)
    qs = head_q32(h_select, w_online, b_online)
    qo = head_q32(h_online, w_online, b_online)
    targets, sel = ensemble_targets(qo, qn, qs, actions, rewards, game_overs, masks, discount, H)
    dq = np.zeros_like(qo)
    dw = np.zeros((K, H * A), F32)
    db = np.zeros(H * A, F32)
    losses = np.zeros(H, F32)
    dz = np.zeros((B, K), F32)
    for h in range(H):
        c = slice(h * A, (h + 1) * A)
        dq[:, c], row = loss_grad32(qo[:, c], targets[:, c], None, huber, B)
        r = backward32(h_online, w_online[:, c], dq[:, c], row, None, B)
        dw[:, c], db[c], losses[h] = r["dw"], r["db"], r["loss"]
        s = np.zeros((B, K), F32)
        for a in range(A):
            s = fma32(dq[:, h * A + a, None], w_online[None, :, h * A + a], s)
        dz = dz + s
    total = losses[0]
    for h in range(1, H):
        total = total + losses[h]
    dh = np.where(np.asarray(h_online) > 0, F32(rescale) * dz, F32(0))
    return dict(q_online=qo, q_next=qn, q_select=qs, targets=targets, dq=dq, dw=dw, db=db, losses=losses, loss=total,
                dh=dh, sel=sel)


def ensemble_backward64(h, w, dq, H, rescale):
    """fp64 dW [K, H A], db, and dh = rescale * sum_h dq_h W_h^T [h > 0] of the given fp32 dq (rescale as fp32)"""
    r = float(F32(rescale))
    b = backward64(h, w, dq)                 # dq [B, H A] against w [K, H A]: the sum over heads and actions at once
    dh, sdh = b["dh"]
    b["dh"] = (r * dh, abs(r) * sdh)
    return b


def ensemble_losses64(q_online, targets, huber, B, H):
    A = q_online.shape[1] // H
    return [loss64(q_online[:, h * A:(h + 1) * A], targets[:, h * A:(h + 1) * A], None, huber, B) for h in range(H)]


# ---- C51 -------------------------------------------------------------------------------------------------------------
def softmax32(x):
    """fp32 softmax in the kernel's steps: max, expf(x - max), sum, divide (the sum sequential here)"""
    x = np.asarray(x, F32)
    m = x.max(-1, keepdims=True)
    e = np.exp(x - m)
    s = np.zeros(x.shape[:-1] + (1,), F32)
    for j in range(x.shape[-1]):
        s = s + e[..., j:j + 1]
    return e / s


def softmax64(x):
    """fp64 softmax of the fp32 logits, and the per-element accumulation length of the fp32 one: N terms in the sum
    plus the rounding of x - max, which is amplified by |x - max| in expf"""
    x64 = np.asarray(x, F64)
    d = x64 - x64.max(-1, keepdims=True)
    e = np.exp(d)
    return e / e.sum(-1, keepdims=True), x.shape[-1] + 10 + np.abs(d)


def projection_overflow(z):
    """(z[-1] - z[0]) / (z[1] - z[0]) > N - 1: a target clamped to v_max lands on bin N"""
    z = np.asarray(z, F64)
    return (z[-1] - z[0]) / (z[1] - z[0]) > z.size - 1


def c51_project(probs, rewards, coef, z, allow_drop=False):
    """the projection of r + coef z_j onto the support, in fp64 in the reference's order: atom j ascending, the floor bin
    credited before the ceil bin, an integral b_j crediting nothing.  probs [B, N] (the target distribution of the
    chosen action, fp64 values), coef [B] = bootstrap * gamma_n.  A share on bin N is an IndexError in the reference:
    this raises AssertionError unless allow_drop, which drops it as the kernel does.  Returns m [B, N] fp64."""
    probs = np.asarray(probs, F64)
    B, N = probs.shape
    z = np.asarray(z, F64)
    r, coef = np.asarray(rewards, F64), np.asarray(coef, F64)
    z0, zl, dz = z[0], z[-1], z[1] - z[0]
    rows = np.arange(B)
    m = np.zeros((B, N))
    for j in range(N):
        tz = r + coef * z[j]
        tz = np.where(tz < z0, z0, np.where(tz > zl, zl, tz))
        bj = (tz - z0) / dz
        lo, hi = np.floor(bj), np.ceil(bj)
        li, ui = lo.astype(np.int64), hi.astype(np.int64)
        if not allow_drop:
            assert ui.max() <= N - 1, "projection index %d > N - 1 = %d" % (ui.max(), N - 1)
        ok = li < N
        m[rows[ok], li[ok]] += probs[ok, j] * (hi[ok] - bj[ok])
        ok = ui < N
        m[rows[ok], ui[ok]] += probs[ok, j] * (bj[ok] - lo[ok])
    return m


def c51_head(nxt, online, select, actions, rewards, coef, z, next_is_prob, allow_drop=False, target_actions=None):
    """cb200_c51_head.  nxt / online / select [B, A, N] fp32 (nxt / select probabilities when next_is_prob); coef [B].
    The target action is the first argmax of sum_j p_j z_j (fp64) of `select` (else `nxt`), or the given
    target_actions.  Returns dict(p_next (fp64 values of the chosen action's fp32 probabilities when next_is_prob, else
    the fp64 softmax), sel, m, q_sel)"""
    B, A, N = online.shape
    src = nxt if select is None else select
    if next_is_prob:
        p_sel = np.asarray(src, F32).astype(F64)
        p_next = np.asarray(nxt, F32).astype(F64)
    else:
        p_sel, p_next = softmax64(src)[0], softmax64(nxt)[0]
    q_sel = p_sel @ np.asarray(z, F64)
    sel = np.argmax(q_sel, axis=1) if target_actions is None else np.asarray(target_actions, np.int64)
    pa = p_next[np.arange(B), sel]
    m = c51_project(pa, rewards, coef, z, allow_drop)
    return dict(sel=sel, q_sel=q_sel, m=m, p_next=pa)


def c51_online64(online, labels, actions, z):
    """fp64 loss rows sum_j lab_j (lse - (x_j - max)) of the given fp32 labels, the softmax, q = sum_j p_j z_j, each with
    S and the accumulation lengths"""
    x64 = np.asarray(online, F64)
    p64, n_soft = softmax64(online)
    mx = x64.max(-1, keepdims=True)
    lse = np.log(np.exp(x64 - mx).sum(-1, keepdims=True))
    lab = np.asarray(labels, F64)
    t = lse - (x64 - mx)
    z = np.asarray(z, F64)
    return dict(p=p64, n_soft=n_soft, loss=(lab * t).sum(-1), loss_S=(np.abs(lab) * (np.abs(t) + 1.0)).sum(-1),
                q=p64 @ z, q_S=p64 @ np.abs(z))
