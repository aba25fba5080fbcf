"""Host references of the learn-step kernels of include/coach_b200.h that every Q-network learn step runs: the operand
plane producers (cb200_split_planes, cb200_permute_f32, cb200_transpose, cb200_u8_s2d_planes), the fixed-order
reductions (cb200_colsum, cb200_sumsq, cb200_regression_head_loss_grad, cb200_dueling_combine_fwd / _bwd), the optimizer
and update kernels (cb200_adam_tf / _tf_dev, cb200_polyak, cb200_clip_by_global_norm, cb200_scale, cb200_clip_by_value)
and the strided glue (cb200_act_backward, cb200_axpby_2d, cb200_dqn_td_targets).  numpy only, importable without CUDA.

Every operation has two evaluations:

* an fp32 emulation in the kernel's documented order, bit for bit.  numpy's fp32 + - * / sqrt are correctly rounded,
  like the kernels' _rn intrinsics and their IEEE-compliant defaults (no --use_fast_math).  An fp32 FMA is emulated
  exactly (``fma32``: round to odd in fp64, then one rounding to fp32);
* an fp64 value together with S, the sum of the absolute values of the terms, for |fp32 - fp64| <= gamma_n S.

Where nvcc may contract a multiply and an add that are not written with _rn intrinsics, the emulation follows the FFMA
the sm_90a SASS of the built library shows (cuobjdump -sass):
  act_backward_kernel (heads.cu:165)      tanh: g = fma(-y, y, 1)                             FFMA R, -y, y, 1
  axpby_2d_kernel (heads.cu:176-177)      v = alpha * src;  beta != 0: fma(beta, dst, v)      FMUL, then FFMA
  regression_head_kernel (learn.cu:58-73) Huber: l = fma(q, 0.5 q, lin), row += l (FADD); MSE: row = fma(e, e, row);
                                          local = fma(w, row, local)
  sumsq_stage1 (learn.cu:670)             fmaf as written; the shared-memory trees are plain FADDs
Every other kernel here has no multiply feeding an add outside an intrinsic.

The plane references are built from tests/gemm_ref.py (split3, tiled_elem, tiled_elem_il, pack_planes).
tests/test_learn_ref_host.py pins this module to oracle/nets.py, to exact rational arithmetic and to gemm_ref.
"""
import numpy as np

import gemm_ref as gr
import head_ref as hr

F32, F64 = np.float32, np.float64
U32 = hr.U32
gamma = hr.gamma
ACT_NONE, ACT_RELU, ACT_TANH = gr.ACT_NONE, gr.ACT_RELU, gr.ACT_TANH


def _cdiv(a, b):
    return -(-a // b)


# ---- launch formulas ---------------------------------------------------------------------------------------------------
def flat_grid(n, sm):
    """learn.cu:774-780: ceil(n / 256) blocks of 256, at most 8 per SM (grid-stride loop beyond)"""
    return int(min(max(_cdiv(n, 256), 1), 8 * sm))


def colsum_split(rows, cols):
    """nn.cu:653-657 and :280-286: (cw, rl, nslab, per) -- column block width, row lanes per block, row slabs (about
    8 rows per lane, at most 1024) and rows per slab; stage 2 (:302-303) uses 1024 // cw lanes"""
    cw = min(cols, 256)
    rl = 256 // cw
    nslab = min(max(_cdiv(rows, rl * 8), 1), 1024)
    return cw, rl, nslab, _cdiv(rows, nslab)


def sumsq_blocks(n):
    """learn.cu:948-949: one block per 4096 elements, at most 1024"""
    return min(_cdiv(n, 4096), 1024)


def regression_threads(B):
    """learn.cu:804-805: the smallest power of two >= B, between 32 and 1024 threads of one CTA"""
    t = 32
    while t < B and t < 1024:
        t *= 2
    return t


def adam_dev_vector(n, *addresses):
    """learn.cu:732: adam_tf_dev_kernel takes its float4 path when n % 4 == 0 and theta, m, v, g are 16-byte aligned"""
    return n % 4 == 0 and all(a % 16 == 0 for a in addresses)


def split_planes_grid(max_segment_elems, sm):
    """nn.cu:638-640: blocks per segment, one thread per 8 columns of a row, at most 4 per SM"""
    return int(min(max((max_segment_elems // 8 + 255) // 256, 1), 4 * sm))


def u8_s2d_threads(B, h, w, s):
    """nn.cu:622 / :249: one thread per (b, Y, pair of X, y % s)"""
    return B * (h // s) * ((w // s + 1) // 2) * s


def u8_s2d_grid(B, h, w, s, sm):
    """nn.cu:623-624: at most 16 blocks of 256 per SM"""
    return int(min(_cdiv(u8_s2d_threads(B, h, w, s), 256), 16 * sm))


# ---- exact fp32 FMA ----------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """fp32 fmaf(a, b, c), exactly.  The fp64 product of two fp32 numbers is exact; the fp64 sum is rounded to odd (a
    TwoSum gives the rounding error; an inexact result with an even significand moves one ulp towards the error), and
    rounding that to fp32 (24 bits, fewer than 53 - 1) is the correctly rounded fused result, subnormals included."""
    a, b, c = (np.asarray(x, F32).astype(F64) for x in (a, b, c))
    with np.errstate(invalid="ignore", over="ignore"):
        p = a * b
        s = np.asarray(p + c)
        bb = s - p
        err = (p - (s - bb)) + (c - bb)
        odd = (np.ascontiguousarray(s).view(np.uint64) & np.uint64(1)) != 0
        fix = np.isfinite(s) & np.isfinite(err) & (err != 0) & ~odd
        s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(F32)


# ---- cb200_colsum (nn.cu:274-315) --------------------------------------------------------------------------------------
def _lanes_sum(blocks, lanes):
    """[groups, n, cols] -> [groups, lanes, cols]: lane k sums rows k, k + lanes, ... sequentially in fp32 from +0; the
    zero padding adds +0 to a sum that is never -0"""
    g, n, cols = blocks.shape
    steps = max(_cdiv(n, lanes), 1)
    pad = np.zeros((g, steps * lanes, cols), F32)
    pad[:, :n] = blocks
    pad = pad.reshape(g, steps, lanes, cols)
    s = np.zeros((g, lanes, cols), F32)
    for j in range(steps):
        s = s + pad[:, j]
    return s


def _fold(s):
    """[groups, lanes, cols] -> [groups, cols]: lane 0, then + lane 1, + lane 2, ... in order"""
    acc = s[:, 0].copy()
    for k in range(1, s.shape[1]):
        acc = acc + s[:, k]
    return acc


def colsum32(x):
    """Stage 1: slab k = rows [k per, (k + 1) per), row lane l of a block sums rows l, l + rl, ... of its slab; the rl
    lanes are folded in order.  Stage 2: the same over the nslab partial rows with 1024 // cw lanes."""
    x = np.asarray(x, F32)
    rows, cols = x.shape
    cw, rl, nslab, per = colsum_split(rows, cols)
    xp = np.zeros((nslab * per, cols), F32)
    xp[:rows] = x
    part = _fold(_lanes_sum(xp.reshape(nslab, per, cols), rl))                  # [nslab, cols]
    return _fold(_lanes_sum(part[None], 1024 // cw))[0]


def colsum64(x):
    """(fp64 column sums, S, n) -- n: the accumulation length of any fp32 order"""
    x64 = np.asarray(x, F64)
    return x64.sum(0), np.abs(x64).sum(0), x64.shape[0]


# ---- cb200_sumsq (learn.cu:664-689) ------------------------------------------------------------------------------------
def _tree(red):
    """shared-memory tree over the last axis: red[t] += red[t + k] for k = len / 2, ..., 1"""
    red = red.copy()
    k = red.shape[-1] // 2
    while k:
        red[..., :k] = red[..., :k] + red[..., k:2 * k]
        k //= 2
    return red[..., 0]


def sumsq32(x):
    """Block b owns the slab [b per, (b + 1) per); thread t accumulates s = fmaf(x_i, x_i, s) over i = lo + t, + 256,
    ...; a 256 -> 1 tree; stage 2: a 1024 -> 1 tree over the partials, zero-padded"""
    x = np.asarray(x, F32).ravel()
    n = x.size
    blocks = sumsq_blocks(n)
    per = _cdiv(n, blocks)
    steps = _cdiv(per, 256)
    xp = np.zeros((blocks, steps * 256), F32)
    flat = np.zeros(blocks * per, F32)
    flat[:n] = x
    xp[:, :per] = flat.reshape(blocks, per)
    xp = xp.reshape(blocks, steps, 256)
    s = np.zeros((blocks, 256), F32)
    for j in range(steps):
        s = fma32(xp[:, j], xp[:, j], s)
    part = np.zeros(1024, F32)
    part[:blocks] = _tree(s)
    return F32(_tree(part))


def sumsq64(x):
    x64 = np.asarray(x, F64).ravel()
    v = float((x64 * x64).sum())
    return v, v, x64.size


# ---- cb200_regression_head_loss_grad (learn.cu:46-82) ------------------------------------------------------------------
def regression_head32(out, target, weights, huber, loss_weight):
    """T = regression_threads(B) threads of one CTA; thread t takes rows t, t + T, ...; per row w = loss_weight *
    weight (loss_weight alone when weights is None), the row loss summed over the W columns in order, d_out =
    (w * (1 / B)) * l'(e); local = fma(w, row, local); a T -> 1 tree; loss = red[0] * (1 / B).
    Returns (d_out [B, W], loss)."""
    out, target = np.asarray(out, F32), np.asarray(target, F32)
    B, W = out.shape
    T = regression_threads(B)
    inv_b = F32(1) / F32(B)
    lw = F32(loss_weight)
    w = np.full(B, lw, F32) if weights is None else lw * np.asarray(weights, F32)
    e = out - target
    row = np.zeros(B, F32)
    if huber:
        ae = np.abs(e)
        q = np.minimum(ae, F32(1))
        lin = ae - q
        l = fma32(q, F32(0.5) * q, lin)
        g = np.where(ae <= 1, e, np.where(e > 0, F32(1), F32(-1))).astype(F32)
        for a in range(W):
            row = row + l[:, a]
    else:
        g = e + e
        for a in range(W):
            row = fma32(e[:, a], e[:, a], row)
    d_out = (w * inv_b)[:, None] * g
    local = np.zeros(T, F32)
    for k in range(_cdiv(B, T)):
        idx = np.arange(k * T, min((k + 1) * T, B))
        local[idx - k * T] = fma32(w[idx], row[idx], local[idx - k * T])
    return d_out.astype(F32), F32(_tree(local) * inv_b)


def regression_head64(out, target, weights, huber, loss_weight):
    """fp64 (d_out, loss, S of the loss), from the fp32 inputs and loss_weight / weights rounded to fp32"""
    e = np.asarray(out, F64) - np.asarray(target, F64)
    B = e.shape[0]
    w = float(F32(loss_weight)) * (np.ones(B) if weights is None else np.asarray(weights, F32).astype(F64))
    if huber:
        ae = np.abs(e)
        q = np.minimum(ae, 1.0)
        l, g = 0.5 * q * q + (ae - q), np.clip(e, -1.0, 1.0)
    else:
        l, g = e * e, 2.0 * e
    lw = w[:, None] * l
    return w[:, None] * g / B, lw.sum() / B, np.abs(lw).sum() / B


# ---- cb200_dueling_combine_fwd / _bwd (learn.cu:642-660) ---------------------------------------------------------------
def _rowsum32(x):
    s = np.zeros(x.shape[0], F32)
    for a in range(x.shape[1]):
        s = s + x[:, a]
    return s


def dueling_fwd32(v, adv):
    """q = v + (adv - (sum_a adv) / A), the sum sequential in fp32"""
    adv = np.asarray(adv, F32)
    mean = _rowsum32(adv) / F32(adv.shape[1])
    return np.asarray(v, F32).reshape(-1)[:, None] + (adv - mean[:, None])


def dueling_bwd32(dq):
    """d_v = sum_a dq (sequential), d_adv = dq - d_v / A"""
    dq = np.asarray(dq, F32)
    s = _rowsum32(dq)
    return s, dq - (s / F32(dq.shape[1]))[:, None]


def dueling64(x):
    """fp64 (row sum, its S, x - mean, its S) of [B, A]"""
    x64 = np.asarray(x, F64)
    s, S = x64.sum(1), np.abs(x64).sum(1)
    A = x64.shape[1]
    return s, S, x64 - (s / A)[:, None], np.abs(x64) + (S / A)[:, None]


# ---- optimizer and updates (learn.cu:691-772) --------------------------------------------------------------------------
def adam_alpha32(lr, beta1_power, beta2_power):
    """alpha = lr * sqrt(1 - beta2_power) / (1 - beta1_power) in fp32: the host (cb200_adam_tf) and the device
    (adam_tf_dev_kernel) evaluate the same correctly rounded steps"""
    one = F32(1)
    return F32(F32(lr) * np.sqrt(one - F32(beta2_power))) / (one - F32(beta1_power))


def adam32(theta, m, v, g, alpha, beta1, beta2, eps):
    """TF-1.x ApplyAdam: m += (g - m) (1 - b1); v += (g g - v) (1 - b2); theta -= (m alpha) / (sqrt(v) + eps).
    Returns the new (theta, m, v)."""
    theta, m, v, g = (np.asarray(x, F32) for x in (theta, m, v, g))
    one = F32(1)
    m = m + (g - m) * (one - F32(beta1))
    v = v + (g * g - v) * (one - F32(beta2))
    return theta - (m * F32(alpha)) / (np.sqrt(v) + F32(eps)), m, v


def adam_state32(state, beta1, beta2):
    """adam_state_advance_kernel: the running powers multiplied once per step"""
    return np.array([F32(state[0]) * F32(beta1), F32(state[1]) * F32(beta2)], F32)


def polyak32(target, online, rate):
    """rate * online + (1 - rate) * target; rate and 1 - rate (evaluated in fp64) rounded to fp32 first"""
    return F32(rate) * np.asarray(online, F32) + F32(1.0 - rate) * np.asarray(target, F32)


def clip_global32(g, sumsq, clip):
    """g * (clip / fmaxf(sqrtf(sumsq), clip)).  fmaxf drops a NaN: sumsq = NaN scales by 1 (g passes unchanged);
    sumsq = +inf scales by 0"""
    c = F32(clip)
    with np.errstate(invalid="ignore", over="ignore"):
        scale = c / np.fmax(np.sqrt(F32(sumsq)), c)
        return np.asarray(g, F32) * scale


def scale32(g, s):
    return np.asarray(g, F32) * F32(s)


def clip_by_value32(g, clip):
    """x < -clip ? -clip : (x > clip ? clip : x) -- NaN passes through"""
    g = np.asarray(g, F32)
    c = F32(clip)
    return np.where(g < -c, -c, np.where(g > c, c, g)).astype(F32)


# ---- strided glue ------------------------------------------------------------------------------------------------------
def act_backward32(dy, y, act):
    """dz = dy * act'(y): relu 1 where y > 0 else 0 (y = 0 exactly gives 0), tanh fma(-y, y, 1), none 1"""
    dy, y = np.asarray(dy, F32), np.asarray(y, F32)
    if act == ACT_RELU:
        g = np.where(y > 0, F32(1), F32(0))
    elif act == ACT_TANH:
        g = fma32(-y, y, F32(1))
    else:
        g = np.ones_like(y)
    return dy * g


def axpby32(src, dst, alpha, beta):
    """v = alpha * src; beta == 0: v (dst is not read), else fma(beta, dst, v)"""
    v = F32(alpha) * np.asarray(src, F32)
    if F32(beta) == 0:
        return v
    return fma32(F32(beta), np.asarray(dst, F32), v)


def dqn_td_targets(q_next, q_select, q_online, actions, rewards, game_overs, discount):
    """cb200_dqn_td_targets: the DQN rule of head_ref.rule_targets (learn.cu:18-41 restates dqn_head_fused's target);
    returns (targets fp32, td_err fp64)"""
    t, td, _ = hr.rule_targets(hr.TARGET_DQN, q_online, q_next, q_select, actions, rewards, game_overs, discount)
    return t, td


# ---- operand planes --------------------------------------------------------------------------------------------------
def scatter_planes(buf, x, offset, stride, layout=0):
    """write the bf16 truncation split of x [rows, cols] into the uint16 buffer `buf` at element `offset`: layout 0
    core-tiled, the three planes `stride` apart; layout 1 row-group interleaved.  Elements the planes do not cover keep
    their contents (a plane matrix whose row count is not a multiple of 8 leaves the rest of its last row group)."""
    x = np.asarray(x, F32)
    rows, cols = x.shape
    r, c = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    parts = gr.split3(x)
    for p in range(3):
        idx = gr.tiled_elem_il(r, c, cols, p) if layout else gr.tiled_elem(r, c, cols) + p * stride
        buf[offset + idx] = parts[p]
    return buf


def split_planes(buf, src, segments, stride):
    """cb200_split_planes: segments = [(src offset, rows, cols, plane offset, layout)]"""
    src = np.asarray(src, F32)
    for soff, rows, cols, poff, layout in segments:
        scatter_planes(buf, src[soff:soff + rows * cols].reshape(rows, cols), poff, stride, layout)
    return buf


def permute(buf, src, table, plane_cols, stride):
    """cb200_permute_f32: dst = src[table]; with planes, dst seen as [n / plane_cols, plane_cols] (stride -1:
    row-group interleaved).  Returns dst."""
    dst = np.asarray(src, F32)[np.asarray(table, np.int64)]
    if buf is not None:
        scatter_planes(buf, dst.reshape(-1, plane_cols), 0, stride, 1 if stride < 0 else 0)
    return dst


def transpose(buf, src, stride):
    """cb200_transpose: dst [cols, rows] = src^T; with planes, dst in the core-tiled format (plane columns = rows)"""
    dst = np.ascontiguousarray(np.asarray(src, F32).T)
    if buf is not None:
        scatter_planes(buf, dst, 0, stride, 0)
    return dst


def u8_s2d_matrix(x, s):
    """uint8 NHWC frames [B, h, w, c] -> the space-to-depth matrix [h/s * w/s * B, s s c]: row (Y (w/s) + X) B + b,
    column ((y % s) s + x % s) c + ch (the reshape of tests/test_tiled_host.py, for any h, w)"""
    B, h, w, c = x.shape
    return x.reshape(B, h // s, s, w // s, s, c).transpose(1, 3, 0, 2, 4, 5).reshape(h // s * (w // s) * B, s * s * c)


def tile_cores(m):
    """[R, C] (multiples of 8) -> its elements in the core-tiled order: (r, c) lands at gr.tiled_elem(r, c, C).  The
    reshape form of gr.pack_planes for large matrices (tests/test_learn_ref_host.py pins the two together)"""
    R, C = m.shape
    return np.ascontiguousarray(np.asarray(m).reshape(R // 8, 8, C // 8, 8).transpose(0, 2, 1, 3)).ravel()


def u8_s2d_plane(x, s):
    """cb200_u8_s2d_planes: the one exact bf16 plane of u8_s2d_matrix, core-tiled (bf16 bits of 0..255 from
    gr.split3)"""
    lut = gr.split3(np.arange(256, dtype=F32))[0]
    return tile_cores(lut[u8_s2d_matrix(np.asarray(x), s)])
