"""The fused Q heads at the C ABI against tests/head_ref.py (fp32 emulation of the header's contract and fp64), for every
case of tests/head_cases.py:

  (a) exact probes: planted Q values (h = [Q | 0], W = [I; 0]) -- Q, targets, td_err and dL/dQ bit for bit, with
      argmax ties, |e| = 1, e = 0, terminal rows and out-of-range actions; small dyadic h / W / rewards / weights, where
      every product and partial sum is exact in fp32 -- every output bit for bit wherever that holds; C51 with
      next_is_prob = 1 -- the projection of the taken action bit for bit;
  (b) random data: the targets bit for bit given the Q values the kernel reports, dL/dQ bit for bit given Q and the
      targets, and every accumulated output within gamma_n S of fp64 and within 4x the fp32 emulation's error (the
      observed e / S are printed);
  (c) invariants: repeated calls give the same bits, a NaN-filled workspace (idle warps write zero partials), canaries
      after every output, dh_planes = dh, NULL optional outputs change nothing else, MMC at rho = 0 and PAL at
      alpha = rho = 0 are DDQN, a one-head ensemble is the DQN head, masked-out ensemble rows have dq = 0, C51 rows are
      isolated from each other;
  (d) the contract: argument errors, the dynamic shared memory opt-in on every device, and a final check that every
      (rule, features) instantiation and both C51 shared-memory paths ran."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import head_cases as hc
import head_ref as hr
from abi_util import GUARD, Outs, _bits, _dev, _lib, _ptr, assert_bits  # noqa: F401

pytestmark = pytest.mark.gpu

RAN = set()


def _planes_to_f32(planes, B, K, stride):
    """tiled bf16 hi / mid / lo planes -> hi + mid + lo (exact in fp64) as [B, K]"""
    p = planes.astype(np.uint32)
    rows, cols = np.meshgrid(np.arange(B), np.arange(K), indexing="ij")
    idx = ((rows >> 3) * (K >> 3) + (cols >> 3)) * 64 + (rows & 7) * 8 + (cols & 7)
    tot = np.zeros((B, K))
    for k in range(3):
        tot += (p[k * stride + idx] << 16).view(np.float32).astype(np.float64)
    return tot


# ---- cb200_dqn_head_fused ----------------------------------------------------------------------------------------------
def run_dqn(c, d, rule=None, out=None, alpha=None, rho=None):
    L, lib = _lib()
    rule = c["rule"] if rule is None else rule
    out = c["out"] if out is None else out
    B, A, K = c["B"], c["A"], c["F"]
    keep = {k: _dev(d[k]) for k in ("h_next", "h_online", "h_select", "h_target_s", "w_target", "b_target",
                                   "w_online", "b_online", "actions", "rewards", "game_overs", "returns", "weights")}
    o = Outs()
    desc = L.DqnHeadDesc()
    desc.h_next, desc.h_online = _ptr(keep["h_next"]), _ptr(keep["h_online"])
    desc.h_select = _ptr(keep["h_select"]) if c["select"] else None
    for k in ("w_target", "b_target", "w_online", "b_online", "actions", "rewards", "game_overs"):
        setattr(desc, k, _ptr(keep[k]))
    desc.weights = _ptr(keep["weights"]) if c["weights"] else None
    desc.discount, desc.huber, desc.batch, desc.features, desc.n_actions = d["discount"], int(c["huber"]), B, K, A
    desc.q_online, desc.targets, desc.dq = (o.add(k, (B, A)) for k in ("q_online", "targets", "dq"))
    desc.td_err = o.add("td_err", (B,), torch.float64)
    desc.dw, desc.db = o.add("dw", (K, A)), o.add("db", (A,))
    full = out == "all"
    if full:
        desc.q_next, desc.loss = o.add("q_next", (B, A)), o.add("loss", (1,))
        if rule != hr.TARGET_DQN:
            desc.q_select = o.add("q_select", (B, A))
        if rule >= hr.TARGET_PAL:
            desc.q_target_s = o.add("q_target_s", (B, A))
    if out in ("all", "dh", "both"):
        desc.dh = o.add("dh", (B, K))
    stride = B * K + 64
    if out in ("planes", "both"):
        desc.dh_planes, desc.dh_plane_stride = o.add("planes", (3 * stride,), torch.int16), stride
    nparts = (B + 15) // 16 * 8
    ws = torch.full((nparts * (K * A + A + 1),), float("nan"), device="cuda")
    desc.target_rule = rule
    desc.h_target_s = _ptr(keep["h_target_s"])
    desc.mc_returns = _ptr(keep["returns"])
    desc.pal_alpha = d["alpha"] if alpha is None else alpha
    desc.mc_mixing_rate = d["rho"] if rho is None else rho
    desc.workspace = ws.data_ptr()
    L.check(lib.cb200_dqn_head_fused(ctypes.byref(desc), L.current_stream()))
    RAN.add(("dqn", rule, K))
    r = o.numpy()
    if "planes" in r:
        r["planes"] = r["planes"].view(np.uint16)
        gap = r["planes"].reshape(3, stride)[:, B * K:]
        assert (gap == 0x5A5A).all(), "planes: write between the planes"
        r["planes_f32"] = _planes_to_f32(r["planes"], B, K, stride)
    return r


def _ref_dqn(c, d, rule=None, alpha=None, rho=None):
    rule = c["rule"] if rule is None else rule
    return hr.dqn_head(rule, d["h_next"], d["h_online"], d["h_select"] if c["select"] else None, d["w_target"],
                       d["b_target"], d["w_online"], d["b_online"], d["actions"], d["rewards"], d["game_overs"],
                       d["discount"], d["weights"] if c["weights"] else None, c["huber"], d["h_target_s"],
                       d["returns"], d["alpha"] if alpha is None else alpha, d["rho"] if rho is None else rho)


def fp32_exact(h, dq, w, weights, row):
    """per element of dW, db, dh and the loss: True where every term and every partial sum is an fp32 number whatever
    the order (all terms multiples of 2^g and the sum of their magnitudes below 2^(24 + g))"""
    def ok(terms, axis):
        t = np.abs(np.asarray(terms, np.float64))
        nz = t != 0
        m, e = np.frexp(np.where(nz, t, 1.0))                     # t = m 2^e, m in [0.5, 1)
        mant = np.ldexp(m, 53).astype(np.uint64)                  # t = mant 2^(e - 53)
        low = mant & (~mant + np.uint64(1))                       # lowest set bit
        lowexp = np.where(nz, e - 53 + np.frexp(low.astype(np.float64))[1] - 1, 10 ** 4)
        g = np.minimum(lowexp.min(axis=axis), 900)
        return t.sum(axis=axis) < np.ldexp(1.0, g + 24)
    h64, d64, w64 = (np.asarray(x, np.float64) for x in (h, dq, w))
    wt = np.ones(h64.shape[0]) if weights is None else np.asarray(weights, np.float64)
    return dict(dw=ok(h64[:, :, None] * d64[:, None, :], 0), db=ok(d64, 0),
                dh=ok(d64[:, None, :] * w64[None, :, :], 2) | (h64 <= 0),
                loss=bool(ok((wt * np.asarray(row, np.float64))[:, None], 0)[0]))


def check_bound(name, got, ref, S, n, emu=None, report=None, floor=0.0):
    got, ref, S = (np.asarray(x, np.float64) for x in (got, ref, S))
    if got.size == 0:                        # e.g. the softmax rows of the other actions at n_actions = 1
        return
    err = np.abs(got - ref)
    bound = hr.gamma(n) * S + floor
    bad = err > bound
    assert not bad.any(), "%s: %d elements beyond gamma_n S, worst err %.3e bound %.3e" % (
        name, bad.sum(), err[bad].max(), bound[bad][np.argmax(err[bad])])
    ratio = float((err / np.maximum(S, 1e-300)).max()) if err.size else 0.0
    if emu is not None:
        e_emu = float(np.abs(np.asarray(emu, np.float64) - ref).max())
        # the same error as the kernel's summation order gives, up to 4x (one unit of S below the emulation's error)
        assert err.max() <= 4 * max(e_emu, hr.U32 * float(S.max())), "%s: err %.3e > 4 x fp32 emulation %.3e" % (
            name, err.max(), e_emu)
    if report is not None:
        report.append("%-10s n=%-6d max e/S = %.2e (gamma_n = %.2e)" % (name, int(np.max(n)), ratio,
                                                                       float(np.max(hr.gamma(n)))))


def _optional_outputs_agree(c, r, full):
    for k in r:
        if k in full and k not in ("planes", "planes_f32"):
            assert_bits(r[k], full[k], "%s with NULL optional outputs" % k)


@pytest.mark.parametrize("c", hc.DQN_CASES, ids=hc.case_id)
def test_dqn_head_planted_q_values(c):
    d = hc.dqn_planted(c)
    r = run_dqn(c, d, out="all")
    ref = _ref_dqn(c, d)
    B, A = c["B"], c["A"]
    q = lambda k: d[k][:, :A]                                                                   # noqa: E731
    assert_bits(r["q_online"], q("h_online"), "q_online")
    assert_bits(r["q_next"], q("h_next"), "q_next")
    if c["rule"] != hr.TARGET_DQN:
        assert_bits(r["q_select"], q("h_select"), "q_select")
    if c["rule"] >= hr.TARGET_PAL:
        assert_bits(r["q_target_s"], q("h_target_s"), "q_target_s")
    for k in ("targets", "td_err", "dq"):
        assert_bits(r[k], ref[k], k)
    ok = (d["actions"] < 0) | (d["actions"] >= A)
    assert_bits(r["targets"][ok], q("h_online")[ok], "out-of-range rows keep Q(s)")
    assert (r["td_err"][ok] == 0).all() and (r["dq"][ok] == 0).all()


@pytest.mark.parametrize("c", hc.DQN_CASES, ids=hc.case_id)
def test_dqn_head_dyadic_exact(c):
    d = hc.dqn_dyadic(c)
    r = run_dqn(c, d, out="all")
    ref = _ref_dqn(c, d)
    for k in ("q_online", "q_next", "targets", "td_err", "dq"):
        assert_bits(r[k], ref[k], k)
    _, row = hr.loss_grad32(r["q_online"], r["targets"], d["weights"] if c["weights"] else None, c["huber"], c["B"])
    ex = fp32_exact(d["h_online"], r["dq"], d["w_online"], d["weights"] if c["weights"] else None, row)
    b64 = hr.backward64(d["h_online"], d["w_online"], r["dq"])
    pow2 = c["B"] & (c["B"] - 1) == 0
    for k in ("dw", "db", "dh"):
        if pow2:
            assert ex[k].all(), "%s: the dyadic probe is not exact in fp32" % k
        assert_bits(r[k][ex[k]], b64[k][0][ex[k]], k)
    l64, _ = hr.loss64(r["q_online"], r["targets"], d["weights"] if c["weights"] else None, c["huber"], c["B"])
    if ex["loss"] and pow2:
        assert_bits(r["loss"][0], np.float32(l64), "loss")


@pytest.mark.parametrize("c", hc.DQN_CASES, ids=hc.case_id)
def test_dqn_head_random_against_fp64(c):
    d = hc.dqn_random(c)
    r = run_dqn(c, d, out="all")
    B, A, K = c["B"], c["A"], c["F"]
    w = d["weights"] if c["weights"] else None
    emu = _ref_dqn(c, d)
    report = ["case " + hc.case_id(c)]
    q64, S = hr.head_q64(d["h_online"], d["w_online"], d["b_online"])
    check_bound("q_online", r["q_online"], q64, S, hr.dot_terms(K), emu["q_online"], report)
    q64, S = hr.head_q64(d["h_next"], d["w_target"], d["b_target"])
    check_bound("q_next", r["q_next"], q64, S, hr.dot_terms(K), emu["q_next"], report)
    # targets bit for bit given the kernel's Q values; DQN-rule DDQN does not report Q_online(s'): rows whose selection
    # the fp32 emulation cannot decide are left out
    qs = r.get("q_select")
    keep = np.ones(B, bool)
    if c["select"] and qs is None:
        qs = emu["q_select"]
        q64s, Ss = hr.head_q64(d["h_select"], d["w_online"], d["b_online"])
        srt = np.sort(q64s, axis=1)
        gap = srt[:, -1] - srt[:, -2] if A > 1 else np.full(B, np.inf)
        keep = gap > 4 * hr.gamma(hr.dot_terms(K)) * Ss.max(axis=1)
        assert keep.mean() >= 0.95
    t, td, _ = hr.rule_targets(c["rule"], r["q_online"], r["q_next"], qs if c["select"] else None, d["actions"],
                               d["rewards"], d["game_overs"], d["discount"], r.get("q_target_s"), d["returns"],
                               d["alpha"], d["rho"])
    assert_bits(r["targets"][keep], t[keep], "targets")
    assert_bits(r["td_err"][keep], td[keep], "td_err")
    dq, row = hr.loss_grad32(r["q_online"], r["targets"], w, c["huber"], B)
    assert_bits(r["dq"], dq, "dq")
    check_bound("dq", r["dq"], hr.dq64(r["q_online"], r["targets"], w, c["huber"], B),
                np.abs(hr.dq64(r["q_online"], r["targets"], w, c["huber"], B)), 4, report=report)
    e32 = hr.backward32(d["h_online"], d["w_online"], r["dq"], row, w, B)
    b64 = hr.backward64(d["h_online"], d["w_online"], r["dq"])
    check_bound("dw", r["dw"], b64["dw"][0], b64["dw"][1], B + 8, e32["dw"], report)
    check_bound("db", r["db"], b64["db"][0], b64["db"][1], B + 8, e32["db"], report)
    check_bound("dh", r["dh"], b64["dh"][0], b64["dh"][1], A, e32["dh"], report)
    l64, ls = hr.loss64(r["q_online"], r["targets"], w, c["huber"], B)
    check_bound("loss", r["loss"][0], l64, ls, B * A + 10, e32["loss"], report)
    print("\n  ".join(report))


@pytest.mark.parametrize("c", hc.DQN_CASES, ids=hc.case_id)
def test_dqn_head_invariants(c):
    d = hc.dqn_random(c, seed=7)
    r1, r2 = run_dqn(c, d), run_dqn(c, d)
    for k in r1:
        assert_bits(r1[k], r2[k], "%s run twice" % k)
    full = run_dqn(c, d, out="both" if c["B"] % 8 == 0 else "all")
    _optional_outputs_agree(c, r1, full)
    if "planes_f32" in full:
        assert_bits(full["planes_f32"], full["dh"].astype(np.float64), "dh_planes reconstruct dh")
    if "planes" in r1 and "planes" in full:
        assert_bits(r1["planes"], full["planes"], "planes only = planes + fp32")
    if c["rule"] != hr.TARGET_DQN:
        ddqn = run_dqn(c, d, rule=hr.TARGET_DQN, out="all")
        zero = run_dqn(c, d, out="all", alpha=0.0, rho=0.0)
        for k in ("q_online", "q_next", "targets", "dq", "dw", "db", "dh", "loss"):
            assert_bits(zero[k], ddqn[k], "%s: rho = alpha = 0 vs DDQN" % k)
        # td_err of these rules is measured from the fp32 target, the DQN rule's from the fp64 one
        rows, a = np.arange(c["B"]), np.clip(d["actions"], 0, c["A"] - 1)
        ok = (d["actions"] >= 0) & (d["actions"] < c["A"])
        want = np.where(ok, np.abs(ddqn["targets"][rows, a].astype(np.float64) - ddqn["q_online"][rows, a]), 0.0)
        assert_bits(zero["td_err"], want, "td_err: rho = alpha = 0")


# ---- cb200_ensemble_head_fused -----------------------------------------------------------------------------------------
def run_ens(c, d, out=None, masks=None, rescale=None):
    L, lib = _lib()
    out = c["out"] if out is None else out
    B, A, K, H = c["B"], c["A"], c["F"], c["H"]
    keep = {k: _dev(d[k]) for k in ("h_next", "h_online", "h_select", "w_target", "b_target", "w_online", "b_online",
                                   "actions", "rewards", "game_overs")}
    keep["masks"] = _dev(d["masks"] if masks is None else masks)
    o = Outs()
    e = L.EnsembleHeadDesc()
    for k in keep:
        setattr(e, k, _ptr(keep[k]))
    e.discount, e.huber, e.batch, e.features, e.heads, e.n_actions = d["discount"], int(c["huber"]), B, K, H, A
    e.grad_rescale = c["rescale"] if rescale is None else rescale
    e.q_online, e.targets, e.dq = (o.add(k, (B, H * A)) for k in ("q_online", "targets", "dq"))
    e.losses, e.dw, e.db = o.add("losses", (H,)), o.add("dw", (K, H * A)), o.add("db", (H * A,))
    if out == "all":
        e.q_next, e.q_select, e.loss = o.add("q_next", (B, H * A)), o.add("q_select", (B, H * A)), o.add("loss", (1,))
    if out in ("all", "dh", "both"):
        e.dh = o.add("dh", (B, K))
    stride = B * K + 64
    if out in ("planes", "both"):
        e.dh_planes, e.dh_plane_stride = o.add("planes", (3 * stride,), torch.int16), stride
    nparts = (B + 15) // 16 * 8
    ws = torch.full((nparts * H * (K * A + A + 1),), float("nan"), device="cuda")
    e.workspace = ws.data_ptr()
    L.check(lib.cb200_ensemble_head_fused(ctypes.byref(e), L.current_stream()))
    RAN.add(("ens", K))
    r = o.numpy()
    if "planes" in r:
        r["planes"] = r["planes"].view(np.uint16)
        r["planes_f32"] = _planes_to_f32(r["planes"], B, K, stride)
    return r


@pytest.mark.parametrize("c", hc.ENS_CASES, ids=hc.case_id)
def test_ensemble_head_against_fp64(c):
    d = hc.ens_data(c)
    r = run_ens(c, d, out="all")
    B, A, K, H = c["B"], c["A"], c["F"], c["H"]
    emu = hr.ensemble_head(d["h_next"], d["h_online"], d["h_select"], d["w_target"], d["b_target"], d["w_online"],
                           d["b_online"], d["actions"], d["rewards"], d["game_overs"], d["masks"], d["discount"], H,
                           c["huber"], c["rescale"])
    report = ["case " + hc.case_id(c)]
    for k, hk, wk, bk in (("q_online", "h_online", "w_online", "b_online"), ("q_next", "h_next", "w_target", "b_target"),
                          ("q_select", "h_select", "w_online", "b_online")):
        q64, S = hr.head_q64(d[hk], d[wk], d[bk])
        check_bound(k, r[k], q64, S, hr.dot_terms(K), emu[k], report)
    t, _ = hr.ensemble_targets(r["q_online"], r["q_next"], r["q_select"], d["actions"], d["rewards"], d["game_overs"],
                               d["masks"], d["discount"], H)
    assert_bits(r["targets"], t, "targets")
    for h in range(H):
        cols = slice(h * A, (h + 1) * A)
        dq, _ = hr.loss_grad32(r["q_online"][:, cols], r["targets"][:, cols], None, c["huber"], B)
        assert_bits(r["dq"][:, cols], dq, "dq head %d" % h)
        off = d["masks"][:, h] == 0
        assert (r["dq"][off, cols] == 0).all(), "masked-out rows of head %d have dq != 0" % h
    b64 = hr.ensemble_backward64(d["h_online"], d["w_online"], r["dq"], H, c["rescale"])
    check_bound("dw", r["dw"], b64["dw"][0], b64["dw"][1], B + 8, emu["dw"], report)
    check_bound("db", r["db"], b64["db"][0], b64["db"][1], B + 8, emu["db"], report)
    check_bound("dh", r["dh"], b64["dh"][0], b64["dh"][1], H * A + 2, emu["dh"], report)
    l64 = hr.ensemble_losses64(r["q_online"], r["targets"], c["huber"], B, H)
    check_bound("losses", r["losses"], [v for v, _ in l64], [s for _, s in l64], B * A + 10, emu["losses"], report)
    total = r["losses"][0]
    for h in range(1, H):
        total = total + r["losses"][h]
    assert_bits(r["loss"][0], total, "loss = sum of the head losses in head order")
    print("\n  ".join(report))


@pytest.mark.parametrize("c", hc.ENS_CASES, ids=hc.case_id)
def test_ensemble_head_invariants(c):
    d = hc.ens_data(c, seed=8)
    r1, r2 = run_ens(c, d), run_ens(c, d)
    for k in r1:
        assert_bits(r1[k], r2[k], "%s run twice" % k)
    full = run_ens(c, d, out="both" if c["B"] % 8 == 0 else "all")
    _optional_outputs_agree(c, r1, full)
    if "planes_f32" in full:
        assert_bits(full["planes_f32"], full["dh"].astype(np.float64), "dh_planes reconstruct dh")
    if "dh" in full:
        # the rescale is one fp32 product applied to the unscaled sum
        one = run_ens(c, d, out="dh", rescale=1.0)
        assert_bits(full["dh"], np.float32(np.float32(c["rescale"])) * one["dh"], "dh = fp32(r * dh at r = 1)")


@pytest.mark.parametrize("c", [x for x in hc.ENS_CASES if x["H"] == 1], ids=hc.case_id)
def test_one_head_ensemble_is_the_dqn_head(c):
    d = hc.ens_data(c, seed=9)
    masks = np.ones((c["B"], 1), np.uint8)
    ens = run_ens(c, d, out="all", masks=masks, rescale=1.0)
    dc = dict(rule=hr.TARGET_DQN, F=c["F"], A=c["A"], B=c["B"], select=True, weights=False, huber=c["huber"])
    dd = dict(d, h_target_s=d["h_next"], returns=np.zeros(c["B"]), weights=None, alpha=0.0, rho=0.0)
    dqn = run_dqn(dc, dd, out="all")
    for k in ("q_online", "q_next", "targets", "dq", "dw", "db", "dh"):
        assert_bits(ens[k], dqn[k], k)
    assert_bits(ens["losses"], dqn["loss"], "losses")
    assert_bits(ens["loss"], dqn["loss"], "loss")


# ---- cb200_c51_head ----------------------------------------------------------------------------------------------------
def run_c51(c, d, perm=None):
    L, lib = _lib()
    B, A, N = c["B"], c["A"], c["N"]
    if perm is not None:
        d = {k: (v[perm] if k != "z" and isinstance(v, np.ndarray) else v) for k, v in d.items()}
    keep = {k: _dev(d[k]) for k in ("next", "online", "select", "actions", "rewards", "game_overs", "bootstrap", "z")}
    o = Outs()
    ptrs = [o.add("labels", (B, A, N)), o.add("dlogits", (B, A, N)), o.add("loss_rows", (B, A)),
            o.add("total", (1,)), o.add("td_err", (B,), torch.float64), o.add("q_online", (B, A), torch.float64),
            o.add("target_actions", (B,), torch.int64)]
    L.check(lib.cb200_c51_head(_ptr(keep["next"]), _ptr(keep["online"]), _ptr(keep["select"]), _ptr(keep["actions"]),
                               _ptr(keep["rewards"]), _ptr(keep["game_overs"]) if d["bootstrap"] is None else None,
                               _ptr(keep["bootstrap"]), _ptr(keep["z"]), d["gamma_n"], B, A, N,
                               int(c["next_is_prob"]), *ptrs, L.current_stream()))
    RAN.add(("c51", "opt-in" if 64 * N > 48 * 1024 else "default"))
    return o.numpy()


def _coef(d):
    boot = d["bootstrap"] if d["bootstrap"] is not None else 1.0 - d["game_overs"].astype(np.float64)
    return boot * d["gamma_n"]


@pytest.mark.parametrize("c", hc.C51_CASES, ids=hc.case_id)
def test_c51_head_against_fp64(c):
    d = hc.c51_data(c)
    r = run_c51(c, d)
    B, A, N = c["B"], c["A"], c["N"]
    rows = np.arange(B)
    report = ["case " + hc.case_id(c)]
    ref = hr.c51_head(d["next"], d["online"], d["select"], d["actions"], d["rewards"], _coef(d), d["z"],
                      c["next_is_prob"], allow_drop=c["guard"])
    # the target action: the first maximum of the fp64 Q values, up to the rounding of the kernel's lane-order sum
    qs = ref["q_sel"]
    sel = r["target_actions"]
    slack = 1e-12 if c["next_is_prob"] else float(hr.gamma(N + 10 + 160)) * np.abs(d["z"]).max()
    assert (qs[rows, sel] >= qs.max(axis=1) - slack).all()
    exact_rows = (qs.max(axis=1) - np.where(np.arange(A)[None] == ref["sel"][:, None], -np.inf, qs).max(axis=1)) > slack
    np.testing.assert_array_equal(sel[exact_rows], ref["sel"][exact_rows])
    ref = hr.c51_head(d["next"], d["online"], d["select"], d["actions"], d["rewards"], _coef(d), d["z"],
                      c["next_is_prob"], allow_drop=c["guard"], target_actions=sel)
    act = d["actions"]
    lab_a = r["labels"][rows, act]
    if c["next_is_prob"]:
        assert_bits(lab_a, ref["m"].astype(np.float32), "projection")
    else:
        _, n_soft = hr.softmax64(np.asarray(d["next"])[rows, sel])
        check_bound("m", lab_a, ref["m"], ref["m"], n_soft.max() + 1, report=report, floor=N * hr.TINY32)
    on = hr.c51_online64(d["online"], r["labels"], act, d["z"])
    other = np.ones((B, A), bool)
    other[rows, act] = False
    check_bound("softmax", r["labels"][other], on["p"][other], on["p"][other], on["n_soft"][other],
                emu=hr.softmax32(d["online"])[other], report=report, floor=hr.TINY32)
    assert (r["dlogits"][other] == 0).all(), "dlogits of the other actions must be exactly 0"
    p_a = on["p"][rows, act]
    check_bound("dlogits", r["dlogits"][rows, act], p_a - lab_a.astype(np.float64), p_a + np.abs(lab_a),
                on["n_soft"][rows, act] + 2, report=report, floor=2 * hr.TINY32)
    check_bound("loss_rows", r["loss_rows"], on["loss"], on["loss_S"], N + 10, report=report)
    assert_bits(r["td_err"], r["loss_rows"][rows, act].astype(np.float64), "td_err = loss of the taken action")
    lr = r["loss_rows"].astype(np.float64)
    check_bound("total", r["total"][0], lr.sum(), np.abs(lr).sum(), B * A + 10, report=report)
    check_bound("q_online", r["q_online"], on["q"], on["q_S"], N + 10, report=report,
                floor=N * hr.TINY32 * np.abs(d["z"]).max())
    print("\n  ".join(report))


@pytest.mark.parametrize("c", hc.C51_CASES, ids=hc.case_id)
def test_c51_head_invariants(c):
    """repeated calls give the same bits; every sample's outputs depend on that sample only (a permuted batch gives the
    permuted outputs): no projection share leaves its row"""
    d = hc.c51_data(c, seed=11)
    r1, r2 = run_c51(c, d), run_c51(c, d)
    for k in r1:
        assert_bits(r1[k], r2[k], "%s run twice" % k)
    perm = np.random.RandomState(3).permutation(c["B"])
    rp = run_c51(c, d, perm=perm)
    for k in ("labels", "dlogits", "loss_rows", "td_err", "q_online", "target_actions"):
        assert_bits(rp[k], r1[k][perm], "%s of a permuted batch" % k)


# ---- the contract ------------------------------------------------------------------------------------------------------
def test_argument_errors():
    L, lib = _lib()
    x = torch.zeros(1 << 20, device="cuda")
    p = x.data_ptr()
    d = L.DqnHeadDesc()
    for f in ("h_next", "h_online", "h_select", "w_target", "b_target", "w_online", "b_online", "actions", "rewards",
              "game_overs", "q_online", "targets", "td_err", "dq", "dw", "db", "workspace"):
        setattr(d, f, p)
    d.batch, d.features, d.n_actions = 16, 256, 4
    call = lambda: lib.cb200_dqn_head_fused(ctypes.byref(d), L.current_stream())                # noqa: E731
    for a in (0, 9):
        d.n_actions = a
        assert call() == -1, a
    d.n_actions = 4
    for f in (0, 128, 384, 1024):
        d.features = f
        assert call() == -1, f
    d.features, d.batch, d.dh_planes, d.dh_plane_stride = 256, 12, p, 8
    assert call() == -1
    e = L.EnsembleHeadDesc()
    for f in ("h_next", "h_online", "h_select", "w_target", "b_target", "w_online", "b_online", "actions", "rewards",
              "game_overs", "masks", "q_online", "targets", "dq", "losses", "dw", "db", "workspace"):
        setattr(e, f, p)
    e.batch, e.features, e.n_actions, e.heads = 16, 256, 4, 2
    ecall = lambda: lib.cb200_ensemble_head_fused(ctypes.byref(e), L.current_stream())          # noqa: E731
    for h in (0, 65):
        e.heads = h
        assert ecall() == -1, h
    e.heads = 2
    for a in (0, 9):
        e.n_actions = a
        assert ecall() == -1, a
    e.n_actions, e.features = 4, 384
    assert ecall() == -1
    e.features, e.batch, e.dh_planes, e.dh_plane_stride = 256, 12, p, 8
    assert ecall() == -1
    for n in (1, 1025):
        assert lib.cb200_c51_head(p, p, None, p, p, p, None, p, 0.99, 4, 2, n, 0, p, p, p, p, p, None, None,
                                  L.current_stream()) == -1, n
    torch.cuda.synchronize()


_TWO_DEVICES = r"""
import ctypes, sys
import numpy as np, torch
sys.path.insert(0, sys.argv[1])
import head_cases as hc
from test_head_kernels_gpu import run_ens
c = dict(H=10, F=512, A=6, B=32, masks="random", rescale=0.1, huber=True, out="both")
d = hc.ens_data(c)
outs = []
for dev in (0, 1):
    torch.cuda.set_device(dev)
    outs.append(run_ens(c, d))
for k in outs[0]:
    assert np.array_equal(outs[0][k].view(np.uint8), outs[1][k].view(np.uint8)), k
print("ok")
"""


def test_ensemble_opt_in_on_every_device():
    """the 64 KB opt-in of the F = 512 ensemble kernel is per device: the same call on device 0, then on device 1"""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    res = subprocess.run([sys.executable, "-c", _TWO_DEVICES, here], capture_output=True, text=True, timeout=600,
                         cwd=os.path.dirname(here))
    assert res.returncode == 0 and "ok" in res.stdout, res.stdout + res.stderr


REQUIRED = {("dqn", r, f) for r in hc.RULES for f in hc.FEATURES} | {("ens", f) for f in hc.FEATURES} | \
    {("c51", "default"), ("c51", "opt-in")}


def test_every_head_variant_was_run():
    """every (rule, features) instantiation of the DQN head, both ensemble instantiations and both C51 shared-memory
    paths ran above (those that did not run in this session are run now); a new variant belongs in this list"""
    if not REQUIRED <= RAN:
        for c in hc.DQN_CASES:
            if ("dqn", c["rule"], c["F"]) not in RAN:
                run_dqn(c, hc.dqn_random(c))
        for c in hc.ENS_CASES:
            if ("ens", c["F"]) not in RAN:
                run_ens(c, hc.ens_data(c))
        for c in hc.C51_CASES:
            if ("c51", "opt-in" if 64 * c["N"] > 48 * 1024 else "default") not in RAN:
                run_c51(c, hc.c51_data(c))
    assert REQUIRED <= RAN, sorted(REQUIRED - RAN)
