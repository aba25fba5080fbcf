"""Pins tests/learn_ref.py (no GPU): the exact FMA against rational arithmetic, Adam and polyak against oracle/nets.py
bit for bit, the fp32 reductions against fp64 within gamma_n S, and the plane references against gemm_ref's packers."""
from fractions import Fraction

import numpy as np
import pytest
import torch

import gemm_ref as gr
import learn_ref as lr
from oracle import nets as on

F32, F64 = np.float32, np.float64


# ---- fma32 -------------------------------------------------------------------------------------------------------------
def _round_f32(q):
    """the fp32 number nearest to the rational q (ties to even), inf beyond the range; subnormals included"""
    neg = q < 0
    q = -q if neg else q
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    n, r = divmod(q, ulp)
    n = int(n)
    if 2 * r > ulp or (2 * r == ulp and n % 2 == 1):
        n += 1
    v = n * ulp
    out = np.inf if v >= Fraction(2) ** 128 else float(v)
    return F32(-out if neg else out)


def _fma_exact(a, b, c):
    q = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if q == 0:                                   # the sign of an exact zero: IEEE rules of the exact fp64 sum
        return F32(F64(a) * F64(b) + F64(c))
    return _round_f32(q)


def _triples(rng):
    n = 60000
    out = []
    # random magnitudes across the whole range
    for lo, hi in ((-20, 20), (-64, 64), (-149, -100)):
        a = rng.choice([-1, 1], n) * 2.0 ** rng.uniform(lo, hi, n)
        b = rng.choice([-1, 1], n) * 2.0 ** rng.uniform(lo, hi, n)
        c = rng.choice([-1, 1], n) * 2.0 ** rng.uniform(2 * lo, 2 * hi, n) * (rng.rand(n) < 0.9)
        out.append((a, b, c))
    # cancellation: c = -fl(a b), the result is the product's rounding error
    a = rng.randn(n).astype(F32)
    b = rng.randn(n).astype(F32)
    out.append((a, b, -(a * b)))
    # ties and near-ties: short significands, c a signed power of two
    a = rng.randint(1, 1 << 12, n) * 2.0 ** rng.randint(-12, 12, n)
    b = rng.randint(1, 1 << 13, n) * 2.0 ** rng.randint(-12, 12, n)
    c = rng.choice([-1, 1], n) * 2.0 ** rng.randint(-30, 30, n)
    out.append((a, b, c))
    # the double-rounding trap of a plain fp64 add: a b = half an ulp of c times (1 - 2^-46), c with an odd significand
    e = rng.randint(-100, 100, n)
    c = rng.choice([-1, 1], n) * (2 * rng.randint(1 << 22, 1 << 23, n) + 1) * 2.0 ** (e - 23)
    k = rng.randint(-20, 20, n)
    sgn = rng.choice([-1, 1], n)
    out.append(((1 + 2.0 ** -23) * 2.0 ** k, sgn * (1 - 2.0 ** -23) * 2.0 ** (e - 24 - k), c))
    # subnormal results and exact zeros of both signs
    a = rng.choice([-1, 1], 2000) * 2.0 ** rng.uniform(-80, -60, 2000)
    out.append((a, a, rng.choice([-1, 1], 2000) * 2.0 ** rng.uniform(-149, -127, 2000)))
    out.append((np.array([0.0, -0.0, 0.0, -0.0, 1.0, -1.0]), np.array([1.0, 1.0, -1.0, -1.0, 1.0, 1.0]),
                np.array([0.0, -0.0, -0.0, 0.0, -1.0, 1.0])))
    return [tuple(np.asarray(x, F64).astype(F32) for x in t) for t in out]


def test_fma32_is_the_correctly_rounded_fused_multiply_add():
    """learn_ref.fma32 against exact rational arithmetic on about 360 000 random and adversarial triples; the
    double-rounding family must defeat a plain fp64 add, or it tests nothing"""
    rng = np.random.RandomState(0)
    naive_wrong = 0
    for a, b, c in _triples(rng):
        got = lr.fma32(a, b, c)
        want = np.array([_fma_exact(*t) for t in zip(a, b, c)], F32)
        bad = got.view(np.uint32) != want.view(np.uint32)
        assert not bad.any(), (a[bad][:3], b[bad][:3], c[bad][:3], got[bad][:3], want[bad][:3])
        naive = (a.astype(F64) * b.astype(F64) + c.astype(F64)).astype(F32)
        naive_wrong += int((naive.view(np.uint32) != want.view(np.uint32)).sum())
    assert naive_wrong > 1000, naive_wrong


def test_fma32_special_values():
    inf, nan = np.inf, np.nan
    got = lr.fma32([inf, inf, 1e20, 3e38, 0.0], [1.0, 0.0, 1e20, 2.0, inf], [-1.0, 1.0, 0.0, -3e38, 1.0])
    assert got[0] == inf and np.isnan(got[1]) and got[2] == inf and got[3] == F32(3e38) and np.isnan(got[4])
    assert np.isnan(lr.fma32(nan, 1.0, 1.0))


# ---- optimizer against the oracle --------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 5, 1023, 100003])
def test_adam_matches_oracle_adamtf_bit_for_bit(n):
    """five TF-1.x Adam steps: learn_ref.adam32 with the running fp32 powers equals oracle.nets.AdamTF (torch fp32)"""
    rng = np.random.RandomState(n)
    theta = rng.randn(n).astype(F32)
    lr_, b1, b2, eps = 2.5e-4, 0.9, 0.99, 1e-4
    opt = on.AdamTF([torch.from_numpy(theta)], lr_, b1, b2, eps)
    t_ref = torch.from_numpy(theta.copy())
    th, m, v = theta.copy(), np.zeros(n, F32), np.zeros(n, F32)
    state = np.array([b1, b2], F32)
    for step in range(5):
        g = (rng.randn(n) * 2.0 ** rng.uniform(-10, 10, n)).astype(F32)
        g[::7] = 0
        alpha = lr.adam_alpha32(lr_, state[0], state[1])
        assert alpha == F32(F32(lr_) * np.sqrt(F32(1) - opt.b2p)) / (F32(1) - opt.b1p)
        th, m, v = lr.adam32(th, m, v, g, alpha, b1, b2, eps)
        t_ref = opt.step([t_ref], [torch.from_numpy(g)])[0]
        state = lr.adam_state32(state, b1, b2)
        assert state[0] == opt.b1p and state[1] == opt.b2p
        for got, want, name in ((th, t_ref.numpy(), "theta"), (m, opt.m[0].numpy(), "m"), (v, opt.v[0].numpy(), "v")):
            assert (got.view(np.uint32) == want.view(np.uint32)).all(), (step, name)


@pytest.mark.parametrize("rate", [0.0, 1.0, 1e-3, 5e-3, 1.0 / 3])
def test_polyak_matches_oracle(rate):
    rng = np.random.RandomState(1)
    t, o = rng.randn(1001).astype(F32), rng.randn(1001).astype(F32)
    want = on.polyak({"w": t}, {"w": o}, rate)["w"]
    assert (lr.polyak32(t, o, rate).view(np.uint32) == want.view(np.uint32)).all()


# ---- reductions against fp64 -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols", [(1, 1), (7, 3), (9, 257), (4096, 32), (204800, 32), (3000, 100)])
def test_colsum32_within_gamma_n_of_fp64(rows, cols):
    x = np.random.RandomState(rows + cols).randn(rows, cols).astype(F32)
    got = lr.colsum32(x).astype(F64)
    v, S, n = lr.colsum64(x)
    assert (np.abs(got - v) <= lr.gamma(n + 1024 + 256) * S).all()
    cw, rl, nslab, per = lr.colsum_split(rows, cols)
    assert nslab * per >= rows and (nslab - 1) * per < rows + per


def test_colsum32_order():
    """a column [2^24, 1, 1, ...] in one lane: the fp32 order drops every 1 that follows 2^24, so the emulation's
    order is visible (1 + 1 + ... first would give 2^24 + 7)"""
    x = np.ones((8, 1), F32)
    x[0] = 2.0 ** 24
    assert lr.colsum32(x)[0] == F32(2.0 ** 24)


@pytest.mark.parametrize("n", [1, 255, 4097, 4096 * 1024 + 1])
def test_sumsq32_within_gamma_n_of_fp64(n):
    rng = np.random.RandomState(n % 1000)
    x = (rng.randn(n) * 2.0 ** rng.uniform(-20, 20, n)).astype(F32)
    v, S, m = lr.sumsq64(x)
    assert abs(float(lr.sumsq32(x)) - v) <= lr.gamma(m + 1) * S


@pytest.mark.parametrize("B,A", [(1, 1), (255, 6), (257, 18)])
def test_dueling32_within_gamma_n_of_fp64(B, A):
    rng = np.random.RandomState(A)
    v, adv = rng.randn(B).astype(F32), rng.randn(B, A).astype(F32)
    q = lr.dueling_fwd32(v, adv).astype(F64)
    s, S, dev, dS = lr.dueling64(adv)
    assert (np.abs(q - (v[:, None] + dev)) <= lr.gamma(A + 3) * (np.abs(v)[:, None] + dS)).all()
    d_v, d_adv = lr.dueling_bwd32(adv)
    assert (np.abs(d_v - s) <= lr.gamma(A) * S).all()
    assert (np.abs(d_adv - dev) <= lr.gamma(A + 2) * dS).all()


@pytest.mark.parametrize("huber", [True, False])
def test_regression_head32_within_gamma_n_of_fp64(huber):
    rng = np.random.RandomState(5)
    B, W = 1025, 6
    out, tgt = rng.randn(B, W).astype(F32) * 2, rng.randn(B, W).astype(F32) * 2
    w = rng.rand(B).astype(F32)
    d32, l32 = lr.regression_head32(out, tgt, w, huber, 0.7)
    d64, l64, S = lr.regression_head64(out, tgt, w, huber, 0.7)
    assert (np.abs(d32 - d64) <= lr.gamma(4) * np.abs(d64)).all()
    assert abs(float(l32) - l64) <= lr.gamma(B * W + 16) * S


# ---- planes against gemm_ref's packers ---------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols", [(8, 8), (16, 64), (40, 24)])
def test_plane_references_match_pack_planes(rows, cols):
    x = np.random.RandomState(rows).randn(rows, cols).astype(F32)
    n = rows * cols
    buf = lr.scatter_planes(np.zeros(3 * (n + 16), np.uint16), x, 0, n + 16, 0)
    packed = gr.pack_planes(x)
    for p in range(3):
        assert (buf[p * (n + 16):p * (n + 16) + n] == packed[p]).all()
    assert (lr.scatter_planes(np.zeros(3 * n, np.uint16), x, 0, 0, 1) == gr.pack_planes_il(x)).all()
    tb = np.zeros(3 * n, np.uint16)
    assert (lr.transpose(tb, x.T.copy(), n) == x).all()
    assert (tb.reshape(3, n) == packed).all()
    perm = np.random.RandomState(0).permutation(n)
    pb = np.zeros(3 * n, np.uint16)
    lr.permute(pb, x.ravel()[np.argsort(perm)], perm, cols, -1)
    assert (pb == gr.pack_planes_il(x)).all()


def test_u8_s2d_plane_matches_the_layer_layout():
    """the header's element map: plane row ((y / s) (w / s) + x / s) B + b, column ((y % s) s + x % s) c + ch"""
    rng = np.random.RandomState(2)
    B, h, w, c, s = 8, 12, 20, 2, 4
    x = rng.randint(0, 256, (B, h, w, c)).astype(np.uint8)
    m = lr.u8_s2d_matrix(x, s)
    for b, y, xx, ch in zip(*(rng.randint(0, k, 50) for k in (B, h, w, c))):
        assert m[((y // s) * (w // s) + xx // s) * B + b, ((y % s) * s + xx % s) * c + ch] == x[b, y, xx, ch]
    assert (lr.u8_s2d_plane(x, s) == gr.pack_planes(m.astype(F32), nplanes=1)[0]).all()
