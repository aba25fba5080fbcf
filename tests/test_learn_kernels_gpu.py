"""The learn-step kernels at the C ABI against tests/learn_ref.py, bit for bit, at the shapes and edges of
tests/learn_cases.py:

  (a) plane producers (split_planes, permute_f32, transpose, u8_s2d_planes): every plane element, and the canaries
      around and between the planes;
  (b) reductions (colsum, sumsq, regression_head_loss_grad, dueling_combine_*): bit for bit with the fp32 emulation of
      the kernel's order, and within gamma_n S of fp64;
  (c) optimizer and updates (adam_tf, adam_tf_dev, polyak, clip_by_global_norm, scale, clip_by_value) and strided glue
      (act_backward, axpby_2d, dqn_td_targets): bit for bit, five consecutive Adam steps, a graph-replayed Adam step;
  (d) invariants: repeat calls give the same bits, NaN-filled workspaces change nothing, every output is followed by
      canaries, and cb200_launch_count rises by the documented number per call;
  (e) the contract: argument errors, and a final check, from the launch formulas, that every path ran."""
import ctypes

import numpy as np
import pytest
import torch

import gemm_ref as gr
import learn_cases as lc
import learn_ref as lr
from abi_util import _lib, assert_bits

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
RAN = set()
GUARD_BYTES = 256
FILL = 0xA5                                  # canary byte around every buffer (0xA5A5A5A5 is an fp32 NaN)
_SM = []


def sm():
    if not _SM:
        L, lib = _lib()
        n, a, b = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
        L.check(lib.cb200_device_info(ctypes.byref(n), ctypes.byref(a), ctypes.byref(b)))
        _SM.append(n.value)
    return _SM[0]


class Buf(object):
    """a device copy of a numpy array `offset` bytes into a buffer of canary bytes, GUARD_BYTES of them after it"""

    def __init__(self, x, offset=0):
        x = np.ascontiguousarray(x)
        self.dtype, self.shape, self.nb, self.off = x.dtype, x.shape, x.nbytes, offset
        self.t = torch.full((offset + x.nbytes + GUARD_BYTES,), FILL, dtype=torch.uint8, device="cuda")
        if x.nbytes:
            self.t[offset:offset + x.nbytes] = torch.from_numpy(x.reshape(-1).view(np.uint8)).cuda()

    @property
    def ptr(self):
        return self.t.data_ptr() + self.off

    def get(self):
        torch.cuda.synchronize()
        h = self.t.cpu().numpy()
        assert (h[:self.off] == FILL).all() and (h[self.off + self.nb:] == FILL).all(), "write outside the buffer"
        return h[self.off:self.off + self.nb].view(self.dtype).reshape(self.shape)


def nan_ws(n):
    return Buf(np.full(n, np.nan, F32))


def call(name, *args, launches=1):
    L, lib = _lib()
    c0 = lib.cb200_launch_count()
    L.check(getattr(lib, name)(*(args + (L.current_stream(),))))
    assert lib.cb200_launch_count() - c0 == launches, "%s: launch count" % name


def assert_bits_or_nan(got, want, name):
    """bit for bit, except that a NaN only has to be a NaN (the device returns the canonical NaN)"""
    nan = np.isnan(want)
    assert np.isnan(got[nan]).all(), "%s: NaN expected" % name
    assert_bits(got[~nan], want[~nan], name)


def canary16(n):
    return np.full(n, FILL * 0x101, np.uint16)


# ---- (a) operand planes -------------------------------------------------------------------------------------------------
def _split_layout(rng):
    """segments (src offset, rows, cols, plane offset, layout) of one fp32 buffer; plane 0 regions back to back (the
    interleaved ones take 3 rows * cols there), then a gap of canaries before planes 1 and 2"""
    shapes = [(8, 8, 0), (24, 64, 1), (512, 512, 0), (40, 16, 1), (16, 24, 0), (8, 8, 0)]
    segs, soff, poff = [], 4, 0            # src offsets stay 16-byte aligned, not 0
    for rows, cols, layout in shapes:
        segs.append((soff, rows, cols, poff, layout))
        soff += rows * cols + 4
        poff += rows * cols * (3 if layout else 1) + 64
    src = lc.spread(rng, soff, -30, 30)
    for k, (o, rows, cols, _, _) in enumerate(segs[:-1]):
        src[o:o + cols] = lc.special_row(cols)
    o, _, cols, _, _ = segs[-1]
    src[o:o + 8] = np.array([np.nan, np.inf, -np.inf, 1.0, -0.0, 2.0 ** -140, 3.0, -1.5], F32)
    src[o + 8:o + 16].view(np.uint32)[:] = [0x7F800001, 0xFFC00000, 0x7FBFFFFF, 0x7F7FFFFF, 0xFF800000, 0x00000001,
                                            0x80000000, 0x3F800001]
    return src, segs, poff + 64


@pytest.mark.parametrize("max_elems", ["largest", 2048])
def test_split_planes(max_elems):
    """several segments in one call, both layouts, segment offsets, and max_segment_elems below the largest segment
    (the grid-stride loop).  The last segment holds NaN / +-inf: its hi plane is the top half-word of the input and its
    mid / lo planes are NaN (x - hi is NaN), pinned as documented behaviour"""
    rng = np.random.RandomState(1)
    src, segs, stride = _split_layout(rng)
    largest = max(r * c for _, r, c, _, _ in segs)
    me = largest if max_elems == "largest" else max_elems
    planes = Buf(canary16(3 * stride))
    d_src, d_segs = Buf(src), Buf(np.array(segs, np.int64))
    call("cb200_split_planes", d_src.ptr, planes.ptr, stride, d_segs.ptr, len(segs), me)
    got = planes.get()
    gx = lr.split_planes_grid(me, sm())
    if largest // 8 > gx * 256:
        RAN.add(("split_planes", "grid-stride"))
    RAN.update(("split_planes", "layout%d" % s[4]) for s in segs)
    want = lr.split_planes(canary16(3 * stride), src, segs, stride)
    o, rows, cols, poff, _ = segs[-1]
    x = src[o:o + rows * cols].reshape(rows, cols)
    r, c = np.nonzero(~np.isfinite(x))
    e = poff + gr.tiled_elem(r, c, cols)
    lower = np.zeros(got.size, bool)
    lower[np.concatenate([e + stride, e + 2 * stride])] = True
    assert_bits(got[~lower], want[~lower], "split_planes")
    assert_bits(got[e], (x[r, c].view(np.uint32) >> 16).astype(np.uint16), "hi plane of non-finite values")
    b = got[lower].astype(np.uint32)
    assert (((b >> 7) & 0xFF) == 0xFF).all() and ((b & 0x7F) != 0).all(), "mid / lo planes of non-finite values"


@pytest.mark.parametrize("table", ["perm", "repeat"])
@pytest.mark.parametrize("stride", ["tiled", "interleaved", "none"])
@pytest.mark.parametrize("rows,cols", [(24, 64), (8, 8), (4800, 64)])
def test_permute_f32(table, stride, rows, cols):
    rng = np.random.RandomState(rows + cols)
    n = rows * cols
    src = lc.spread(rng, n + 17)
    src[:10] = lc.special_row(10)
    tab = (rng.permutation(n) if table == "perm" else rng.randint(0, n + 17, n)).astype(np.int32)
    ps = {"tiled": n + 64, "interleaved": -1, "none": 0}[stride]
    nbuf = 3 * (n + 64)
    planes = Buf(canary16(nbuf)) if stride != "none" else None
    dst = Buf(np.full(n, np.nan, F32))
    d_src, d_tab = Buf(src), Buf(tab)
    call("cb200_permute_f32", d_src.ptr, d_tab.ptr, n, dst.ptr, planes.ptr if planes else None, ps, cols)
    want_planes = canary16(nbuf) if planes else None
    want = lr.permute(want_planes, src, tab, cols, ps)
    assert_bits(dst.get(), want, "permute dst")
    if planes:
        assert_bits(planes.get(), want_planes, "permute planes")
    if n > lr.flat_grid(n, sm()) * 256:
        RAN.add(("permute", "grid-stride"))


@pytest.mark.parametrize("rows", lc.TRANSPOSE_DIMS)
@pytest.mark.parametrize("cols", lc.TRANSPOSE_DIMS)
def test_transpose(rows, cols):
    """dst = src^T; with planes (rows % 8 == 0) the planes of dst [cols, rows]; when cols % 8 != 0 the rows of the last
    row group past cols keep their contents"""
    rng = np.random.RandomState(rows * 7 + cols)
    src = lc.spread(rng, (rows, cols))
    with_planes = rows % 8 == 0
    stride = rows * ((cols + 7) // 8 * 8) + 64
    planes = Buf(canary16(3 * stride)) if with_planes else None
    dst = Buf(np.full(rows * cols, np.nan, F32))
    d_src = Buf(src)
    call("cb200_transpose", d_src.ptr, rows, cols, dst.ptr, planes.ptr if planes else None, stride if planes else 0)
    want_planes = canary16(3 * stride) if planes else None
    want = lr.transpose(want_planes, src, stride)
    assert_bits(dst.get().reshape(cols, rows), want, "transpose dst")
    if planes:
        assert_bits(planes.get(), want_planes, "transpose planes")
        RAN.add(("transpose", "planes", cols % 8 == 0))


@pytest.mark.parametrize("case", lc.U8_S2D_CASES, ids=lambda c: "B%d_h%d_w%d_c%d_s%d" % c)
def test_u8_s2d_planes(case):
    B, h, w, c, s = case
    rng = np.random.RandomState(B + h + w)
    x = rng.randint(0, 256, (B, h, w, c)).astype(np.uint8)
    x.reshape(-1)[:4] = [0, 255, 1, 128]
    n = h * w * B * c
    plane = Buf(canary16(n))
    d_x = Buf(x)
    call("cb200_u8_s2d_planes", d_x.ptr, B, h, w, c, s, plane.ptr)
    assert_bits(plane.get(), lr.u8_s2d_plane(x, s), "u8 s2d plane")
    if lr.u8_s2d_threads(B, h, w, s) > lr.u8_s2d_grid(B, h, w, s, sm()) * 256:
        RAN.add(("u8_s2d", "grid-stride"))
    if (w // s) % 2:
        RAN.add(("u8_s2d", "odd-x-pair"))
    RAN.add(("u8_s2d", "s%d" % s))


# ---- (b) reductions -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,cols", lc.COLSUM_CASES)
def test_colsum(rows, cols):
    """bit for bit with the emulation of the slab / row-lane order, within gamma_n S of fp64; a NaN-filled workspace,
    a repeat call, two launches"""
    rng = np.random.RandomState(rows % 9973 + cols)
    x = (rng.randn(rows, cols) * 2.0 ** rng.uniform(-8, 8, cols)).astype(F32)
    d_x = Buf(x)
    outs = []
    for _ in range(2):
        out = Buf(np.full(cols, np.nan, F32))
        ws = nan_ws(1024 * cols)
        call("cb200_colsum", d_x.ptr, rows, cols, out.ptr, ws.ptr, launches=2)
        outs.append(out.get())
    assert_bits(outs[1], outs[0], "colsum repeat")
    assert_bits(outs[0], lr.colsum32(x), "colsum")
    v, S, n = lr.colsum64(x)
    cw, rl, nslab, per = lr.colsum_split(rows, cols)
    assert (np.abs(outs[0] - v) <= lr.gamma(n + rl + 1024 // cw) * S).all()
    if nslab == 1024 and rows > 1024 * rl * 8:
        RAN.add(("colsum", "slab-cap"))
    if 256 % cw:
        RAN.add(("colsum", "idle-lanes"))
    if cols > 256:
        RAN.add(("colsum", "column-blocks"))
    if nslab > 1024 // cw:
        RAN.add(("colsum", "stage2-lanes"))


@pytest.mark.parametrize("n", lc.SUMSQ_N)
@pytest.mark.parametrize("overflow", [False, True])
def test_sumsq(n, overflow):
    rng = np.random.RandomState(n % 10007)
    x = lc.sumsq_data(n, rng, overflow and n > 1)
    d_x = Buf(x)
    got = []
    for _ in range(2):
        out = Buf(np.full(1, np.nan, F32))
        ws = nan_ws(1024)
        call("cb200_sumsq", d_x.ptr, n, out.ptr, ws.ptr, launches=2)
        got.append(out.get())
    assert_bits(got[1], got[0], "sumsq repeat")
    assert_bits(got[0], np.array([lr.sumsq32(x)], F32), "sumsq")
    if overflow and n > 1:
        assert got[0][0] == np.inf
    else:
        v, S, m = lr.sumsq64(x)
        assert abs(float(got[0][0]) - v) <= lr.gamma(m + 1) * S
    if -(-n // 4096) > 1024:
        RAN.add(("sumsq", "block-cap"))
    if -(-n // lr.sumsq_blocks(n)) > 256:
        RAN.add(("sumsq", "strided-thread"))


def _regression_cases():
    out = []
    k = 0
    for B in lc.REGRESSION_B:
        for W in lc.REGRESSION_W:
            for huber in (True, False):
                out.append((B, W, huber, k % 2 == 0, (1.0, 0.7, 2.5)[k % 3], k % 4 != 3))
                k += 1
    return out


@pytest.mark.parametrize("B,W,huber,weights,loss_weight,with_loss", _regression_cases())
def test_regression_head_loss_grad(B, W, huber, weights, loss_weight, with_loss):
    rng = np.random.RandomState(B * 31 + W)
    out = (rng.randn(B, W) * 2).astype(F32)
    tgt = (rng.randn(B, W) * 2).astype(F32)
    e1 = rng.rand(B, W) < 0.1                                           # |e| = 1 exactly
    out[e1] = rng.randint(-8, 8, e1.sum()) / 4
    tgt[e1] = out[e1] + rng.choice([-1.0, 1.0], e1.sum())
    w = rng.rand(B).astype(F32) if weights else None
    d_out, d_t, d_w = Buf(np.full((B, W), np.nan, F32)), Buf(out), Buf(tgt)
    dw = Buf(w) if weights else None
    loss = Buf(np.full(1, np.nan, F32)) if with_loss else None
    call("cb200_regression_head_loss_grad", d_t.ptr, d_w.ptr, dw.ptr if dw else None, B, W, int(huber), loss_weight,
         d_out.ptr, loss.ptr if loss else None)
    want_d, want_l = lr.regression_head32(out, tgt, w, huber, loss_weight)
    assert_bits(d_out.get(), want_d, "d_out")
    if with_loss:
        got_l = loss.get()[0]
        assert_bits(got_l, want_l, "loss")
        _, l64, S = lr.regression_head64(out, tgt, w, huber, loss_weight)
        assert abs(float(got_l) - l64) <= lr.gamma(B * W + 12) * S
    T = lr.regression_threads(B)
    RAN.add(("regression", "rows-per-thread>1" if B > T else "rows-per-thread=1"))
    if T > B:
        RAN.add(("regression", "idle-threads"))


@pytest.mark.parametrize("A", lc.DUELING_A)
@pytest.mark.parametrize("B", lc.DUELING_B)
def test_dueling_combine(A, B):
    rng = np.random.RandomState(A * 7 + B)
    v, adv, dq = (lc.spread(rng, s, -6, 6) for s in ((B,), (B, A), (B, A)))
    q = Buf(np.full((B, A), np.nan, F32))
    d_v, d_adv, d_dq = Buf(v), Buf(adv), Buf(dq)
    call("cb200_dueling_combine_fwd", d_v.ptr, d_adv.ptr, B, A, q.ptr)
    gv, gadv = Buf(np.full(B, np.nan, F32)), Buf(np.full((B, A), np.nan, F32))
    call("cb200_dueling_combine_bwd", d_dq.ptr, B, A, gv.ptr, gadv.ptr)
    got_q, got_v, got_adv = q.get(), gv.get(), gadv.get()
    assert_bits(got_q, lr.dueling_fwd32(v, adv), "q")
    want_v, want_adv = lr.dueling_bwd32(dq)
    assert_bits(got_v, want_v, "d_v")
    assert_bits(got_adv, want_adv, "d_adv")
    s, S, dev, dS = lr.dueling64(adv)
    assert (np.abs(got_q - (v[:, None] + dev)) <= lr.gamma(A + 3) * (np.abs(v)[:, None] + dS)).all()
    s, S, dev, dS = lr.dueling64(dq)
    assert (np.abs(got_v - s) <= lr.gamma(A) * S).all()
    assert (np.abs(got_adv - dev) <= lr.gamma(A + 2) * dS).all()


# ---- (c) optimizer and updates ------------------------------------------------------------------------------------------
def _adam_n(n):
    big = 4 * 8 * sm() * 256 + 4 * 123
    return {"big": big, "big+1": big + 1}.get(n, n)


@pytest.mark.parametrize("n", lc.ADAM_N)
@pytest.mark.parametrize("offset", [0, 4])
@pytest.mark.parametrize("lr_", [2.5e-4, 0.0])
def test_adam_five_steps(n, offset, lr_):
    """five steps of adam_tf_dev and of adam_tf (host alpha from the same fp32 powers): theta, m, v and the device
    powers bit for bit after every step.  offset 4: every pointer one element past a 16-byte boundary (the scalar
    path).  g = 0 entries, v = 0 at the start, and entries whose g * g overflows"""
    n = _adam_n(n)
    rng = np.random.RandomState(n % 1009 + offset)
    b1, b2, eps = 0.9, 0.99, 1e-4
    theta = rng.randn(n).astype(F32)
    dev = [Buf(theta, offset), Buf(np.zeros(n, F32), offset), Buf(np.zeros(n, F32), offset)]
    host = [Buf(theta, offset), Buf(np.zeros(n, F32), offset), Buf(np.zeros(n, F32), offset)]
    state = Buf(np.array([b1, b2], F32))
    th, m, v = theta, np.zeros(n, F32), np.zeros(n, F32)
    powers = np.array([b1, b2], F32)
    vec = lr.adam_dev_vector(n, *(b.ptr for b in dev))
    for step in range(5):
        g = lc.spread(rng, n, -12, 12)
        g[::3] = 0
        g[1::11] = F32(2e19) * (1 if step % 2 else -1)              # g * g overflows
        d_g = Buf(g, offset)
        call("cb200_adam_tf_dev", *(b.ptr for b in dev), d_g.ptr, n, lr_, b1, b2, eps, state.ptr, launches=2)
        call("cb200_adam_tf", *(b.ptr for b in host), d_g.ptr, n, lr_, b1, b2, eps, float(powers[0]),
             float(powers[1]))
        th, m, v = lr.adam32(th, m, v, g, lr.adam_alpha32(lr_, powers[0], powers[1]), b1, b2, eps)
        powers = lr.adam_state32(powers, b1, b2)
        # an entry whose v overflowed turns NaN on the next step (inf - inf), as in TF
        for name, b, want in zip(("theta", "m", "v"), dev, (th, m, v)):
            assert_bits_or_nan(b.get(), want, "adam_tf_dev %s step %d" % (name, step))
        for name, b, want in zip(("theta", "m", "v"), host, (th, m, v)):
            assert_bits_or_nan(b.get(), want, "adam_tf %s step %d" % (name, step))
        assert_bits(state.get(), powers, "state step %d" % step)
    if lr_ == 0:
        assert_bits_or_nan(dev[0].get(), np.where(np.isnan(th), th, theta), "lr = 0 leaves theta")
    grid = lr.flat_grid(n, sm())
    RAN.add(("adam_dev", "vector" if vec else "scalar"))
    if (n // 4 if vec else n) > grid * 256:
        RAN.add(("adam_dev", "vector-grid-stride" if vec else "scalar-grid-stride"))


def test_adam_dev_graph_replay_equals_eager_steps():
    """one adam_tf_dev step captured in a CUDA graph and replayed three times = three eager steps (the powers advance
    on the device)"""
    L, lib = _lib()
    n = 100004
    rng = np.random.RandomState(3)
    theta, g = rng.randn(n).astype(F32), rng.randn(n).astype(F32)
    runs = []
    for graph in (False, True):
        bufs = [Buf(theta), Buf(np.zeros(n, F32)), Buf(np.zeros(n, F32)), Buf(g), Buf(np.array([0.9, 0.99], F32))]
        args = [b.ptr for b in bufs[:4]] + [n, 2.5e-4, 0.9, 0.99, 1e-4, bufs[4].ptr]
        if graph:
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            gr_ = torch.cuda.CUDAGraph()
            with torch.cuda.stream(s):
                torch.cuda.synchronize()
                with torch.cuda.graph(gr_, stream=s):
                    L.check(lib.cb200_adam_tf_dev(*(args + [L.current_stream()])))
            torch.cuda.synchronize()
            assert_bits(bufs[0].get(), theta, "capture does not run the step")
            for _ in range(3):
                gr_.replay()
        else:
            for _ in range(3):
                L.check(lib.cb200_adam_tf_dev(*(args + [L.current_stream()])))
        runs.append([b.get() for b in bufs])
    for k, name in enumerate(("theta", "m", "v", "g", "state")):
        assert_bits(runs[1][k], runs[0][k], "graph replay %s" % name)
    RAN.add(("adam_dev", "graph"))


@pytest.mark.parametrize("rate", lc.POLYAK_RATES)
@pytest.mark.parametrize("n", [1001, "big"])
def test_polyak(rate, n):
    n = 8 * sm() * 256 * 2 + 1 if n == "big" else n
    rng = np.random.RandomState(n % 101)
    t, o = lc.spread(rng, n, -10, 10), lc.spread(rng, n, -10, 10)
    d_t, d_o = Buf(t), Buf(o)
    call("cb200_polyak", d_t.ptr, d_o.ptr, n, rate)
    assert_bits(d_t.get(), lr.polyak32(t, o, rate), "polyak")
    if n > lr.flat_grid(n, sm()) * 256:
        RAN.add(("polyak", "grid-stride"))


@pytest.mark.parametrize("case", ["below", "equal", "above", "zero", "inf", "nan"])
@pytest.mark.parametrize("n", [1000, "big"])
def test_clip_by_global_norm(case, n):
    """sqrt(sumsq) <= clip leaves the bits untouched; above, g * (clip / norm); +inf scales by 0; NaN by 1"""
    n = 8 * sm() * 256 + 77 if n == "big" else n
    rng = np.random.RandomState(7)
    g = lc.spread(rng, n, -10, 10)
    clip, s = {"below": (1.0, 0.01), "equal": (0.5, 0.25), "above": (1.0, 100.0), "zero": (2.0, 0.0),
               "inf": (1.0, np.inf), "nan": (1.0, np.nan)}[case]
    d_g, d_s = Buf(g), Buf(np.array([s], F32))
    call("cb200_clip_by_global_norm", d_g.ptr, n, d_s.ptr, clip)
    got = d_g.get()
    assert_bits(got, lr.clip_global32(g, s, clip), "clip_by_global_norm")
    if case in ("below", "equal", "zero", "nan"):
        assert_bits(got, g, "clip leaves g untouched")
    if case == "inf":
        assert (got == 0).all()
    if n > lr.flat_grid(n, sm()) * 256:
        RAN.add(("clip", "grid-stride"))


@pytest.mark.parametrize("n", [1000, "big"])
def test_scale_and_clip_by_value(n):
    n = 8 * sm() * 256 * 3 + 5 if n == "big" else n
    rng = np.random.RandomState(9)
    g = lc.spread(rng, n, -10, 10)
    g[:6] = [np.nan, np.inf, -np.inf, 3.0, -3.0, -0.0]
    for s in (0.5, 1.0 / 3, 0.125):
        d_g = Buf(g)
        call("cb200_scale", d_g.ptr, n, s)
        got = d_g.get()
        assert_bits(got[1:], lr.scale32(g, s)[1:], "scale")
        assert np.isnan(got[0])
    d_g = Buf(g)
    call("cb200_clip_by_value", d_g.ptr, n, 3.0)
    assert_bits(d_g.get(), lr.clip_by_value32(g, 3.0), "clip_by_value (NaN passes through)")
    if n > lr.flat_grid(n, sm()) * 256:
        RAN.add(("scale", "grid-stride"))


def test_add_i64():
    x = Buf(np.array([5, -7], np.int64))
    call("cb200_add_i64", x.ptr, -12)
    call("cb200_add_i64", x.ptr + 8, 1 << 40)
    assert (x.get() == [-7, (1 << 40) - 7]).all()


# ---- (c) strided glue ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("act", [lr.ACT_NONE, lr.ACT_RELU, lr.ACT_TANH])
@pytest.mark.parametrize("rows,cols,ld", [(1, 1, 1), (33, 5, 9), (300, 64, 70), (4096, 17, 17)])
def test_act_backward(act, rows, cols, ld):
    """dz on a column block of wider buffers: the gap columns between cols and ld keep their canaries; relu at y = 0
    exactly gives 0"""
    rng = np.random.RandomState(rows + cols + act)
    dy = lc.spread(rng, (rows, ld + 2), -6, 6)
    y = (rng.randn(rows, ld + 1) if act != lr.ACT_TANH else np.tanh(rng.randn(rows, ld + 1))).astype(F32)
    y[::3, 0] = 0
    y[1::3, 0] = -0.0
    dz0 = lc.spread(rng, (rows, ld), -6, 6)
    dz = Buf(dz0)
    d_dy, d_y = Buf(dy), Buf(y)
    call("cb200_act_backward", d_dy.ptr, ld + 2, d_y.ptr, ld + 1, rows, cols, act, dz.ptr, ld)
    got = dz.get()
    assert_bits(got[:, :cols], lr.act_backward32(dy[:, :cols], y[:, :cols], act), "dz")
    assert_bits(got[:, cols:], dz0[:, cols:], "dz gap columns")
    if act == lr.ACT_RELU:
        assert (got[::3, 0] == 0).all()


@pytest.mark.parametrize("alpha,beta", [(1.0, 0.0), (-0.5, 0.0), (1.0, 1.0), (-0.25, 0.75), (3.0, -1.0 / 3)])
@pytest.mark.parametrize("rows,cols,ld", [(1, 1, 1), (33, 5, 9), (4096, 17, 24)])
def test_axpby_2d(alpha, beta, rows, cols, ld):
    """beta = 0 over a NaN-filled dst: dst is not read; the gap columns keep their canaries"""
    rng = np.random.RandomState(rows + cols)
    src = lc.spread(rng, (rows, ld + 3), -6, 6)
    dst0 = np.full((rows, ld), np.nan, F32) if beta == 0 else lc.spread(rng, (rows, ld), -6, 6)
    gap = dst0[:, cols:].copy()
    dst = Buf(dst0)
    d_src = Buf(src)
    call("cb200_axpby_2d", d_src.ptr, ld + 3, rows, cols, alpha, beta, dst.ptr, ld)
    got = dst.get()
    assert_bits(got[:, :cols], lr.axpby32(src[:, :cols], dst0[:, :cols], alpha, beta), "axpby")
    assert_bits(got[:, cols:], gap, "axpby gap columns")


@pytest.mark.parametrize("A", lc.TD_A)
@pytest.mark.parametrize("double", [False, True])
def test_dqn_td_targets(A, double):
    """ties (quarter-integer Q values), terminal rows, out-of-range actions (-1 and A)"""
    rng = np.random.RandomState(A + 10 * double)
    B = 300
    qn, qo = (rng.randint(-4, 4, (B, A)) / 4).astype(F32), lc.spread(rng, (B, A), -4, 4)
    qs = (rng.randint(-2, 2, (B, A)) / 2).astype(F32) if double else qn
    act = rng.randint(-1, A + 1, B).astype(np.int64)
    r = rng.randn(B) * 3
    go = (rng.rand(B) < 0.2).astype(np.uint8)
    tg = Buf(np.full((B, A), np.nan, F32))
    td = Buf(np.full(B, np.nan, F64))
    bufs = [Buf(x) for x in (qn, qs, qo, act, r, go)]
    call("cb200_dqn_td_targets", *(b.ptr for b in bufs), 0.99, B, A, tg.ptr, td.ptr)
    want_t, want_td = lr.dqn_td_targets(qn, qs, qo, act, r, go, 0.99)
    assert_bits(tg.get(), want_t, "targets")
    assert_bits(td.get(), want_td, "td_err")


# ---- (e) the contract ---------------------------------------------------------------------------------------------------
def test_argument_errors():
    L, lib = _lib()
    x = torch.zeros(1 << 16, device="cuda")
    p = x.data_ptr()
    st = L.current_stream()
    bad = [
        lib.cb200_colsum(p, 0, 4, p, p, st), lib.cb200_colsum(p, 4, 0, p, p, st), lib.cb200_colsum(None, 4, 4, p, p, st),
        lib.cb200_sumsq(p, 0, p, p, st), lib.cb200_sumsq(p, 4, p, None, st),
        lib.cb200_adam_tf(p, p, p, p, 0, 1e-3, 0.9, 0.99, 1e-4, 0.9, 0.99, st),
        lib.cb200_adam_tf_dev(p, p, p, p, 4, 1e-3, 0.9, 0.99, 1e-4, None, st),
        lib.cb200_polyak(p, p, 0, 0.5, st), lib.cb200_clip_by_global_norm(p, 4, p, 0.0, st),
        lib.cb200_clip_by_global_norm(p, 4, None, 1.0, st), lib.cb200_scale(p, 0, 1.0, st),
        lib.cb200_clip_by_value(p, 4, -1.0, st), lib.cb200_add_i64(None, 1, st),
        lib.cb200_regression_head_loss_grad(p, p, None, 0, 1, 1, 1.0, p, None, st),
        lib.cb200_regression_head_loss_grad(p, p, None, 1, 0, 1, 1.0, p, None, st),
        lib.cb200_dueling_combine_fwd(p, p, 0, 2, p, st), lib.cb200_dueling_combine_bwd(p, 2, 0, p, p, st),
        lib.cb200_dqn_td_targets(p, p, p, p, p, None, 0.99, 4, 2, p, p, st),
        lib.cb200_dqn_td_targets(p, p, p, p, p, p, 0.99, 4, 0, p, p, st),
        lib.cb200_act_backward(p, 3, p, 4, 2, 4, 1, p, 4, st), lib.cb200_act_backward(p, 4, p, 4, 0, 4, 1, p, 4, st),
        lib.cb200_axpby_2d(p, 4, 2, 4, 1.0, 0.0, p, 3, st), lib.cb200_axpby_2d(p, 4, 2, 0, 1.0, 0.0, p, 4, st),
        lib.cb200_split_planes(p, p, 12, p, 1, 64, st), lib.cb200_split_planes(p + 4, p, 8, p, 1, 64, st),
        lib.cb200_split_planes(p, p, 8, p, 0, 64, st),
        lib.cb200_permute_f32(p, p, 64, p, p, 72, 12, st), lib.cb200_permute_f32(p, p, 72, p, p, 80, 8, st),
        lib.cb200_u8_s2d_planes(p, 12, 8, 8, 4, 2, p, st), lib.cb200_u8_s2d_planes(p, 8, 8, 8, 2, 2, p, st),
        lib.cb200_u8_s2d_planes(p, 8, 9, 8, 4, 2, p, st),
        lib.cb200_transpose(p, 12, 8, p, p, 4096, st), lib.cb200_transpose(p, 16, 8, p, p, 4100, st),
        lib.cb200_transpose(p, 16, 9, p, p, 128, st),
    ]
    torch.cuda.synchronize()
    assert all(rc == -1 for rc in bad), [k for k, rc in enumerate(bad) if rc != -1]
    y = torch.zeros(1 << 12, device="cuda")
    assert lib.cb200_transpose(p, 16, 9, y.data_ptr(), y.data_ptr() + 4 * 256, 16 * 16, st) == 0
    torch.cuda.synchronize()


REQUIRED = {("split_planes", "grid-stride"), ("split_planes", "layout0"), ("split_planes", "layout1"),
            ("permute", "grid-stride"), ("transpose", "planes", True), ("transpose", "planes", False),
            ("u8_s2d", "grid-stride"), ("u8_s2d", "odd-x-pair"), ("u8_s2d", "s1"), ("u8_s2d", "s2"), ("u8_s2d", "s4"),
            ("colsum", "slab-cap"), ("colsum", "idle-lanes"), ("colsum", "column-blocks"), ("colsum", "stage2-lanes"),
            ("sumsq", "block-cap"), ("sumsq", "strided-thread"),
            ("regression", "rows-per-thread>1"), ("regression", "rows-per-thread=1"), ("regression", "idle-threads"),
            ("adam_dev", "vector"), ("adam_dev", "scalar"), ("adam_dev", "vector-grid-stride"),
            ("adam_dev", "scalar-grid-stride"), ("adam_dev", "graph"), ("polyak", "grid-stride"),
            ("clip", "grid-stride"), ("scale", "grid-stride")}


def test_every_path_ran():
    """every path named by the launch formulas of learn_ref ran in this session; a new path belongs in this list.  When
    only part of the file ran, the cases that reach the missing paths are run now."""
    if not REQUIRED <= RAN:
        test_split_planes(2048)
        test_permute_f32("perm", "tiled", 4800, 64)
        for r, c in ((8, 8), (8, 7)):
            test_transpose(r, c)
        for case in lc.U8_S2D_CASES:
            test_u8_s2d_planes(case)
        for r, c in ((10 ** 6, 32), (4096, 3), (4096, 257)):
            test_colsum(r, c)
        test_sumsq(4096 * 1024 + 1, False)
        test_regression_head_loss_grad(4096, 6, True, True, 1.0, True)
        test_regression_head_loss_grad(31, 6, False, False, 0.7, True)
        for n, off in (("big", 0), ("big+1", 0)):
            test_adam_five_steps(n, off, 2.5e-4)
        test_adam_dev_graph_replay_equals_eager_steps()
        test_polyak(5e-3, "big")
        test_clip_by_global_norm("above", "big")
        test_scale_and_clip_by_value("big")
    assert REQUIRED <= RAN, sorted(REQUIRED - RAN)
