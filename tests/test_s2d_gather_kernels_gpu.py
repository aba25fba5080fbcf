"""The fused sample + gather + space-to-depth kernel (sample_gather_s2d_kernel, replay.cu) at the C ABI, through
cb200_gather_s2d and cb200_per_sample_gather_s2d, against exact references at the shapes of tests/replay_cases.py:

  (a) the verbatim ring: every bf16 plane element bit for bit with tests/learn_ref.u8_s2d_plane of the gathered frames
      (bf16 holds 0..255 exactly), every small-column byte, and the canary bytes after every output; the launch-plan
      mirror (replay_ref.s2d_plan) names the band / chunk / conversion regime each case ran in;
  (b) prioritized sampling: indices bit for bit with the C oracle and with cb200_per_sample on the same tree and
      uniforms, importance weights (fp64 and fp32) bit for bit with cb200_per_sample, planes as in (a);
  (c) the frame store: the planes of replay_ref.gather_stack's stacks, with the frame_tma knob off and on, at every
      copy path replay_ref.s2d_one_box names (one 2-D TMA box, four per-frame copies, the partial-chunk fallback);
  (d) the contract: one launch per call, repeat calls and a CUDA-graph replay give the same bits, every argument error
      raises ValueError and writes nothing, and a final check that every regime of replay_cases.S2D_REQUIRED ran."""
import functools

import numpy as np
import pytest
import torch

import learn_ref as lr
import replay_cases as rc
import replay_ref as rr
from abi_util import _lib, assert_bits
from test_learn_kernels_gpu import FILL, Buf, call, canary16, sm

pytestmark = pytest.mark.gpu

RAN = set()
U8, I64, F64, F32 = np.uint8, np.int64, np.float64, np.float32
BETA = 0.4


@pytest.fixture
def frame_tma():
    """sets the process-global frame_tma knob of one test; it is off again whatever happens"""
    L, lib = _lib()
    try:
        yield lambda v: L.check(lib.cb200_tune(b"frame_tma", v))
    finally:
        lib.cb200_tune(b"frame_tma", 0)


@functools.lru_cache(maxsize=4)
def _ring(rows, row_bytes):
    rng = np.random.RandomState(rows % 9973 + row_bytes)
    return np.frombuffer(rng.bytes(rows * row_bytes), U8).reshape(rows, row_bytes)


def _planes(n, h, w, c, s, n_img):
    return [Buf(canary16(h * w * c * n)) for _ in range(n_img)]


def _small(kind, n, rows):
    """the small columns of a case: (src, dst, row_bytes), sources of `rows` rows, both bases at the case's offset"""
    spec = rc.SMALL_MIX if kind == "mix" else ()
    return [(Buf(_ring(rows, rb), off), Buf(np.full((n, rb), 0x5A, U8), off), rb) for rb, off in spec]


def _columns(img_src, planes, row_bytes, small):
    L, _ = _lib()
    img, n_img = L.make_columns([(s.ptr, p.ptr, row_bytes) for s, p in zip(img_src, planes)])
    sm_cols, n_small = L.make_columns([(s.ptr, d.ptr, rb) for s, d, rb in small]) if small else (None, 0)
    return img, n_img, sm_cols, n_small


def _check_outputs(planes, want_x, s, small, idx, rows, name):
    """planes against u8_s2d_plane of the gathered NHWC frames, small columns against the ring rows; Buf.get checks
    the canary bytes after every output"""
    for k, (p, x) in enumerate(zip(planes, want_x)):
        assert_bits(p.get(), lr.u8_s2d_plane(x, s), "%s: plane %d" % (name, k))
    for src, dst, rb in small:
        assert_bits(dst.get(), _ring(rows, rb)[idx], "%s: small column of %d bytes" % (name, rb))
        RAN.add(("copy", rr.copy_path(dst.ptr, src.ptr, rb)))
    RAN.add(("small", len(small)))


def _note(kind, plan, fidx_rows=None):
    RAN.update((kind, r) for r in plan["regimes"])
    if plan["frame_tma"] and fidx_rows is not None:
        full = rr.s2d_chunk_full(plan)
        RAN.update(("box", r) for r in rr.s2d_box_regimes(rr.s2d_one_box(fidx_rows, full), full))


# ---- (a) the verbatim ring -----------------------------------------------------------------------------------------------
def _ring_case(case, rep=1):
    n, n_img, h, w, c, s, small_kind = case
    L, lib = _lib()
    cap, row = rc.S2D_CAPACITY, h * w * c
    plan = rr.s2d_plan(n, n_img, h, w, c, s, sm())
    assert plan["refusal"] is None
    idx = rc.gather_idx(np.random.RandomState(n + row), n, cap)
    srcs = [Buf(_ring(cap + k, row)) for k in range(n_img)]
    planes = _planes(n, h, w, c, s, n_img)
    small = _small(small_kind, n, cap)
    img, n_img_, sm_cols, n_small = _columns(srcs, planes, row, small)
    d_idx = Buf(idx)
    name = "gather_s2d %s, regimes %s" % (case, sorted(plan["regimes"]))
    for _ in range(rep):
        call("cb200_gather_s2d", d_idx.ptr, n, img, n_img_, h, w, c, s, sm_cols, n_small, None, 0)
        _check_outputs(planes, [_ring(cap + k, row)[idx].reshape(n, h, w, c) for k in range(n_img)], s, small, idx,
                       cap, name)
    _note("ring", plan)


@pytest.mark.parametrize("case", rc.S2D_RING, ids=lambda c: "B%d_img%d_h%d_w%d_c%d_s%d_%s" % c)
def test_gather_s2d_ring(case):
    _ring_case(case)


# ---- (b) prioritized sampling --------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=2)
def _tree(size):
    leaves, m = rc.tree_leaves(np.random.RandomState(size + 1), size)
    return (rr.tree_from_leaves(leaves, rr.SUM), rr.tree_from_leaves(np.where(leaves > 0, leaves, np.inf), rr.MIN),
            m)


@pytest.mark.parametrize("case", rc.S2D_PER, ids=lambda c: "size%d_B%d_img%d_h%d_w%d_c%d_s%d_frames%d_%s" % (
    c[:8] + ("-".join(c[8]) or "none",)))
def test_per_sample_gather_s2d(case):
    size, n, n_img, h, w, c, s, frames, outs = case
    tree, mn, m = _tree(size)
    u = np.random.RandomState(size % 997 + n).rand(n)
    u[0], u[-1] = 0.0, np.nextafter(1.0, 0.0)
    idx_o, w_o = rr.oracle_sample(tree, mn, u, 2 * m, BETA)
    plan = rr.s2d_plan(n, n_img, h, w, c, s, sm(), frames, 64 if frames else 0)
    if frames:
        fidx = rc.frame_table(np.random.RandomState(size), size, 64)
        fr = np.frombuffer(np.random.RandomState(n).bytes(64 * h * w), U8).reshape(64, h * w)
        d_frames, srcs, row = Buf(fr), [Buf(fidx) for _ in range(n_img)], 4 * c
        want_x = [rr.gather_stack(fr, fidx, idx_o).reshape(n, h, w, c)] * n_img
    else:
        d_frames, row = None, h * w * c
        srcs = [Buf(_ring(size + k, row)) for k in range(n_img)]
        want_x = [_ring(size + k, row)[idx_o].reshape(n, h, w, c) for k in range(n_img)]
    planes = _planes(n, h, w, c, s, n_img)
    small = _small("mix" if size <= 128 else "none", n, size)
    img, n_img_, sm_cols, n_small = _columns(srcs, planes, row, small)
    d_s, d_m, d_u = Buf(tree), Buf(mn), Buf(u)
    d_idx = Buf(np.full(n, -7, I64))
    d_w = Buf(np.full(n, np.nan, F64)) if "w" in outs else None
    d_w32 = Buf(np.full(n, np.nan, F32)) if "w32" in outs else None
    call("cb200_per_sample_gather_s2d", d_s.ptr, d_m.ptr, size, d_u.ptr, n, 2 * m, BETA, d_idx.ptr,
         d_w.ptr if d_w else None, d_w32.ptr if d_w32 else None, img, n_img_, h, w, c, s, sm_cols, n_small,
         d_frames.ptr if frames else None, 64 if frames else 0)
    idx = d_idx.get()
    assert_bits(idx, idx_o, "indices against the oracle")
    d_idx2, d_w2, d_w322 = Buf(np.full(n, -7, I64)), Buf(np.full(n, np.nan, F64)), Buf(np.full(n, np.nan, F32))
    call("cb200_per_sample", d_s.ptr, d_m.ptr, size, d_u.ptr, n, 2 * m, BETA, d_idx2.ptr, d_w2.ptr, d_w322.ptr)
    assert_bits(d_idx2.get(), idx, "indices against cb200_per_sample")
    w2 = d_w2.get()
    assert rr.ulp_diff(w2, w_o).max() <= 4
    if d_w:
        assert_bits(d_w.get(), w2, "weights against cb200_per_sample")
    if d_w32:
        assert_bits(d_w32.get(), d_w322.get(), "fp32 weights against cb200_per_sample")
    _check_outputs(planes, want_x, s, small, idx_o, size, "per_sample_gather_s2d %s" % (case,))
    _note("frames" if frames else "ring", plan, fidx[idx_o] if frames else None)
    RAN.update(("per", o) for o in outs or ("no-weights",))
    RAN.add(("per", "size=%d" % size))
    if frames:
        RAN.add(("per", "frames"))


# ---- (c) the frame store -------------------------------------------------------------------------------------------------
def _frame_case(case, knob):
    """cb200_gather_s2d on a frame store; returns the plan, the outputs, the reference stacks, the sampled frame slots
    and the call's arguments (with the buffers they point into)"""
    n, n_img, h, w, slots, small_kind = case
    cap = rc.S2D_FRAME_CAPACITY
    rng = np.random.RandomState(n + h + slots)
    fidx = rc.frame_table(rng, cap, slots)
    idx = rc.frame_idx(rng, n, fidx)
    fr = np.frombuffer(rng.bytes(slots * h * w), U8).reshape(slots, h * w)
    plan = rr.s2d_plan(n, n_img, h, w, 4, 4, sm(), True, slots, knob)
    d_frames, d_idx = Buf(fr), Buf(idx)
    srcs = [Buf(fidx) for _ in range(n_img)]
    planes = _planes(n, h, w, 4, 4, n_img)
    small = _small(small_kind, n, cap)
    img, n_img_, sm_cols, n_small = _columns(srcs, planes, 16, small)
    args = (d_idx.ptr, n, img, n_img_, h, w, 4, 4, sm_cols, n_small, d_frames.ptr, slots)
    call("cb200_gather_s2d", *args)
    want = rr.gather_stack(fr, fidx, idx).reshape(n, h, w, 4)
    return plan, planes, small, want, fidx[idx], (args, d_frames, d_idx, srcs)


@pytest.mark.parametrize("knob", [0, 1], ids=["bulk", "tma"])
@pytest.mark.parametrize("case", rc.S2D_FRAMES, ids=lambda c: "B%d_img%d_h%d_w%d_slots%d_%s" % c)
def test_gather_s2d_frame_store(frame_tma, case, knob):
    frame_tma(knob)
    plan, planes, small, want, fidx_rows, (args, _, d_idx, _) = _frame_case(case, knob)
    name = "frame store %s knob %d, regimes %s" % (case, knob, sorted(plan["regimes"]))
    _check_outputs(planes, [want] * len(planes), 4, small, d_idx.get(), rc.S2D_FRAME_CAPACITY, name)
    _note("frames", plan, fidx_rows)


# ---- (d) the contract ----------------------------------------------------------------------------------------------------
def test_repeat_calls_and_graph_replay(frame_tma):
    """the Atari case with a partial chunk and empty bands twice in a row; then the frame-store case with a stage
    refill and TMA boxes eagerly, reset to canaries, captured in a CUDA graph (nothing runs) and replayed: the same
    bits each time"""
    L, lib = _lib()
    _ring_case((128, 2, 84, 84, 4, 4, "mix"), rep=2)
    frame_tma(1)
    plan, planes, small, want, _, (args, *keep) = _frame_case((512, 2, 84, 84, 64, "mix"), 1)
    assert plan["frame_tma"] and "refill" in plan["regimes"]
    outs = planes + [d for _, d, _ in small]
    eager = [b.get() for b in outs]
    for e in eager[:len(planes)]:
        assert_bits(e, lr.u8_s2d_plane(want, 4), "eager call before the capture")
    for b in outs:
        b.t.fill_(FILL)
    st = torch.cuda.Stream()
    st.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(st):
        torch.cuda.synchronize()
        with torch.cuda.graph(g, stream=st):
            c0 = lib.cb200_launch_count()
            L.check(lib.cb200_gather_s2d(*(args + (L.current_stream(),))))
            assert lib.cb200_launch_count() - c0 == 1
    torch.cuda.synchronize()
    assert all((b.t == FILL).all() for b in outs), "the capture ran the kernel"
    for rep in range(2):
        g.replay()
        for k, (b, e) in enumerate(zip(outs, eager)):
            assert_bits(b.get(), e, "graph replay %d, output %d" % (rep, k))
    RAN.add(("contract", "graph"))


def test_argument_errors():
    """every refusal raises ValueError, launches nothing and writes nothing; the library and torch work after them
    (a refused shared-memory size leaves no CUDA error behind)"""
    L, lib = _lib()
    n, h, w, c, s, cap = 8, 8, 8, 2, 4, 16
    row = h * w * c
    ring = Buf(_ring(cap, row))
    idx = Buf(np.arange(n, dtype=I64))
    plane = Buf(canary16(row * n))
    small = _small("mix", n, cap)
    sm_cols, n_small = L.make_columns([(sr.ptr, d.ptr, rb) for sr, d, rb in small])
    tree, mn, m = _tree(1 << 7)
    d_s, d_m, d_u = Buf(tree), Buf(mn), Buf(np.linspace(0, 0.99, 16))
    d_out_idx = Buf(np.full(16, -7, I64))
    fidx, frames = Buf(np.zeros((cap, 4), np.int32)), Buf(np.zeros((8, 4096), U8))

    def cols(src, dst, rb, k=1):
        return L.make_columns([(src, dst, rb)] * k) if k else (L.make_columns([(src, dst, rb)])[0], 0)

    # the geometries only the launch plan refuses: valid rings and planes, so nothing else trips
    big = {}
    for geo in (rc.S2D_OVER_SMEM, rc.S2D_S64):
        gn, _, gh, gw, gc, gs = geo
        big[geo] = (Buf(_ring(cap, gh * gw * gc)), Buf(canary16(gh * gw * gc * gn)))
    bad = [
        (12, cols(ring.ptr, plane.ptr, row), (h, w, c, s), None),                    # n % 8
        (n, cols(ring.ptr, plane.ptr, row, 0), (h, w, c, s), None),                  # no image column
        (n, cols(ring.ptr, plane.ptr, row, 3), (h, w, c, s), None),                  # three image columns
        (n, cols(ring.ptr + 1, plane.ptr, row), (h, w, c, s), None),                 # unaligned ring
        (n, cols(ring.ptr, plane.ptr + 8, row), (h, w, c, s), None),                 # unaligned plane
        (n, cols(ring.ptr, plane.ptr, row + 16), (h, w, c, s), None),                # row_bytes != h w c
        (n, cols(fidx.ptr, plane.ptr, 4 * 4), (8, 8, 4, 2), frames.ptr),             # frame store with s != 4
        (n, cols(fidx.ptr, plane.ptr, 4 * 2), (8, 8, 2, 4), frames.ptr),             # frame store with c != 4
    ]
    for geo, (src, pl) in big.items():
        gn, _, gh, gw, gc, gs = geo
        assert rr.s2d_plan(*geo, sm())["refusal"] == ("smem" if geo == rc.S2D_OVER_SMEM else "s>32")
        bad.append((gn, cols(src.ptr, pl.ptr, gh * gw * gc), (gh, gw, gc, gs), None))
    c0 = lib.cb200_launch_count()
    for k, (bn, (img, ni), geom, fr) in enumerate(bad):
        with pytest.raises(ValueError):
            L.check(lib.cb200_gather_s2d(idx.ptr, bn, img, ni, *geom, sm_cols, n_small, fr, 8 if fr else 0,
                                         L.current_stream()))
        with pytest.raises(ValueError):
            L.check(lib.cb200_per_sample_gather_s2d(d_s.ptr, d_m.ptr, 1 << 7, d_u.ptr, bn, 2 * m, BETA, d_out_idx.ptr,
                                                    None, None, img, ni, *geom, sm_cols, n_small, fr, 8 if fr else 0,
                                                    L.current_stream()))
    # the sampler's own refusals: a tree size that is not a power of 2, no idx_out
    img, ni = cols(ring.ptr, plane.ptr, row)
    for size, out in ((6, d_out_idx.ptr), (1 << 7, None)):
        with pytest.raises(ValueError):
            L.check(lib.cb200_per_sample_gather_s2d(d_s.ptr, d_m.ptr, size, d_u.ptr, n, 2 * m, BETA, out, None, None,
                                                    img, ni, h, w, c, s, sm_cols, n_small, None, 0,
                                                    L.current_stream()))
    with pytest.raises(ValueError):
        L.check(lib.cb200_gather_s2d(None, n, img, ni, h, w, c, s, sm_cols, n_small, None, 0, L.current_stream()))
    assert lib.cb200_launch_count() == c0, "a refused call launched"
    assert_bits(plane.get(), canary16(row * n), "plane after refusals")
    for _, pl in big.values():
        assert_bits(pl.get(), canary16(pl.nb // 2), "plane of a refused geometry")
    for _, d, rb in small:
        assert (d.get() == 0x5A).all(), "small column of %d bytes after refusals" % rb
    assert (d_out_idx.get() == -7).all()
    # a valid call, and torch, still work
    torch.zeros(16, device="cuda").add_(1)
    call("cb200_gather_s2d", idx.ptr, n, img, ni, h, w, c, s, sm_cols, n_small, None, 0)
    _check_outputs([plane], [_ring(cap, row)[np.arange(n)].reshape(n, h, w, c)], s, small, np.arange(n), cap,
                   "after the refusals")


def test_every_regime_ran(frame_tma):
    """every regime of replay_cases.S2D_REQUIRED ran in this session; a new regime belongs in that list.  When only
    part of the file ran, the cases that reach the missing ones are run now."""
    if not rc.S2D_REQUIRED <= RAN:
        for case in rc.S2D_RING:
            if case[0] < 4096:
                _ring_case(case)
        for case in rc.S2D_PER:
            test_per_sample_gather_s2d(case)
        for case in rc.S2D_FRAMES:
            for knob in (0, 1):
                test_gather_s2d_frame_store(frame_tma, case, knob)
    assert rc.S2D_REQUIRED <= RAN, sorted(rc.S2D_REQUIRED - RAN)
