"""The replay kernels at the C ABI against tests/replay_ref.py, at the shapes and edges of tests/replay_cases.py:

  (a) row copies (cb200_gather, cb200_per_sample_gather, cb200_gather_at, cb200_gather_stack, cb200_scatter_ring /
      _packed): every output byte, and the canary bytes around every output, over the gather_ctas_per_sm x
      gather_stages knob grid; the launch-plan mirror names the pipeline regime each case ran in;
  (b) segment trees (cb200_per_init, per_store, per_update, per_sample): every node bit for bit against the C oracle at
      every update path, indices bit for bit, importance weights within 4 ulp;
  (c) priorities (cb200_per_priorities_device, cb200_host_priorities): device pow within 2 ulp of Python's **, host
      bit for bit, invalid errors flagged / refused;
  (d) the contract: argument errors, repeat calls, cb200_launch_count deltas, and a final check that every path
      named by the mirrors ran."""
import functools

import numpy as np
import pytest
import torch

import replay_cases as rc
import replay_ref as rr
from abi_util import _lib, assert_bits
from test_learn_kernels_gpu import Buf, call, sm

pytestmark = pytest.mark.gpu

RAN = set()
U8, F64, I64 = np.uint8, np.float64, np.int64
TUNE_DEFAULTS = {"gather_ctas_per_sm": rr.DEFAULT_CTAS_PER_SM, "gather_stages": 0, "per_update_sorted": 1}
BETA = 0.4


@pytest.fixture
def tune():
    """sets the process-global tune knobs of one test; the defaults come back whatever happens"""
    L, lib = _lib()

    def set_knob(key, value):
        L.check(lib.cb200_tune(key.encode(), value))
    try:
        yield set_knob
    finally:
        for k, v in TUNE_DEFAULTS.items():
            lib.cb200_tune(k.encode(), v)


@functools.lru_cache(maxsize=None)
def _ring(row_bytes, rows=rc.CAPACITY):
    return rc.ring(np.random.RandomState(row_bytes), rows, row_bytes)


def _columns(row_list, n, idx, off=0, rows=rc.CAPACITY):
    """device rings and outputs (src and dst bases `off` bytes past 256-byte alignment) and the column table"""
    L, _ = _lib()
    srcs = [Buf(_ring(rb, rows), off) for rb in row_list]
    dsts = [Buf(np.full((n, rb), 0x5A, U8), off) for rb in row_list]
    arr, cnt = L.make_columns([(s.ptr, d.ptr, rb) for s, d, rb in zip(srcs, dsts, row_list)])
    want = [_ring(rb, rows)[idx] for rb in row_list]
    return arr, cnt, srcs, dsts, want


def _note_plan(plan, kind):
    RAN.update((kind, r) for r in rr.pipeline_regimes(plan))
    if plan["big"]:
        RAN.add(("gather", "bulk"))
    if plan["small"]:
        RAN.add(("gather", "small"))


# ---- (a) row copies ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", rc.GATHER_N)
@pytest.mark.parametrize("off", rc.OFFSETS)
@pytest.mark.parametrize("row_bytes", rc.ROW_BYTES)
def test_gather_rows(row_bytes, off, n):
    """one column at default knobs: bulk and LSU rows, 16-byte / 4-byte / byte alignment, duplicates and both ends
    of the ring"""
    idx = rc.gather_idx(np.random.RandomState(n + row_bytes), n, rc.CAPACITY)
    arr, cnt, srcs, dsts, want = _columns([row_bytes], n, idx, off)
    d_idx = Buf(idx)
    plan = rr.gather_plan([(row_bytes, srcs[0].ptr, dsts[0].ptr)], n, sm())
    call("cb200_gather", arr, cnt, d_idx.ptr, n, launches=rr.gather_launches(plan))
    assert_bits(dsts[0].get(), want[0], "gather %d bytes" % row_bytes)
    _note_plan(plan, "pipeline")
    if plan["small"]:
        RAN.add(("copy", rr.copy_path(dsts[0].ptr, srcs[0].ptr, row_bytes)))


@pytest.mark.parametrize("n", rc.MIX_N + (rc.WIDE_N,))
@pytest.mark.parametrize("ctas,stages", rc.KNOB_GRID)
def test_gather_knob_grid(tune, ctas, stages, n):
    """eight columns (four bulk, four LSU) at n = 7 and 512, and one Atari column at n = 4096, at every knob setting:
    one-stage pipelines with several items per CTA, stages refilled many times, everything in flight at once"""
    tune("gather_ctas_per_sm", ctas)
    tune("gather_stages", stages)
    rows = rc.WIDE if n == rc.WIDE_N else rc.MIX
    idx = rc.gather_idx(np.random.RandomState(ctas * 10 + stages + n), n, rc.CAPACITY)
    arr, cnt, srcs, dsts, want = _columns(rows, n, idx)
    d_idx = Buf(idx)
    plan = rr.gather_plan([(rb, s.ptr, d.ptr) for rb, s, d in zip(rows, srcs, dsts)], n, sm(), ctas, stages)
    for rep in range(2):
        call("cb200_gather", arr, cnt, d_idx.ptr, n, launches=rr.gather_launches(plan))
        got = [d.get() for d in dsts]
        for c, (g, w) in enumerate(zip(got, want)):
            assert_bits(g, w, "column %d (%d bytes), call %d" % (c, rows[c], rep))
    _note_plan(plan, "pipeline")


@functools.lru_cache(maxsize=None)
def _sample_tree(size):
    leaves, m = rc.tree_leaves(np.random.RandomState(size + 1), size)
    return (rr.tree_from_leaves(leaves, rr.SUM), rr.tree_from_leaves(np.where(leaves > 0, leaves, np.inf), rr.MIN),
            m)


def _fused(row_list, n, ctas, stages, u_seed, outs=("w", "w32")):
    """cb200_per_sample_gather on a 1024-leaf tree over a ring of as many rows, checked against the oracle, against
    cb200_per_sample on the same tree and against the ring rows; returns the launch plan"""
    size = 1024
    s, mn, m = _sample_tree(size)
    u = np.random.RandomState(u_seed).rand(n)
    u[0], u[-1] = 0.0, np.nextafter(1.0, 0.0)
    d_s, d_m, d_u = Buf(s), Buf(mn), Buf(u)
    d_idx = Buf(np.full(n, -7, I64))
    d_w = Buf(np.full(n, np.nan, F64)) if "w" in outs else None
    d_w32 = Buf(np.full(n, np.nan, np.float32)) if "w32" in outs else None
    idx_o, w_o = rr.oracle_sample(s, mn, u, 2 * m, BETA)
    arr, cnt, srcs, dsts, want = _columns(row_list, n, idx_o, rows=size)
    cols = [(rb, sr.ptr, d.ptr) for rb, sr, d in zip(row_list, srcs, dsts)]
    plan = rr.gather_plan(cols, n, sm(), ctas, stages, fused=True)
    fallback = rr.fused_fallback(plan)
    launches = 1 + rr.gather_launches(rr.gather_plan(cols, n, sm(), ctas, stages)) if fallback else 1
    call("cb200_per_sample_gather", d_s.ptr, d_m.ptr, size, d_u.ptr, n, 2 * m, BETA, d_idx.ptr,
         d_w.ptr if d_w else None, d_w32.ptr if d_w32 else None, arr, cnt, launches=launches)
    idx = d_idx.get()
    assert_bits(idx, idx_o, "indices against the oracle")
    # the unfused sampler on the same tree draws the same leaves and weights
    d_idx2, d_w2 = Buf(np.full(n, -7, I64)), Buf(np.full(n, np.nan, F64))
    call("cb200_per_sample", d_s.ptr, d_m.ptr, size, d_u.ptr, n, 2 * m, BETA, d_idx2.ptr, d_w2.ptr, None)
    assert_bits(d_idx2.get(), idx, "indices against cb200_per_sample")
    w2 = d_w2.get()
    assert rr.ulp_diff(w2, w_o).max() <= 4
    if d_w:
        assert_bits(d_w.get(), w2, "weights against cb200_per_sample")
    if d_w32:
        assert_bits(d_w32.get(), w2.astype(np.float32), "fp32 weights")
    for c, (d, w) in enumerate(zip(dsts, want)):
        assert_bits(d.get(), w, "column %d (%d bytes)" % (c, row_list[c]))
    if not fallback:
        _, count = rr.fused_owners(plan, n)
        assert (count == 1).all(), "a sample's small columns must be copied by exactly one CTA"
        RAN.add(("fused", "fused"))
        _note_plan(plan, "fused")
    else:
        RAN.add(("fused", "fallback"))
    return plan


@pytest.mark.parametrize("n", rc.MIX_N)
@pytest.mark.parametrize("ctas,stages", rc.KNOB_GRID)
def test_per_sample_gather_knob_grid(tune, ctas, stages, n):
    tune("gather_ctas_per_sm", ctas)
    tune("gather_stages", stages)
    _fused(rc.MIX, n, ctas, stages, ctas + stages + n)


def test_per_sample_gather_fallback(tune):
    """one 2048-byte column, n = 4096, one CTA per SM: 32 samples per CTA exceed kMaxCtaSamples, so the call samples
    and then gathers (two launches)"""
    tune("gather_ctas_per_sm", 1)
    plan = _fused((2048,), 4096, 1, 0, 3)
    assert rr.fused_fallback(plan)


@pytest.mark.parametrize("outs", [("w",), ("w32",), ()])
def test_per_sample_gather_optional_weights(outs):
    _fused((rc.ATARI, 8, 1), 64, rr.DEFAULT_CTAS_PER_SM, 0, 11, outs)


@pytest.mark.parametrize("where", ["start", "middle", "end"])
@pytest.mark.parametrize("with_idx", [True, False])
@pytest.mark.parametrize("off", [0, 1])
def test_gather_at(where, with_idx, off):
    """dst[c][i] = src[c][idx[*offset + i]] (idx NULL: row *offset + i) for a device offset at the start, the middle
    and the end of idx; 4-byte rows (68, 1040 bytes) and byte rows (3 bytes, or a base one byte off)"""
    n, total = 100, 300
    offset = {"start": 0, "middle": 137, "end": total - n}[where]
    rng = np.random.RandomState(offset + 2 * with_idx + off)
    perm = rng.permutation(rc.CAPACITY)[:total].astype(I64)
    perm[offset + n - 1] = rc.CAPACITY - 1
    rows_used = perm[offset:offset + n] if with_idx else np.arange(offset, offset + n)
    row_list = (68, 1040, 3)
    arr, cnt, srcs, dsts, want = _columns(row_list, n, rows_used, off)
    d_perm, d_off = Buf(perm), Buf(np.array([offset], I64))
    call("cb200_gather_at", arr, cnt, d_perm.ptr if with_idx else None, d_off.ptr, n)
    for c, (d, w) in enumerate(zip(dsts, want)):
        assert_bits(d.get(), w, "gather_at column %d" % c)
        RAN.add(("gather_at", 4 if rr.copy_path(d.ptr, srcs[c].ptr, row_list[c]) in (4, 16) else 1))
    RAN.add(("gather_at", "idx" if with_idx else "rows"))


@pytest.mark.parametrize("stack", [1, 2, 3, 4])
@pytest.mark.parametrize("frame_bytes", [7057, 7056])
def test_gather_stack(stack, frame_bytes):
    """out[i, pix, c] = frames[frame_index[idx[i], c], pix]: frame sizes that are not word multiples, stacks that
    repeat one frame slot (an episode start), and repeated transitions"""
    rng = np.random.RandomState(stack * 10 + frame_bytes % 7)
    slots, cap, n = 40, 50, 64
    frames = rng.randint(0, 256, (slots, frame_bytes)).astype(U8)
    fidx = rng.randint(0, slots, (cap, stack)).astype(np.int32)
    fidx[0] = 0                                    # every frame of the stack in slot 0
    fidx[1] = slots - 1
    idx = rc.gather_idx(rng, n, cap)
    idx[5] = 0
    d_f, d_fi, d_idx = Buf(frames), Buf(fidx), Buf(idx)
    out = Buf(np.full((n, frame_bytes, stack), 0x5A, U8))
    call("cb200_gather_stack", d_f.ptr, frame_bytes, d_fi.ptr, stack, d_idx.ptr, n, out.ptr)
    assert_bits(out.get(), rr.gather_stack(frames, fidx, idx), "gather_stack")


SCATTER_ROWS = (3, 68, 4100)                     # byte rows, word rows, a row of two 4 KiB pieces with a 4-byte tail


@pytest.mark.parametrize("cursor,n", [(0, 0), (0, 5), (30, 5), (35, 10), (0, 37), (20, 37)])
def test_scatter_ring(cursor, n):
    """ring[(cursor + i) % capacity] = staged[i]: the cursor wraps, n == capacity, rows outside the written range keep
    their bytes"""
    L, _ = _lib()
    cap = 37
    rng = np.random.RandomState(cursor * 40 + n)
    rings0 = [rc.ring(rng, cap, rb) for rb in SCATTER_ROWS]
    staged = [rc.ring(rng, max(n, 1), rb) for rb in SCATTER_ROWS]
    d_rings, d_staged = [Buf(r) for r in rings0], [Buf(s) for s in staged]
    arr, cnt = L.make_columns([(r.ptr, s.ptr, rb) for r, s, rb in zip(d_rings, d_staged, SCATTER_ROWS)])
    call("cb200_scatter_ring", arr, cnt, cursor, cap, n, launches=len(SCATTER_ROWS) if n else 0)
    for r, r0, s in zip(d_rings, rings0, staged):
        assert_bits(r.get(), rr.scatter_ring(r0, s, cursor, n), "scatter_ring")
    # the packed staging area: one record per transition, the columns back to back, an odd record stride
    stride = sum(SCATTER_ROWS) + 1
    rec = np.full((max(n, 1), stride), 0xEE, U8)
    col_off = np.cumsum((0,) + SCATTER_ROWS[:-1])
    for o, s, rb in zip(col_off, staged, SCATTER_ROWS):
        rec[:, o:o + rb] = s
    d_rec = Buf(rec)
    d_rings = [Buf(r) for r in rings0]
    arr, cnt = L.make_columns([(r.ptr, d_rec.ptr + int(o), rb) for r, o, rb in zip(d_rings, col_off, SCATTER_ROWS)])
    call("cb200_scatter_ring_packed", arr, cnt, stride, cursor, cap, n, launches=1 if n else 0)
    for r, r0, s in zip(d_rings, rings0, staged):
        assert_bits(r.get(), rr.scatter_ring(r0, s, cursor, n), "scatter_ring_packed")
    if cursor + n > cap:
        RAN.add(("scatter", "wrap"))
    if n == cap:
        RAN.add(("scatter", "full"))


# ---- (b) segment trees -------------------------------------------------------------------------------------------------
def _trees(trees, size):
    return [Buf(t) for t in trees] + [Buf(np.full(size, -1, np.int32))]


@pytest.mark.parametrize("size", rc.TREE_SIZES)
def test_per_init(size):
    bufs = [Buf(np.full(2 * size - 1, 7.0)) for _ in range(3)] + [Buf(np.zeros(size, np.int32))]
    call("cb200_per_init", *(b.ptr for b in bufs), size)
    for op, (b, t) in enumerate(zip(bufs, rr.oracle_init(size))):
        assert_bits(b.get(), t, "init tree %d" % op)
    assert (bufs[3].get() == -1).all()


@functools.lru_cache(maxsize=None)
def _start_trees(size):
    leaves, m = rc.tree_leaves(np.random.RandomState(size), size)
    raw = leaves * 3
    return (rr.tree_from_leaves(leaves, rr.SUM), rr.tree_from_leaves(np.where(leaves > 0, leaves, np.inf), rr.MIN),
            rr.tree_from_leaves(np.where(leaves > 0, raw, -np.inf), rr.MAX))


UPDATE_CASES = [(s, n, k) for s in rc.TREE_SIZES for n in rc.UPDATE_N for k in (1, 0)] + [(1 << 20, 512, 1)]


@pytest.mark.parametrize("size,n,sorted_knob", UPDATE_CASES)
def test_per_update(tune, size, n, sorted_knob):
    """last writer wins among duplicates, a negative p_alpha (the invalid-error marker) and an out-of-range leaf are
    skipped, the latter flagged in bit 1; every node of the three trees, max_priority_out and the winner scratch (back
    at -1) bit for bit, at every update path"""
    tune("per_update_sorted", sorted_knob)
    rng = np.random.RandomState(size % 9973 + n + sorted_knob)
    idx, pa, pr = rc.update_batch(rng, n, size)
    if n >= 3:
        pa[1] = pr[1] = -1.0
        idx[2] = size if n % 2 else -1
    want = [t.copy() for t in _start_trees(size)]
    flags = rr.oracle_update(want, idx, pa, pr)
    bufs = _trees(_start_trees(size), size)
    d_idx, d_pa, d_pr = Buf(idx), Buf(pa), Buf(pr)
    d_max, d_flags = Buf(np.full(1, np.nan)), Buf(np.zeros(1, np.int32))
    path = rr.update_path(n, size, sorted_knob)
    call("cb200_per_update", *(b.ptr for b in bufs), size, d_idx.ptr, d_pa.ptr, d_pr.ptr, n, d_max.ptr, d_flags.ptr,
         launches=rr.update_launches(n, size, sorted_knob))
    for op, (b, t) in enumerate(zip(bufs, want)):
        assert_bits(b.get(), t, "tree %d (%s path)" % (op, path))
    assert (bufs[3].get() == -1).all(), "winner scratch not restored"
    assert d_flags.get()[0] == flags
    if path != "none":
        assert_bits(d_max.get(), want[2][:1], "max_priority_out")
    RAN.add(("update", path))
    if path == "cta" and n <= rr.UPD_SORT_THREADS:
        RAN.add(("update", "cta-by-knob" if not sorted_knob else "cta-by-depth"))


STORE_CASES = [(s, n) for s in rc.TREE_SIZES for n in sorted({0, 1, 512, 513, 1025, s}) if n <= s]


@pytest.mark.parametrize("size,n", STORE_CASES)
def test_per_store(size, n):
    """n consecutive leaves from a cursor three slots before the end (wrapping), n == size included"""
    cursor = max(size - 3, 0)
    want = [t.copy() for t in _start_trees(size)]
    p_alpha = rr.oracle_store(want, cursor, n, 1.5, 0.6)
    bufs = _trees(_start_trees(size), size)
    call("cb200_per_store", *(b.ptr for b in bufs), size, cursor, n, p_alpha, 1.5,
         launches=rr.update_launches(n, size, 1, max_out=False))
    for op, (b, t) in enumerate(zip(bufs, want)):
        assert_bits(b.get(), t, "tree %d" % op)
    assert (bufs[3].get() == -1).all()
    RAN.add(("store", rr.update_path(n, size)))
    if cursor + n > size:
        RAN.add(("store", "wrap"))


@pytest.mark.parametrize("n", rc.SAMPLE_N)
@pytest.mark.parametrize("size", rc.TREE_SIZES)
def test_per_sample(size, n):
    """indices bit for bit with the oracle (u = 0 and nextafter(1, 0) included); a zero-priority leaf only for the
    last draw, whose value rounds to the tree total, and then the last leaf, as in the reference; weights within 4 ulp
    of the oracle, their fp32 copy the rounding of the device's own fp64 weight"""
    s, mn, m = _sample_tree(size)
    u = np.random.RandomState(size % 997 + n).rand(n)
    u[0], u[-1] = 0.0, np.nextafter(1.0, 0.0)
    idx_o, w_o = rr.oracle_sample(s, mn, u, 2 * m, BETA)
    d_s, d_m, d_u = Buf(s), Buf(mn), Buf(u)
    d_idx, d_w, d_w32 = Buf(np.full(n, -7, I64)), Buf(np.full(n, np.nan)), Buf(np.full(n, np.nan, np.float32))
    call("cb200_per_sample", d_s.ptr, d_m.ptr, size, d_u.ptr, n, 2 * m, BETA, d_idx.ptr, d_w.ptr, d_w32.ptr)
    idx, w = d_idx.get(), d_w.get()
    assert_bits(idx, idx_o, "indices")
    tail = idx >= m
    assert not tail[:-1].any() and (idx[tail] == size - 1).all()
    if tail.any():
        RAN.add(("sample", "zero-priority-tail"))
    assert rr.ulp_diff(w, w_o).max() <= 4
    assert_bits(d_w32.get(), w.astype(np.float32), "fp32 weights")
    RAN.add(("descent", sum(rr.descent_rounds(size))))


# ---- (c) priorities ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [0, 1, 1000])
@pytest.mark.parametrize("invalid", [None, "negative", "nan"])
def test_priorities(n, invalid):
    L, lib = _lib()
    rng = np.random.RandomState(n)
    err = np.abs(rng.randn(n)) * 2.0 ** rng.uniform(-20, 4, n)
    if n:
        err[0] = 0.0
    if invalid == "negative" and n:
        err[-1] = -0.5
        err[n // 2] = -1e-300
    elif invalid == "nan" and n:
        err[-1] = np.nan
    bad = ~(err >= 0)
    eps, alpha = 1e-6, 0.6
    want_a, want_r = rr.host_priorities(err, eps, alpha)
    d_err, d_pa, d_pr = Buf(err), Buf(np.full(n, np.nan)), Buf(np.full(n, np.nan))
    d_flag = Buf(np.zeros(1, np.int32))
    call("cb200_per_priorities_device", d_err.ptr, n, eps, alpha, d_pa.ptr, d_pr.ptr, d_flag.ptr,
         launches=1 if n else 0)
    pa, pr = d_pa.get(), d_pr.get()
    assert d_flag.get()[0] == int(bad.any())
    assert (pa[bad] == -1).all() and (pr[bad] == -1).all()
    assert_bits(pr[~bad], want_r[~bad], "p_raw")
    assert rr.ulp_diff(pa[~bad], want_a[~bad]).max(initial=0) <= 2
    # host: libm pow, bit for bit; an invalid error refuses the whole batch and writes nothing
    h_a, h_r = np.full(n, 7.0), np.full(n, 7.0)
    rc_ = lib.cb200_host_priorities(err.ctypes.data, n, eps, alpha, h_a.ctypes.data, h_r.ctypes.data)
    if bad.any():
        assert rc_ == -1 and (h_a == 7.0).all() and (h_r == 7.0).all()
    else:
        assert rc_ == 0
        assert_bits(h_a, want_a, "host p_alpha")
        assert_bits(h_r, want_r, "host p_raw")


# ---- (d) the contract --------------------------------------------------------------------------------------------------
def test_argument_errors():
    L, lib = _lib()
    x = torch.zeros(1 << 16, dtype=torch.float64, device="cuda")
    p = x.data_ptr()
    st = L.current_stream()
    ok_cols, _ = L.make_columns([(p, p + 8192, 64)])
    bad_cols, _ = L.make_columns([(p, None, 64)])
    nine = (_lib()[0].Column * 9)()
    for c in nine:
        c.src, c.dst, c.row_bytes = p, p + 8192, 64
    bad = [
        lib.cb200_per_init(p, p, p, p, 3, st), lib.cb200_per_init(p, p, None, p, 4, st),
        lib.cb200_per_init(p, p, p, p, 0, st),
        lib.cb200_per_update(p, p, p, p, 6, p, p, p, 1, None, None, st),
        lib.cb200_per_update(p, p, p, None, 8, p, p, p, 1, None, None, st),
        lib.cb200_per_update(p, p, p, p, 8, None, p, p, 1, None, None, st),
        lib.cb200_per_update(p, p, p, p, 8, p, p, p, -1, None, None, st),
        lib.cb200_per_store(p, p, p, p, 8, 0, 9, 1.0, 1.0, st), lib.cb200_per_store(p, p, p, p, 8, 8, 1, 1.0, 1.0, st),
        lib.cb200_per_store(p, p, p, p, 12, 0, 1, 1.0, 1.0, st), lib.cb200_per_store(None, p, p, p, 8, 0, 1, 1.0, 1.0, st),
        lib.cb200_per_sample(p, p, 6, p, 4, 8, 0.4, p, None, None, st),
        lib.cb200_per_sample(p, p, 8, p, 0, 8, 0.4, p, None, None, st),
        lib.cb200_per_sample(p, p, 8, p, 4, 8, 0.4, None, None, None, st),
        lib.cb200_per_sample(p, p, 8, None, 4, 8, 0.4, p, None, None, st),
        lib.cb200_per_priorities_device(None, 4, 1e-6, 0.6, p, p, None, st),
        lib.cb200_per_priorities_device(p, -1, 1e-6, 0.6, p, p, None, st),
        lib.cb200_host_priorities(None, 4, 1e-6, 0.6, None, None),
        lib.cb200_gather(ok_cols, 0, p, 4, st), lib.cb200_gather(nine, 9, p, 4, st),
        lib.cb200_gather(ok_cols, 1, None, 4, st), lib.cb200_gather(ok_cols, 1, p, 0, st),
        lib.cb200_gather(bad_cols, 1, p, 4, st), lib.cb200_gather(None, 1, p, 4, st),
        lib.cb200_per_sample_gather(p, p, 8, p, 4, 8, 0.4, p, None, None, ok_cols, 0, st),
        lib.cb200_per_sample_gather(p, p, 8, p, 4, 8, 0.4, p, None, None, nine, 9, st),
        lib.cb200_per_sample_gather(p, p, 8, p, 4, 8, 0.4, None, None, None, ok_cols, 1, st),
        lib.cb200_per_sample_gather(p, p, 6, p, 4, 8, 0.4, p, None, None, ok_cols, 1, st),
        lib.cb200_per_sample_gather(p, p, 8, p, 4, 8, 0.4, p, None, None, bad_cols, 1, st),
        lib.cb200_gather_at(ok_cols, 0, p, p, 4, st), lib.cb200_gather_at(nine, 9, p, p, 4, st),
        lib.cb200_gather_at(ok_cols, 1, p, p, 0, st), lib.cb200_gather_at(bad_cols, 1, p, p, 4, st),
        lib.cb200_gather_stack(None, 64, p, 4, p, 4, p, st), lib.cb200_gather_stack(p, 0, p, 4, p, 4, p, st),
        lib.cb200_gather_stack(p, 64, p, 0, p, 4, p, st), lib.cb200_gather_stack(p, 64, p, 4, None, 4, p, st),
        lib.cb200_scatter_ring(ok_cols, 0, 0, 8, 1, st), lib.cb200_scatter_ring(nine, 9, 0, 8, 1, st),
        lib.cb200_scatter_ring(ok_cols, 1, 8, 8, 1, st), lib.cb200_scatter_ring(ok_cols, 1, 0, 8, 9, st),
        lib.cb200_scatter_ring(bad_cols, 1, 0, 8, 1, st),
        lib.cb200_scatter_ring_packed(ok_cols, 1, 32, 0, 8, 1, st),
        lib.cb200_scatter_ring_packed(ok_cols, 1, 64, 0, 8, 9, st),
        lib.cb200_scatter_ring_packed(nine, 9, 64, 0, 8, 1, st),
    ]
    torch.cuda.synchronize()
    assert all(r == -1 for r in bad), [k for k, r in enumerate(bad) if r != -1]


def test_repeat_calls_give_the_same_bytes():
    """tree update on the level path and the fused sample + gather, twice from the same inputs"""
    size, n = 1 << 14, 1025
    idx, pa, pr = rc.update_batch(np.random.RandomState(9), n, size)
    got = []
    for _ in range(2):
        bufs = _trees(_start_trees(size), size)
        d = [Buf(x) for x in (idx, pa, pr)]
        call("cb200_per_update", *(b.ptr for b in bufs), size, d[0].ptr, d[1].ptr, d[2].ptr, n, None, None,
             launches=rr.update_launches(n, size, max_out=False))
        got.append([b.get() for b in bufs])
    for a, b in zip(*got):
        assert_bits(a, b, "repeat update")
    _fused(rc.MIX, 512, rr.DEFAULT_CTAS_PER_SM, 0, 5)
    _fused(rc.MIX, 512, rr.DEFAULT_CTAS_PER_SM, 0, 5)


REQUIRED = {("gather", "bulk"), ("gather", "small"), ("copy", 16), ("copy", 4), ("copy", 1),
            ("pipeline", "one-stage-multi"), ("pipeline", "reuse>=3"), ("pipeline", "all-in-flight"),
            ("pipeline", "refill"), ("fused", "fused"), ("fused", "fallback"), ("fused", "one-stage-multi"),
            ("fused", "refill"), ("gather_at", "idx"), ("gather_at", "rows"), ("gather_at", 4), ("gather_at", 1),
            ("scatter", "wrap"), ("scatter", "full"),
            ("update", "none"), ("update", "sorted"), ("update", "cta"), ("update", "levels"),
            ("update", "cta-by-knob"), ("update", "cta-by-depth"),
            ("store", "none"), ("store", "sorted"), ("store", "cta"), ("store", "levels"), ("store", "wrap"),
            ("descent", 0), ("descent", 1), ("descent", 7), ("descent", 14), ("descent", 21),
            ("sample", "zero-priority-tail")}


def test_every_path_ran(tune):
    """every regime the mirrors name ran in this session; a new regime belongs in this list.  When only part of the
    file ran, the cases that reach the missing ones are run now."""
    if not REQUIRED <= RAN:
        for rb, off in ((1040, 0), (68, 0), (3, 0), (rc.ATARI, 0)):
            test_gather_rows(rb, off, 512)
        for ctas, stages, n in ((1, 1, 512), (1, 0, rc.WIDE_N), (4, 0, 7)):
            test_gather_knob_grid(tune, ctas, stages, n)
        test_per_sample_gather_knob_grid(tune, 14, 0, 512)
        test_per_sample_gather_knob_grid(tune, 1, 2, 512)
        test_per_sample_gather_fallback(tune)
        tune("gather_ctas_per_sm", rr.DEFAULT_CTAS_PER_SM)
        tune("gather_stages", 0)
        for w, i, o in (("start", True, 0), ("end", False, 1)):
            test_gather_at(w, i, o)
        test_scatter_ring(20, 37)
        for size, n, k in ((1 << 7, 0, 1), (1 << 7, 512, 1), (1 << 7, 512, 0), (1 << 21, 512, 1), (1 << 7, 1025, 1)):
            test_per_update(tune, size, n, k)
        for size, n in ((1 << 7, 0), (1 << 7, 1), (1 << 14, 513), (1 << 14, 1025)):
            test_per_store(size, n)
        for size in rc.TREE_SIZES:
            test_per_sample(size, 513)
    assert REQUIRED <= RAN, sorted(REQUIRED - RAN)
