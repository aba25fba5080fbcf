"""Pins tests/replay_ref.py (no GPU): the launch-plan mirrors against plans worked out by hand from replay.cu, the
protocol model of the bulk-copy pipeline (which plans hung before the one-stage fix, and that none does now), the
regimes the GPU tests' cases reach, the tree references against the sequential C oracle, and the space-to-depth mirror
and plane reference of the fused sample + gather + space-to-depth kernel."""
import numpy as np
import pytest

import learn_ref as lr
import replay_cases as rc
import replay_ref as rr

SM = 132                                   # H100 SXM multiprocessors: the hand-worked plans below assume it
A = rc.ATARI


def _plan(rows, n, ctas=4, stages=0, fused=False, off=0):
    return rr.gather_plan([(rb, off, off) for rb in rows], n, SM, ctas, stages, fused)


# ---- gather plans ----------------------------------------------------------------------------------------------------
def test_split_row_by_hand():
    assert rr.split_row(A) == (4, 7056, 7056)            # ceil(28224 / 8192) = 4 chunks of 28224 / 4
    assert rr.split_row(2048) == (1, 2048, 2048)
    assert rr.split_row(8192) == (1, 8192, 8192)
    assert rr.split_row(8208) == (2, 4112, 4096)         # ceil(8208 / 2) = 4104 -> 4112 (16-byte multiple)
    assert rr.split_row(16400) == (3, 5472, 5456)


# (ctas, n, fused) -> (grid, items of the fullest CTA, stages)
#   budget = 200 KiB / ctas - 256 (- 256 fused); stages = min(budget // 7168, items per CTA)
ATARI_PLANS = {
    (4, 512, False): (528, 4, 4),          # 2048 items on 528 CTAs; budget 50944 -> 7 stages, capped at 4 items
    (14, 512, False): (1848, 2, 2),        # budget 14628 - 256 = 14372 -> 2 stages
    (14, 512, True): (1848, 2, 1),         # 14372 - 256 = 14116 -> 1 stage: hung before the fix
    (15, 512, False): (1980, 2, 1),        # 13653 - 256 = 13397 -> 1 stage, 68 CTAs with 2 items: hung before the fix
    (16, 512, False): (2048, 1, 1),        # one item per CTA: 1 stage is enough, never hung
    (16, 4096, False): (2112, 8, 1),       # 16384 items on 2112 CTAs, 12544 -> 1 stage: hung before the fix
}


@pytest.mark.parametrize("key", sorted(ATARI_PLANS))
def test_atari_plans_by_hand(key):
    ctas, n, fused = key
    grid, per_cta, stages = ATARI_PLANS[key]
    p = _plan([A], n, ctas, 0, fused)
    assert [(b["nchunk"], b["chunk_bytes"], b["last_bytes"]) for b in p["big"]] == [(4, 7056, 7056)]
    assert p["stage_bytes"] == 7168 and p["items_per_sample"] == 4 and p["total_items"] == 4 * n
    assert (p["grid"], int(p["cta_items"].max()), p["stages"]) == (grid, per_cta, stages)
    assert p["cta_items"].sum() == 4 * n and p["cta_items"].min() == (4 * n) // grid
    hangs = stages == 1 and per_cta >= 2
    assert ("one-stage-multi" in rr.pipeline_regimes(p)) == hangs
    assert (rr.pipeline_run(stages, per_cta, fixed=False)[0] is not None) == hangs
    assert rr.pipeline_run(stages, per_cta)[0] is None


def test_2048_byte_row_by_hand():
    p = _plan([2048], 512)
    assert p["big"][0]["nchunk"] == 1 and p["stage_bytes"] == 2048
    assert (p["grid"], p["stages"], int(p["cta_items"].max())) == (512, 1, 1)     # grid capped at the 512 items
    # the fused fallback case: 4096 one-item samples on 132 CTAs = 32 samples per CTA > kMaxCtaSamples
    p = _plan([2048], 4096, ctas=1, fused=True)
    assert (p["grid"], p["stages"], int(p["cta_items"].max())) == (132, 32, 32)  # 204288 // 2048 = 99 -> 32 items
    assert rr.fused_fallback(p)
    assert not rr.fused_fallback(_plan([2048], 512, ctas=1, fused=True))          # 4 items: 5 samples at most
    # an offset base demotes the row to the LSU copy
    p = _plan([2048], 512, off=4)
    assert not p["big"] and p["small"] == [0] and rr.fused_fallback(p)


def test_unaligned_rows_by_hand():
    """8193 and 33000 bytes are not 16-byte multiples: no bulk chunks (so no 1-byte last chunk either), LSU copy with
    byte (8193, odd) or 4-byte accesses (33000 = 16 * 2062 + 8)"""
    for rb, width in ((8193, 1), (33000, 4), (2047, 1), (68, 4), (3, 1), (1040, 16)):
        p = _plan([rb], 7)
        assert not p["big"] and p["small"] == [0] and p["grid"] == 0 and rr.gather_launches(p) == 1
        assert rr.copy_path(0, 0, rb) == width
    assert rr.copy_path(4, 4, 2048) == 4 and rr.copy_path(1, 1, 2048) == 1 and rr.copy_path(256, 512, 2048) == 16


def test_mixed_columns_by_hand():
    p = _plan(rc.MIX, 512, ctas=1)
    assert [b["col"] for b in p["big"]] == [0, 1, 2, 3] and p["small"] == [4, 5, 6, 7]
    assert [b["first_item"] for b in p["big"]] == [0, 4, 8, 9] and p["items_per_sample"] == 11
    assert p["stage_bytes"] == 7168 and p["grid"] == 132 and p["stages"] == 28          # 204544 // 7168 = 28
    assert int(p["cta_items"].max()) == 43 and rr.gather_launches(p) == 2


# ---- the pipeline protocol model -------------------------------------------------------------------------------------
def test_pipeline_model_hangs_only_with_one_stage_before_the_fix():
    for S in range(1, rr.MAX_STAGES + 1):
        for cnt in range(0, 3 * S + 4):
            err_old, _ = rr.pipeline_run(S, cnt, fixed=False)
            err_new, fills = rr.pipeline_run(S, cnt)
            assert err_new is None, (S, cnt, err_new)
            assert sum(fills) == cnt and max(fills) == -(-cnt // S)
            if S == 1 and cnt >= 2:
                assert err_old == "hang: waits for item 1, whose load was never issued"
            else:
                assert err_old is None, (S, cnt, err_old)


def test_knob_grid_reaches_every_pipeline_regime():
    """by the mirror, the GPU test's knob grid puts a CTA in the one-stage pipeline with two or more items (the case
    that hung before the fix: gather_stages = 1, or 14-16 CTAs per SM on Atari rows), refills one stage three or more
    times, and keeps the fused kernel fused (the fallback has a case of its own)"""
    seen, hang = set(), []
    for ctas, stages in rc.KNOB_GRID:
        for n in rc.MIX_N:
            for fused in (False, True):
                p = _plan(rc.MIX, n, ctas, stages, fused)
                seen |= rr.pipeline_regimes(p)
                if "one-stage-multi" in rr.pipeline_regimes(p):
                    hang.append((ctas, stages, n, fused))
        p = _plan(rc.WIDE, rc.WIDE_N, ctas, stages)
        seen |= rr.pipeline_regimes(p)
    assert {"one-stage-multi", "reuse>=3", "all-in-flight", "refill"} <= seen
    assert (1, 1, 512, False) in hang and (16, 0, 512, False) in hang and (14, 0, 512, True) in hang
    assert not any(rr.fused_fallback(_plan(rc.MIX, n, c, s, True)) for c, s in rc.KNOB_GRID for n in rc.MIX_N)


# ---- tree paths and references ---------------------------------------------------------------------------------------
def test_update_paths_by_hand():
    assert rr.update_path(0, 1 << 14) == "none"
    assert rr.update_path(512, 1 << 20) == "sorted" and rr.update_path(512, 1 << 21) == "cta"   # 21 > 9 + 11 levels
    assert rr.update_path(1, 1) == "sorted" and rr.update_path(512, 1 << 14, sorted_knob=0) == "cta"
    assert rr.update_path(513, 2) == "cta" and rr.update_path(1024, 1 << 7) == "cta"
    assert rr.update_path(1025, 1 << 14) == "levels"
    assert rr.update_launches(1025, 1 << 14) == 3 + 14 + 1 and rr.update_launches(1025, 1, max_out=False) == 3
    assert rr.descent_rounds(1 << 21) == [7, 7, 7] and rr.descent_rounds(1 << 14) == [7, 7]
    assert rr.descent_rounds(1 << 7) == [7] and rr.descent_rounds(2) == [1] and rr.descent_rounds(1) == []
    paths = {rr.update_path(n, s, k) for s in rc.TREE_SIZES for n in rc.UPDATE_N for k in (0, 1)}
    assert paths == {"none", "sorted", "cta", "levels"}


@pytest.mark.parametrize("size", [1, 2, 1 << 7, 1 << 12])
def test_tree_from_leaves_equals_sequential_oracle(size):
    rng = np.random.RandomState(size)
    leaves, _ = rc.tree_leaves(rng, size)
    trees = rr.oracle_init(size)
    order = rng.permutation(size)
    rr.oracle_update(trees, order, leaves[order], leaves[order] * 3)
    for op, t in enumerate(trees):
        np.testing.assert_array_equal(rr.tree_from_leaves(leaves * (3 if op == rr.MAX else 1), op), t)


def test_oracle_update_skips_and_last_writer_wins():
    trees = rr.oracle_init(8)
    flags = rr.oracle_update(trees, [3, 3, 8, -1, 5], [1.0, 2.0, 4.0, 4.0, -1.0], [5.0, 6.0, 7.0, 7.0, -1.0])
    assert flags == 2
    assert trees[0][7 + 3] == 2.0 and trees[2][7 + 3] == 6.0 and trees[0][0] == 2.0 and trees[1][0] == 2.0
    assert trees[0][7 + 5] == 0.0 and np.isinf(trees[1][7 + 5])


@pytest.mark.parametrize("size", rc.TREE_SIZES + (1024,))
def test_oracle_draws_zero_priority_tail_only_at_the_total(size):
    """the trees of the GPU sample tests (zero priorities after the first 3/4 of the leaves), u = 0 and
    nextafter(1, 0) included: a zero-priority leaf is drawn only by the last sample (u = nextafter(1, 0)), when its
    value rounds to the tree total or above it and the descent's subtractions then exceed the non-zero sum of a right
    child.  It is then the last leaf, as in the reference.  Some of these cases do draw it."""
    leaves, m = rc.tree_leaves(np.random.RandomState(size + 1), size)
    s, mn = rr.tree_from_leaves(leaves, rr.SUM), rr.tree_from_leaves(np.where(leaves > 0, leaves, np.inf), rr.MIN)
    tail_draws = 0
    for n in rc.SAMPLE_N + rc.MIX_N + (64, 4096):
        u = np.random.RandomState(size + n).rand(n)
        u[0], u[-1] = 0.0, np.nextafter(1.0, 0.0)
        idx, w = rr.oracle_sample(s, mn, u, 2 * m, 0.4)
        tail = idx >= m
        assert idx.min() >= 0 and (w > 0).all()
        assert not tail[:-1].any() and (idx[tail] == size - 1).all()
        assert (rr.sample_values(s[0], u)[tail] >= s[0] * (1 - 2.0 ** -50)).all()
        assert (w[~tail] <= 1.0).all()
        tail_draws += tail.sum()
    assert (tail_draws > 0) == (size in (1024, 1 << 21))


def test_oracle_store_wraps_at_the_cursor():
    trees = rr.oracle_init(8)
    pa = rr.oracle_store(trees, 6, 8, 1.5, 0.6)
    assert pa == 1.5 ** 0.6
    assert (trees[0][7:] == pa).all() and (trees[1][7:] == pa).all() and (trees[2][7:] == 1.5).all()
    want = rr.oracle_init(8)
    rr.oracle_update(want, (6 + np.arange(8)) % 8, np.full(8, pa), np.full(8, 1.5))
    for a, b in zip(trees, want):
        np.testing.assert_array_equal(a, b)


def test_host_priorities_reference():
    pa, pr = rr.host_priorities([0.0, 1.5, -0.5, np.nan], 1e-6, 0.6)
    assert pr[0] == 1e-6 and pa[1] == (1.5 + 1e-6) ** 0.6 and np.isnan(pa[2:]).all() and np.isnan(pr[2:]).all()


# ---- the fused sample + gather + space-to-depth kernel -------------------------------------------------------------------
# (n, n_img, sm) -> (parts, per_band, rows_per_chunk, chunk_stride, smem, bands) for Atari frames (84x84x4, s = 4: 21 s2d
# rows of 1344 bytes, 2816 // 1344 = 2 rows per chunk); parts = min(4 sm // (n / 8 * n_img), 21); a stride of an even
# number of 16-byte units gets 16 bytes of padding; smem = 256 + 2 stages * 8 samples * stride
ATARI_S2D = {
    (8, 1, 132): (21, 1, 1, 1360, 22016, [(1, False)] * 21),          # 1344 = 84 x 16 -> 1360; the 16640-byte scratch
    (128, 2, 132): (16, 2, 2, 2704, 43520, [(1, False)] * 10 + [(1, True)] + [(0, False)] * 5),  # 528 // 32 = 16
    (512, 1, 132): (8, 3, 2, 2704, 43520, [(2, True)] * 7 + [(0, False)]),                       # 528 // 64 = 8
    (512, 2, 132): (4, 6, 2, 2704, 43520, [(3, False)] * 3 + [(2, True)]),                       # a stage refill
    (4096, 1, 132): (1, 21, 2, 2704, 43520, [(11, True)]),
    (128, 2, 114): (14, 2, 2, 2704, 43520, [(1, False)] * 10 + [(1, True)] + [(0, False)] * 3),  # 456 // 32 = 14
    (512, 2, 114): (3, 7, 2, 2704, 43520, [(4, True)] * 3),                                      # 456 // 128 = 3
}


@pytest.mark.parametrize("key", sorted(ATARI_S2D))
def test_s2d_atari_plans_by_hand(key):
    n, n_img, sm = key
    p = rr.s2d_plan(n, n_img, 84, 84, 4, 4, sm)
    parts, per_band, rows, stride, smem, bands = ATARI_S2D[key]
    assert (p["parts"], p["per_band"], p["rows_per_chunk"], p["chunk_stride"], p["smem"]) == (
        parts, per_band, rows, stride, smem)
    assert p["bands"] == bands and p["grid"] == n // 8 * n_img * parts and p["refusal"] is None
    assert (p["slots"], p["dyl"], p["dX"], p["frame_tma"]) == (8, 0, 8, False)        # 32 threads per pixel, 21 columns
    assert sum(k * rows - part for k, part in bands) == 21                              # every s2d row exactly once
    reg = p["regimes"]
    assert ("empty-band" in reg) == any(k == 0 for k, _ in bands)
    assert ("partial" in reg) == any(part for _, part in bands)
    assert ("refill" in reg) == (max(k for k, _ in bands) > rr.S2D_STAGES)


def test_s2d_frame_store_plans_by_hand():
    # 84x84 at B = 128, two columns: 2688 = 21 x 128 bytes per sample, a 672-byte (168-word) band: TMA boxes, no padding
    p = rr.s2d_plan(128, 2, 84, 84, 4, 4, SM, True, 64, 1)
    assert p["frame_tma"] and p["chunk_stride"] == 2688 and p["smem"] == 256 + 16 * 2688
    assert list(rr.s2d_chunk_full(p)) == [True] * 10 + [False]
    assert not rr.s2d_plan(128, 2, 84, 84, 4, 4, SM, True, 64, 0)["frame_tma"]           # knob off
    assert not rr.s2d_plan(128, 2, 84, 84, 4, 4, SM, True, 3, 1)["frame_tma"]            # fewer than four slots
    assert rr.s2d_plan(32, 1, 16, 16, 4, 4, SM, True, 4, 1)["frame_tma"]                 # exactly four slots
    # one s2d row per chunk: 1344 bytes per sample is not a multiple of 128 -> bulk copies, 16 bytes of padding
    p = rr.s2d_plan(8, 1, 84, 84, 4, 4, SM, True, 64, 1)
    assert not p["frame_tma"] and p["chunk_stride"] == 1360 and "tma-ineligible" in p["regimes"]
    # 8x272 frames: 4352 = 34 x 128 bytes per sample, but a 1088-byte band is 272 words, wider than a TMA box
    p = rr.s2d_plan(8, 1, 8, 272, 4, 4, SM, True, 64, 1)
    assert not p["frame_tma"] and p["chunk_stride"] == 4368 and p["rows_per_chunk"] == 1


def test_s2d_conversion_and_refusals_by_hand():
    p = rr.s2d_plan(1024, 1, 48, 12, 8, 3, SM)          # 24 threads per pixel: 10 slots, 16 idle threads, 4 columns
    assert (p["slots"], p["dyl"], p["dX"], p["rows_per_chunk"]) == (10, 2, 2, 4)
    assert {"idle-threads", "slots>Ws", "multi-pass-dyl", "run=8k"} <= p["regimes"]
    p = rr.s2d_plan(8, 1, 64, 32, 1, 32, SM)            # 256 threads per pixel: one slot, w / s == 1
    assert (p["slots"], p["dyl"], p["dX"]) == (1, 1, 0) and p["refusal"] is None and "Ws=1" in p["regimes"]
    p = rr.s2d_plan(*rc.S2D_S64, SM)                    # 512 threads per pixel: no slot, the planes would stay unwritten
    assert p["slots"] == 0 and p["refusal"] == "s>32"
    p = rr.s2d_plan(16, 1, 8, 256, 4, 4, SM)            # 4096-byte s2d rows: one per chunk, 4112-byte stride
    assert (p["rows_per_chunk"], p["chunk_stride"], p["smem"]) == (1, 4112, 66048)
    assert rr.s2d_plan(8, 1, 4, 896, 4, 4, SM)["smem"] == 256 + 16 * 14352 <= rr.SMEM_OPTIN
    p = rr.s2d_plan(*rc.S2D_OVER_SMEM, SM)
    assert p["smem"] == 256 + 16 * 16400 > rr.SMEM_OPTIN and p["refusal"] == "smem"


def test_s2d_one_box_by_hand():
    rows = [(0, 1, 2, 3), (5, 5, 5, 5), (5, 5, 6, 7), (62, 63, 0, 1), (60, 61, 62, 63), (7, 8, 9, 9)]
    full = [True, True, False]
    got = rr.s2d_one_box(rows, full)
    want = np.array([[1, 1, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0], [1, 1, 0], [0, 0, 0]], bool)
    np.testing.assert_array_equal(got, want)
    assert rr.s2d_box_regimes(got, full) == {"one-box", "four-copies", "partial-fallback"}
    assert rr.s2d_box_regimes(rr.s2d_one_box(rows[:1], [True]), [True]) == {"one-box"}
    assert rr.s2d_box_regimes(rr.s2d_one_box(rows[1:4], full), full) == {"four-copies"}


def test_frame_tables_hold_every_stack_kind():
    for slots in (64, 4):
        fidx = rc.frame_table(np.random.RandomState(0), rc.S2D_FRAME_CAPACITY, slots)
        assert fidx.shape == (rc.S2D_FRAME_CAPACITY, 4) and fidx.min() >= 0 and fidx.max() < slots
        f = rc.frame_idx(np.random.RandomState(1), 8, fidx)
        s = fidx[f[:4]].astype(np.int64)
        assert (np.diff(s[0]) == 1).all() and (np.diff(s[1]) == 0).all()
        assert list(np.diff(s[2])) == [0, 1, 1] and (np.diff(s[3]) < 0).any()


def _s2d_table_regimes(sm):
    """the regimes the GPU test's case table reaches on `sm` multiprocessors, named as the test names them"""
    ran = set()
    for n, n_img, h, w, c, s, small in rc.S2D_RING:
        p = rr.s2d_plan(n, n_img, h, w, c, s, sm)
        assert p["refusal"] is None
        ran |= {("ring", r) for r in p["regimes"]}
        spec = rc.SMALL_MIX if small == "mix" else ()
        ran |= {("copy", rr.copy_path(off, off, rb)) for rb, off in spec} | {("small", len(spec))}
    for n, n_img, h, w, slots, _ in rc.S2D_FRAMES:
        rng = np.random.RandomState(n + h + slots)
        fidx = rc.frame_table(rng, rc.S2D_FRAME_CAPACITY, slots)
        rows = fidx[rc.frame_idx(rng, n, fidx)]
        for knob in (0, 1):
            p = rr.s2d_plan(n, n_img, h, w, 4, 4, sm, True, slots, knob)
            ran |= {("frames", r) for r in p["regimes"]}
            if p["frame_tma"]:
                full = rr.s2d_chunk_full(p)
                ran |= {("box", r) for r in rr.s2d_box_regimes(rr.s2d_one_box(rows, full), full)}
    for size, n, n_img, h, w, c, s, frames, outs in rc.S2D_PER:
        p = rr.s2d_plan(n, n_img, h, w, c, s, sm, frames, 64 if frames else 0)
        ran |= {("frames" if frames else "ring", r) for r in p["regimes"]}
        ran |= {("per", o) for o in outs or ("no-weights",)} | {("per", "size=%d" % size)}
        ran |= {("per", "frames")} if frames else set()
    return ran


@pytest.mark.parametrize("sm", [132, 114])
def test_s2d_case_table_reaches_every_regime(sm):
    """on an H100 SXM (132 SMs) and PCIe (114 SMs) the case table reaches every regime the GPU test requires; the
    regimes the frame-store cases reach with the TMA boxes on come from the sampled stacks"""
    missing = rc.S2D_REQUIRED - _s2d_table_regimes(sm)
    assert not missing, sorted(missing)


@pytest.mark.parametrize("B,h,w,c,s", [(8, 6, 10, 8, 1), (8, 4, 6, 16, 1), (8, 9, 12, 8, 3), (8, 10, 20, 8, 5),
                                       (16, 12, 12, 4, 6), (8, 16, 16, 1, 8), (8, 64, 32, 1, 32), (8, 8, 8, 2, 4)])
def test_u8_s2d_plane_against_a_plain_loop(B, h, w, c, s):
    """learn_ref.u8_s2d_plane against the definition, element by element: pixel (y, x, ch) of sample b goes to plane
    row (y / s * (w / s) + x / s) * B + b, column ((y % s) s + x % s) c + ch, of the 8x8 core-tiled layout, as the bf16
    bits of its value (the upper half of the fp32)"""
    x = np.random.RandomState(B + h + s).randint(0, 256, (B, h, w, c)).astype(np.uint8)
    ws, cs = w // s, s * s * c
    want = np.zeros(h * w * c * B, np.uint16)
    for b in range(B):
        for y in range(h):
            for xx in range(w):
                for ch in range(c):
                    r = (y // s * ws + xx // s) * B + b
                    col = ((y % s) * s + xx % s) * c + ch
                    e = ((r // 8) * (cs // 8) + col // 8) * 64 + (r % 8) * 8 + col % 8
                    want[e] = np.float32(x[b, y, xx, ch]).view(np.uint32) >> 16
    np.testing.assert_array_equal(lr.u8_s2d_plane(x, s), want)
