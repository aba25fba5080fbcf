"""Pins tests/replay_ref.py (no GPU): the launch-plan mirrors against plans worked out by hand from replay.cu, the
protocol model of the bulk-copy pipeline (which plans hung before the one-stage fix, and that none does now), the
regimes the GPU test's cases reach, and the tree references against the sequential C oracle."""
import numpy as np
import pytest

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
