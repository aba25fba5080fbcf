"""Host references of the replay kernels of include/coach_b200.h (coach_b200/csrc/replay.cu, and cb200_gather_at in
heads.cu): the launch-plan mirrors that tell which regime a call runs in (the row gathers and the fused sample +
gather + space-to-depth kernel), the exact references of the row copies, and the segment-tree references, which run
oracle/segment_tree.c through oracle.memory.  The space-to-depth planes themselves are tests/learn_ref.u8_s2d_plane of
the gathered frames.  numpy only, importable without CUDA.

Bounds: tree nodes, leaf indices, raw priorities and every copied byte are bit for bit; importance weights within 4 ulp
of the oracle (both ends call pow); p_alpha from the device's pow within 2 ulp of Python's `**`, from the host's libm
bit for bit.  tests/test_replay_ref_host.py pins this module to hand-worked plans and to the oracle.
"""
import ctypes

import numpy as np

from oracle import memory as om

# replay.cu:486-490, :247-249
STAGE_BYTES = 8192            # kStageBytes: largest chunk of a row
MAX_STAGES = 32               # kMaxStages
BAR_BYTES = MAX_STAGES * 8    # kBarBytes: the mbarriers ahead of the stages in dynamic shared memory
MAX_CTA_SAMPLES = 16          # kMaxCtaSamples: descents one CTA of the fused kernel can hold
UPD_SORT_THREADS = 512        # kUpdSortThreads
UPD_AHEAD, UPD_TOP_LEVELS = 11, 10
ROUND_LEVELS = 7              # kRoundLevels: tree levels per round of the descent (replay.cu:50)
DEFAULT_CTAS_PER_SM = 4       # replay.cu:942 g_tune_ctas_per_sm


def _cdiv(a, b):
    return -(-a // b)


# ---- launch-plan mirrors -------------------------------------------------------------------------------------------------
def copy_path(dst_addr, src_addr, nbytes):
    """replay.cu:519-529 warp_copy_row (and the same test in heads.cu:142-148 gather_at_kernel, which has no 16-byte
    path): the access width, 16, 4 or 1 bytes, from the OR of both addresses and the byte count"""
    a = dst_addr | src_addr | nbytes
    return 16 if a % 16 == 0 else (4 if a % 4 == 0 else 1)


def split_row(row_bytes):
    """replay.cu:966-975: chunks of a bulk-copied row: (nchunk, chunk_bytes, last_bytes)"""
    nchunk = _cdiv(row_bytes, STAGE_BYTES)
    cb = (_cdiv(row_bytes, nchunk) + 15) // 16 * 16
    while cb > STAGE_BYTES:
        nchunk += 1
        cb = (_cdiv(row_bytes, nchunk) + 15) // 16 * 16
    nchunk = _cdiv(row_bytes, cb)
    return nchunk, cb, row_bytes - cb * (nchunk - 1)


def gather_plan(columns, n, sm_count, ctas_per_sm=DEFAULT_CTAS_PER_SM, forced_stages=0, fused=False):
    """replay.cu:950-1008 build_gather_params + plan_bulk, and :590-593 cta_item_range.

    columns: (row_bytes, src_addr, dst_addr) per column, addresses of row 0 (only their residue mod 16 matters).
    A column goes through the bulk (TMA) pipeline when its rows are 16-byte multiples of at least 2 KiB and both bases
    are 16-byte aligned; every other column is 'small' (one warp per row).  `ctas_per_sm` / `forced_stages` are the
    gather_ctas_per_sm / gather_stages knobs, clamped as tune_get clamps them.  Returns a dict; `cta_items` holds the
    item count of every CTA of the bulk grid."""
    ctas_per_sm = min(max(ctas_per_sm, 1), 16)
    forced_stages = min(max(forced_stages, 0), MAX_STAGES)
    big, small, ips = [], [], 0
    for c, (rb, sa, da) in enumerate(columns):
        if rb % 16 == 0 and sa % 16 == 0 and da % 16 == 0 and rb >= 2048:
            nchunk, cb, last = split_row(rb)
            big.append(dict(col=c, row_bytes=rb, nchunk=nchunk, chunk_bytes=cb, last_bytes=last, first_item=ips))
            ips += nchunk
        else:
            small.append(c)
    total = ips * n
    stage_bytes = (max([16] + [b["chunk_bytes"] for b in big]) + 127) // 128 * 128
    plan = dict(big=big, small=small, items_per_sample=ips, total_items=total, stage_bytes=stage_bytes, grid=0,
                stages=0, cta_items=np.zeros(0, np.int64), fused=fused)
    if not big:
        return plan
    g = max(min(sm_count * ctas_per_sm, total), 1)
    items_per_cta = _cdiv(total, g)
    budget = 200 * 1024 // ctas_per_sm - BAR_BYTES - (MAX_CTA_SAMPLES * 16 if fused else 0)
    st = min(budget // stage_bytes, items_per_cta)
    if 0 < forced_stages < st:
        st = forced_stages
    st = max(min(st, MAX_STAGES), 1)
    b = np.arange(g, dtype=np.int64)
    plan.update(grid=g, stages=st, cta_items=total * (b + 1) // g - total * b // g)
    return plan


def fused_fallback(plan):
    """replay.cu:1204-1212: cb200_per_sample_gather samples first and gathers second (two or three launches) when there
    is no bulk column or when a CTA's item range could span more than kMaxCtaSamples samples"""
    if not plan["big"]:
        return True
    g, ips = plan["grid"], plan["items_per_sample"]
    return (_cdiv(plan["total_items"], g) + ips - 1) // ips + 1 > MAX_CTA_SAMPLES


def fused_owners(plan, n):
    """replay.cu:648-670: the CTA that publishes sample s and copies its small columns is the one holding the sample's
    first item.  Returns the owning CTA of every sample (each sample must have exactly one)"""
    total, g, ips = plan["total_items"], plan["grid"], plan["items_per_sample"]
    b = np.arange(g, dtype=np.int64)
    lo, hi = total * b // g, total * (b + 1) // g
    owners = np.full(n, -1, np.int64)
    count = np.zeros(n, np.int64)
    for cta in range(g):
        if hi[cta] <= lo[cta]:
            continue
        for s in range(lo[cta] // ips, (hi[cta] - 1) // ips + 1):
            if s * ips >= lo[cta]:
                owners[s] = cta
                count[s] += 1
    return owners, count


def gather_launches(plan):
    """replay.cu:1170-1190: one bulk launch when there is a bulk column, one LSU launch when there is a small one"""
    return int(bool(plan["big"])) + int(bool(plan["small"]))


def pipeline_run(S, cnt, fixed=True):
    """A protocol model of bulk_pipeline (replay.cu:534-588) for one CTA: S stages, cnt items.  Item k is loaded into
    stage k % S (mbarrier phase k // S) and stored back from it.  The model replays the thread's program order and
    checks, at every step, what the hardware needs:
      * mbar_wait for item k finds the load of item k issued (otherwise the wait spins for ever);
      * a load into a stage is issued only after the wait for the stage's previous item (the barrier's previous phase)
        and after that item's store has finished reading shared memory (bulk_wait_read<N>: every committed store but
        the newest N).
    `fixed` selects the refill rule: True = the current code (lag 1 with two or more stages, lag 0 with one), False =
    the rule before the fix (always lag 1).  Returns (ok, stage_fills): ok False names the first violation."""
    issued, waited, committed, read_done = set(), set(), [], set()
    fills = [0] * S

    def issue(j):
        prev = j - S
        if prev >= 0 and (prev not in waited or prev not in read_done):
            return "load of item %d into stage %d before item %d left it" % (j, j % S, prev)
        issued.add(j)
        fills[j % S] += 1
        return None

    def wait_read(keep):
        for item in committed[:len(committed) - keep]:
            read_done.add(item)

    for k in range(min(cnt, S)):
        issue(k)
    for k in range(cnt):
        if k not in issued:
            return "hang: waits for item %d, whose load was never issued" % k, fills
        waited.add(k)
        committed.append(k)
        if fixed and S == 1:
            if k + 1 < cnt:
                wait_read(0)
                err = issue(k + 1)
                if err:
                    return err, fills
        elif k >= 1 and k - 1 + S < cnt:
            wait_read(1)
            err = issue(k - 1 + S)
            if err:
                return err, fills
    return None, fills


def pipeline_regimes(plan):
    """the pipeline regimes a bulk plan puts its CTAs in: 'one-stage-multi' (S = 1 and a CTA with two or more items:
    the case that hung before the fix), 'reuse>=3' (a stage filled three or more times), 'all-in-flight' (a CTA whose
    items all fit in the stages at once) and 'refill' (a CTA that refills a stage)"""
    S, out = plan["stages"], set()
    if not plan["big"]:
        return out
    cmax, cmin = int(plan["cta_items"].max()), int(plan["cta_items"][plan["cta_items"] > 0].min())
    if S == 1 and cmax >= 2:
        out.add("one-stage-multi")
    if cmax >= 2 * S + 1:
        out.add("reuse>=3")
    if cmin <= S:
        out.add("all-in-flight")
    if cmax > S:
        out.add("refill")
    return out


def update_path(n, size, sorted_knob=1):
    """replay.cu:1059-1086 run_update: 'none' (n = 0), 'sorted' (n <= 512, at most 20 levels, knob per_update_sorted on:
    one launch), 'cta' (n <= 1024: one launch) or 'levels' (claim, leaf, reset, one launch per level and the max)"""
    levels = int(size).bit_length() - 1
    if n <= 0:
        return "none"
    if n <= UPD_SORT_THREADS and levels <= UPD_TOP_LEVELS - 1 + UPD_AHEAD and sorted_knob:
        return "sorted"
    if n <= 1024:
        return "cta"
    return "levels"


def update_launches(n, size, sorted_knob=1, max_out=True):
    path = update_path(n, size, sorted_knob)
    levels = int(size).bit_length() - 1
    return {"none": 0, "sorted": 1, "cta": 1, "levels": 3 + levels + int(bool(max_out))}[path]


def descent_rounds(size):
    """replay.cu:54-96 warp_descent: levels fetched per round (7, then the rest)"""
    levels, out = int(size).bit_length() - 1, []
    while levels > 0:
        out.append(min(levels, ROUND_LEVELS))
        levels -= out[-1]
    return out


# replay.cu:689-690, :1284-1313: the fused sample + gather + space-to-depth kernel
S2D_THREADS = 256             # kS2dThreads
S2D_STAGES = 2                # kS2dStages
S2D_CHUNK_BUDGET = 2816       # bytes of s2d rows per sample and chunk
S2D_SCRATCH = 256 + 8 * 256 * 8     # phase A: the per-warp descent scratch (kScratchDoubles doubles per warp)
SMEM_DEFAULT = 48 * 1024      # dynamic shared memory a launch gets without the opt-in attribute
SMEM_OPTIN = 227 * 1024       # the opt-in limit of one H100 CTA
TMA_BOX_WORDS = 256           # largest TMA box dimension


def s2d_plan(n, n_img, h, w, c, s, sm_count, frames=False, frame_slots=0, frame_tma_knob=0):
    """replay.cu:1282-1311 launch_gather_s2d (and :1229-1260 frame_store_map), :729-736 / :755 / :805-828 of the kernel.

    CTA = (8-sample group, image column, band of s2d rows): `parts` bands of `per_band` rows, as many CTAs as one wave
    of four per SM holds; each band is streamed in chunks of `rows_per_chunk` s2d rows (about 2816 bytes per sample)
    through two shared-memory stages of 8 * `chunk_stride` bytes.  The frame store fetches a stack of four
    consecutive frame slots with one 2-D TMA box when the knob is on, the per-sample stride is a multiple of 128 bytes
    and the box is at most 256 words wide.  Conversion: 8 S threads per s2d pixel, `slots` pixels per pass, pixel
    index advanced by (dyl rows, dX columns) -- 'multi-pass' when a chunk has more pixels than slots ('-dyl' when a
    step crosses whole rows).  `bands` holds (chunks, last chunk partial) per band; `regimes` names
    what the call exercises; `refusal` names why the library refuses the geometry (None: it launches)."""
    hs, ws = h // s, w // s
    row = s * w * c                                   # s2d_row_bytes: one s2d row of one sample
    groups = n // 8 * n_img
    parts = min(max(4 * sm_count // groups, 1), hs)
    per_band = _cdiv(hs, parts)
    rc = min(max(S2D_CHUNK_BUDGET // row, 1), per_band)
    stride = rc * row
    band_bytes = rc * s * w                           # frame store: bytes of one frame's band of a chunk
    tma_eligible = bool(frames) and frame_slots >= 4 and stride % 128 == 0
    frame_tma = tma_eligible and bool(frame_tma_knob) and band_bytes // 4 <= TMA_BOX_WORDS
    if not frame_tma and (stride // 16) % 2 == 0:
        stride += 16
    smem = max(256 + S2D_STAGES * 8 * stride, S2D_SCRATCH)
    slots = S2D_THREADS // (8 * s)
    dyl, dX = divmod(slots, ws) if slots else (0, 0)
    bands = []
    for p in range(parts):
        rows = max(min(hs, (p + 1) * per_band) - p * per_band, 0)
        bands.append((_cdiv(rows, rc), rows % rc != 0))
    refusal = "s>32" if slots == 0 else ("smem" if smem > SMEM_OPTIN else None)
    reg = set()
    chunks = [k for k, _ in bands if k]
    if max(chunks) == 1:
        reg.add("one-chunk")
    if max(chunks) > S2D_STAGES:
        reg.add("refill")
    if any(part for _, part in bands):
        reg.add("partial")
    if min(k for k, _ in bands) == 0:
        reg.add("empty-band")
    if parts == 1:
        reg.add("one-band")
    if parts == hs and hs > 1:
        reg.add("bands=Hs")
    if row > S2D_CHUNK_BUDGET:
        reg.add("rc=1")
    if smem > SMEM_DEFAULT:
        reg.add("smem>48K")
    if frames:
        reg.add("tma" if frame_tma else ("tma-ineligible" if frame_tma_knob else "bulk"))
    else:
        run = s * c
        reg.add("run=16" if run == 16 else ("run=8" if run == 8 else "run=8k"))
        reg.add("S=%d" % s)
        if S2D_THREADS % (8 * s):
            reg.add("idle-threads")
        if slots > ws:
            reg.add("slots>Ws")
        if ws == 1:
            reg.add("Ws=1")
        if rc * ws > slots > 0:
            reg.add("multi-pass" if dyl == 0 else "multi-pass-dyl")
    return dict(parts=parts, per_band=per_band, rows_per_chunk=rc, chunk_stride=stride, smem=smem,
                frame_tma=frame_tma, slots=slots, dyl=dyl, dX=dX, bands=bands, grid=groups * parts, regimes=reg,
                refusal=refusal)


def s2d_chunk_full(plan):
    """per chunk of every band, in (band, chunk) order: whether it holds rows_per_chunk rows (False: the partial last
    chunk of a band)"""
    out = []
    for k, partial in plan["bands"]:
        out += [True] * (k - 1) + [not partial] if k else []
    return np.array(out, bool)


def s2d_one_box(fidx_rows, rc_full):
    """replay.cu:773-774: with frame_tma on, sample i fetches chunk j with one 2-D TMA box when its stack sits in four
    consecutive frame slots and the chunk is full; otherwise with four per-frame bulk copies.  fidx_rows: the [n, 4]
    frame slots of the sampled stacks; rc_full: s2d_chunk_full.  Returns bool [n, chunks]."""
    f = np.asarray(fidx_rows, np.int64)
    consecutive = (f[:, 1] == f[:, 0] + 1) & (f[:, 2] == f[:, 0] + 2) & (f[:, 3] == f[:, 0] + 3)
    return consecutive[:, None] & np.asarray(rc_full, bool)[None, :]


def s2d_box_regimes(one_box, rc_full):
    """the copy paths a frame-store call takes: 'one-box', 'four-copies' (a stack not in consecutive slots) and
    'partial-fallback' (a consecutive stack copied frame by frame because the chunk is partial)"""
    out = set()
    if one_box.any():
        out.add("one-box")
    consecutive = one_box.any(axis=1)
    if (~consecutive).any():
        out.add("four-copies")
    if consecutive.any() and (~np.asarray(rc_full, bool)).any():
        out.add("partial-fallback")
    return out


# ---- exact references ---------------------------------------------------------------------------------------------------
def gather_stack(frames, fidx, idx):
    """cb200_gather_stack: out[i, pix, c] = frames[fidx[idx[i], c], pix]"""
    return np.stack([frames[fidx[idx, c]] for c in range(fidx.shape[1])], axis=-1)


def scatter_ring(ring, staged, cursor, n):
    """cb200_scatter_ring: ring[(cursor + i) % capacity] = staged[i] for i < n"""
    out = ring.copy()
    out[(cursor + np.arange(n)) % ring.shape[0]] = staged[:n]
    return out


def host_priorities(err, epsilon, alpha):
    """PER._update_priority :197-198 with Python floats: (p ** alpha, p), p = error + epsilon; NaN for an invalid
    (negative or NaN) error"""
    p = [float(e) + epsilon if e >= 0 else np.nan for e in err]
    return np.array([x ** alpha for x in p], np.float64), np.array(p, np.float64)


def ulp_diff(a, b):
    """distance in units of the last place between fp64 arrays of one sign"""
    return np.abs(np.asarray(a, np.float64).view(np.int64) - np.asarray(b, np.float64).view(np.int64))


# ---- segment trees (oracle/segment_tree.c) ------------------------------------------------------------------------------
SUM, MIN, MAX = 0, 1, 2


def _dp(a):
    return a.ctypes.data_as(ctypes.POINTER(ctypes.c_double))


def oracle_init(size):
    """SegmentTree.__init__: (sum, min, max) trees of 2 size - 1 nodes"""
    trees = [np.empty(2 * size - 1, np.float64) for _ in range(3)]
    for op, t in enumerate(trees):
        om.clib().ost_init(_dp(t), size, op)
    return trees


def tree_from_leaves(leaves, op):
    """a tree whose every parent is op(left, right) of its children, built bottom-up.  This is the state the
    reference's sequential updates leave behind (each update recomputes its ancestors from their children); pinned
    against oracle_update in the host test.  Used to start the device tests from large random trees."""
    size = leaves.size
    levels = [np.asarray(leaves, np.float64)]
    while levels[-1].size > 1:
        a, b = levels[-1][0::2], levels[-1][1::2]
        levels.append(a + b if op == SUM else (np.where(b < a, b, a) if op == MIN else np.where(b > a, b, a)))
    return np.concatenate(levels[::-1])


def oracle_update(trees, idx, p_alpha, p_raw):
    """cb200_per_update on host trees, one entry after the other as the reference applies them (last writer wins).
    Entries with a leaf outside [0, size) or a negative p_alpha are skipped.  Returns the error flags the device sets
    (bit 1: an index out of range)."""
    size = (trees[0].size + 1) // 2
    lib, flags = om.clib(), 0
    for i, p_a, p_r in zip(np.asarray(idx, np.int64), p_alpha, p_raw):
        if not 0 <= i < size:
            flags |= 2
            continue
        if p_a < 0:
            continue
        lib.ost_update(_dp(trees[0]), size, SUM, int(i), float(p_a))
        lib.ost_update(_dp(trees[1]), size, MIN, int(i), float(p_a))
        lib.ost_update(_dp(trees[2]), size, MAX, int(i), float(p_r))
    return flags


def oracle_store(trees, cursor, n, p_raw, alpha):
    """PER.store (oper_store) for n transitions from the ring cursor, wrapping at size: the leaves get p_raw ** alpha
    (sum, min) and p_raw (max).  Returns p_raw ** alpha as Python evaluates it, the p_alpha cb200_per_store takes."""
    size = (trees[0].size + 1) // 2
    om.clib().oper_store(_dp(trees[0]), _dp(trees[1]), _dp(trees[2]), size, cursor, n, p_raw, alpha)
    return p_raw ** alpha


def sample_values(total, u):
    """PER.sample :232-244: the value the descent of sample i looks for, a + (b - a) u with a = segment i,
    b = segment (i + 1), segment = total / n.  Rounding can put the last sample's value above the total, and the
    reference then walks to the last leaf even when its priority is zero."""
    n = len(u)
    segment = np.float64(total) / np.float64(n)
    i = np.arange(n, dtype=np.float64)
    a, b = segment * i, segment * (i + 1)
    return a + (b - a) * np.asarray(u, np.float64)


def oracle_sample(sum_tree, min_tree, u, nt, beta):
    """PER.sample :229-253 (oper_sample): leaf indices and normalised importance weights"""
    size = (sum_tree.size + 1) // 2
    u = np.ascontiguousarray(u, np.float64)
    n = u.size
    idx, w = np.empty(n, np.int64), np.empty(n, np.float64)
    om.clib().oper_sample(_dp(sum_tree), _dp(min_tree), size, n, _dp(u), nt, beta,
                          idx.ctypes.data_as(ctypes.POINTER(ctypes.c_int64)), _dp(w), None)
    return idx, w
