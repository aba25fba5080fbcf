"""Case table of tests/test_replay_kernels_gpu.py: the row sizes, batch sizes, tune-knob grid and tree shapes at which
the replay kernels are checked against tests/replay_ref.py, and the data generators (numpy only)."""
import numpy as np

ATARI = 84 * 84 * 4                 # 28224 bytes: four 7056-byte chunks; a 7168-byte stage

# row sizes of cb200_gather: LSU rows of 3 (bytes), 68 (words), 1040 (16-byte vectors) and 2047 bytes; bulk rows of
# one chunk (2048, 2064, 8192), of a short last chunk (8208 = 4112 + 4096) and of four chunks (Atari); 8193 and 33000
# are not 16-byte multiples and go through the LSU copy
ROW_BYTES = (3, 17 * 4, 1040, 2047, 2048, 2064, 8192, 8193, 8208, ATARI, 33000)
GATHER_N = (1, 7, 512, 4096)
OFFSETS = (0, 4, 1)                 # bytes added to the src and dst bases: 16-byte, 4-byte and byte alignment
CAPACITY = 1000                     # ring rows of the gather tests

# gather_ctas_per_sm x gather_stages (0 = automatic)
KNOB_GRID = [(c, s) for c in (1, 4, 14, 16) for s in (0, 1, 2, 3)]
# the column mix of the knob grid: two Atari columns, two more bulk columns and four LSU columns (8 in all)
MIX = (ATARI, ATARI, 2048, 8208, 8, 1, 68, 2047)
MIX_N = (7, 512)
# one Atari column at n = 4096: 125 items per CTA at one CTA per SM, so every stage is refilled several times
WIDE = (ATARI, 8)
WIDE_N = 4096

TREE_SIZES = (1, 2, 1 << 7, 1 << 14, 1 << 21)
UPDATE_N = (0, 1, 512, 513, 1024, 1025)
SAMPLE_N = (1, 7, 513)


def ring(rng, rows, row_bytes):
    return rng.randint(0, 256, (rows, row_bytes)).astype(np.uint8)


def gather_idx(rng, n, capacity):
    """random slots with the first and last slot and duplicates in every batch of two or more"""
    idx = rng.randint(0, capacity, n).astype(np.int64)
    idx[0] = capacity - 1
    if n > 1:
        idx[1] = 0
    if n > 3:
        idx[3] = idx[2]
        idx[-1] = 0
    return idx


def priorities(rng, m):
    """m positive priorities (powers of two apart) with a few exact ties"""
    p = 2.0 ** rng.uniform(-6, 3, m)
    p[::7] = 0.5
    return p


def tree_leaves(rng, size):
    """leaves of a start tree: positive priorities on the first 3/4 (at least one leaf), zeros after them"""
    m = max(1, size * 3 // 4)
    leaves = np.zeros(size, np.float64)
    leaves[:m] = priorities(rng, m)
    return leaves, m


def update_batch(rng, n, size):
    """n entries of cb200_per_update: random leaves with duplicates (in every batch of two or more, the last entry
    repeats the first), p_raw random and p_alpha = p_raw ** 0.6"""
    idx = rng.randint(0, size, n).astype(np.int64)
    if n > 1:
        idx[-1] = idx[0]
    if n > 5:
        idx[5] = idx[3]
    p_raw = priorities(rng, n) * 3
    return idx, p_raw ** 0.6, p_raw


# ---- the fused sample + gather + space-to-depth kernel (cb200_gather_s2d, cb200_per_sample_gather_s2d) -------------------
# verbatim ring: (n, n_img, h, w, c, s, small columns).  Atari frames at B = 8 (one s2d row per band), 128 (a partial
# chunk and empty bands with two columns), 512 (three chunks per band with two columns: a stage refill) and 4096 (one
# band of 11 chunks); every s with small frames: run = s * c of 8, 16 and 24 / 32 / 40 bytes (the 8-byte loop over
# several groups), 256 % (8 s) != 0 (idle threads: s = 3, 5, 6), more pixel slots than s2d columns, w / s == 1, chunks
# of more pixels than slots (each thread converts several, stepping by whole rows when slots >= w / s); s2d rows
# above the 2816-byte chunk budget (one row per chunk, shared memory above 48 KiB), the largest below the 227 KiB
# opt-in limit
S2D_RING = [(n, k, 84, 84, 4, 4, "mix" if n in (8, 512) else "none") for n in (8, 128, 512, 4096) for k in (1, 2)] + [
    (512, 1, 64, 10, 8, 1, "mix"),         # s = 1, run 8: 32 slots over 10 columns, 8 rows per chunk
    (16, 1, 4, 6, 16, 1, "none"),          # s = 1, run 16
    (16, 2, 8, 12, 12, 2, "none"),         # run 24
    (8, 1, 10, 4, 20, 2, "mix"),           # run 40
    (1024, 1, 48, 12, 8, 3, "none"),       # s = 3: 10 slots of 24 threads, 16 idle; 4 rows per chunk
    (8, 1, 8, 8, 2, 4, "none"),            # s = 4, run 8
    (1024, 1, 40, 20, 8, 5, "none"),       # s = 5, run 40: 6 slots of 40 threads; 2 rows per chunk
    (512, 2, 36, 24, 4, 6, "none"),        # s = 6, run 24: 5 slots of 48 threads; 2 rows per chunk
    (16, 1, 16, 16, 1, 8, "none"),         # s = 8, run 8
    (8, 1, 8, 8, 1, 8, "mix"),             # w / s == 1 with 4 slots
    (2048, 1, 128, 8, 1, 8, "none"),       # w / s == 1, 8 rows per chunk: each slot steps 4 rows
    (8, 1, 64, 32, 1, 32, "none"),         # s = 32: one slot of 256 threads, w / s == 1, run 32
    (16, 1, 8, 256, 4, 4, "mix"),          # 4096-byte s2d rows: one per chunk, 66 KiB of shared memory
    (8, 1, 4, 896, 4, 4, "none"),          # 14336-byte s2d rows: 229888 bytes of shared memory
]
S2D_CAPACITY = 300                 # ring rows of the verbatim-ring cases
# the geometries the library refuses: shared memory above the opt-in limit (16384-byte s2d rows: 262656 bytes), and
# s > 32, where 8 s threads per pixel leave no pixel slot (h = w = 64, c = 1, s = 64: rows of 16-byte multiples)
S2D_OVER_SMEM = (8, 1, 4, 1024, 4, 4)
S2D_S64 = (8, 1, 64, 64, 1, 64)

# small columns of a "mix" case: (row_bytes, byte offset of both bases): every warp_copy_row path -- 16-byte vectors
# (16, 1040), words (4, 16 at a 4-byte offset) and bytes (1, 3, 2047, 68 at a 1-byte offset); eight columns, the most
# a call takes
SMALL_MIX = ((1, 0), (3, 0), (4, 0), (16, 0), (2047, 0), (16, 4), (68, 1), (1040, 0))

# frame store (s = c = 4): (n, n_img, h, w, frame slots, small columns).  16x16 frames in one chunk per band (TMA
# eligible: 256-byte stride), 84x84 at B = 128 and 512 with two columns (a partial chunk and empty bands; three chunks:
# a refill; both TMA eligible: 2688-byte stride), 84x84 at B = 8 (one row per chunk, a 1344-byte stride: never TMA),
# 8x272 frames (a 1088-byte band: wider than one TMA box), and a store of exactly four frame slots
S2D_FRAMES = [(32, 2, 16, 16, 64, "mix"), (128, 2, 84, 84, 64, "none"), (512, 2, 84, 84, 64, "none"),
              (8, 1, 84, 84, 64, "none"), (8, 1, 8, 272, 64, "none"), (32, 1, 16, 16, 4, "none")]
S2D_FRAME_CAPACITY = 200           # transitions of the frame tables

# prioritized sampling: (tree size, n, n_img, h, w, c, s, frame store, optional outputs).  The ring (or frame table)
# has one row per leaf, so the 2^21-leaf tree draws from 64-byte rows
S2D_PER = [(1, 8, 1, 8, 8, 2, 4, False, ("w", "w32")),
           (1 << 7, 128, 2, 84, 84, 4, 4, False, ("w",)),
           (1 << 7, 8, 1, 8, 8, 2, 4, False, ()),
           (1 << 7, 512, 2, 84, 84, 4, 4, True, ("w32",)),
           (1 << 21, 64, 1, 8, 8, 1, 8, False, ("w", "w32"))]

S2D_REQUIRED = (
    {("ring", r) for r in ("one-chunk", "refill", "partial", "empty-band", "one-band", "bands=Hs", "rc=1", "smem>48K",
                           "run=8", "run=16", "run=8k", "idle-threads", "slots>Ws", "Ws=1", "multi-pass",
                           "multi-pass-dyl")} |
    {("ring", "S=%d" % s) for s in (1, 2, 3, 4, 5, 6, 8, 32)} |
    {("frames", r) for r in ("one-chunk", "refill", "partial", "empty-band", "bands=Hs", "tma", "bulk",
                             "tma-ineligible")} |
    {("box", r) for r in ("one-box", "four-copies", "partial-fallback")} |
    {("small", 0), ("small", 8), ("copy", 16), ("copy", 4), ("copy", 1)} |
    {("per", r) for r in ("size=1", "size=128", "size=2097152", "w", "w32", "no-weights", "frames")})


def frame_table(rng, capacity, slots):
    """the [capacity, 4] int32 frame slots of the stacks a frame store holds: episodes of 1 to 12 transitions, each
    opening with its first frame repeated -- (k, k, k, k), (k, k, k, k+1), (k, k, k+1, k+2) -- then four consecutive
    slots; slot numbers wrap at `slots` (starting two slots before the end), so some stacks wrap the store"""
    rows, f = [], slots - 2
    while len(rows) < capacity:
        frames = [f] * 3
        for _ in range(rng.randint(1, 13)):
            frames.append(f)
            rows.append(frames[-4:])
            f = (f + 1) % slots
    return np.array(rows[:capacity], np.int32)


def frame_idx(rng, n, fidx):
    """n sampled transitions of a frame table: the first four are a stack in four consecutive slots, (k, k, k, k),
    (k, k, k+1, k+2) and a stack that wraps the store (when the table has them), the rest random"""
    idx = rng.randint(0, fidx.shape[0], n).astype(np.int64)
    d = np.diff(fidx.astype(np.int64), axis=1)
    kinds = [(d == 1).all(1), (d == 0).all(1), (d[:, 0] == 0) & (d[:, 1] == 1) & (d[:, 2] == 1), (d < 0).any(1)]
    for i, kind in enumerate(kinds):
        if kind.any():
            idx[i] = np.flatnonzero(kind)[0]
    return idx
