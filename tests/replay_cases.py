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
