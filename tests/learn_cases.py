"""Case table of tests/test_learn_kernels_gpu.py: the shapes and edge values at which the learn-step kernels are checked
against tests/learn_ref.py, and the data generators (numpy only)."""
import numpy as np

F32 = np.float32

# the Atari DQN's parameters (8x8x4x32, 4x4x32x64, 3x3x64x64 convolutions, Dense(512) on 3136 features, Dense(6)), each
# tensor padded to a multiple of 8 elements as in the flat parameter buffer
ATARI_PARAMS = sum((k + 7) // 8 * 8 for k in (8 * 8 * 4 * 32, 32, 4 * 4 * 32 * 64, 64, 3 * 3 * 64 * 64, 64,
                                              3136 * 512, 512, 512 * 6, 6))

COLSUM_COLS = (1, 2, 3, 6, 7, 31, 32, 100, 255, 256, 257, 512, 3136)
COLSUM_ROWS = (1, 7, 8, 9, 512, 4096, 204800, 10 ** 6)
COLSUM_MAX_ELEMS = 1 << 25          # the larger products (e.g. 3136 x 10^6) repeat a covered path at 100x the memory
COLSUM_CASES = [(r, c) for c in COLSUM_COLS for r in COLSUM_ROWS if r * c <= COLSUM_MAX_ELEMS]

SUMSQ_N = (1, 255, 256, 4095, 4096, 4097, 4096 * 1024, 4096 * 1024 + 1, ATARI_PARAMS)

ADAM_N = (1, 3, 4, 5, 8, 1023, "big", "big+1")     # "big": 4 * 8 * SM * 256 + 4 * 123, past the float4 grid-stride
POLYAK_RATES = (0.0, 1.0, 1e-3, 5e-3, 1.0 / 3)

TRANSPOSE_DIMS = (1, 7, 8, 31, 32, 33, 512, 3136)

# (batch, h, w, c, s): s in {1, 2, 4}, c in {2, 4, 8} with s c % 8 == 0, odd w / s (the X-pair loop), h / s = 1, and the
# Atari geometry at batch 8, 520 and 4096 (past the 16-per-SM grid cap)
U8_S2D_CASES = [(8, 6, 10, 8, 1), (8, 4, 6, 4, 2), (520, 8, 6, 8, 2), (8, 4, 12, 2, 4), (8, 4, 4, 4, 4),
                (520, 8, 20, 8, 4), (8, 84, 84, 4, 4), (520, 84, 84, 4, 4), (4096, 84, 84, 4, 4)]

REGRESSION_B = (1, 31, 32, 33, 1024, 1025, 4096)
REGRESSION_W = (1, 6, 18)
DUELING_A = (1, 2, 3, 6, 18)
DUELING_B = (1, 255, 256, 257, 4096)
TD_A = (1, 2, 18)


def spread(rng, shape, lo=-20, hi=20):
    """magnitudes 2^U[lo, hi], random sign"""
    return (rng.choice([-1.0, 1.0], size=shape) * 2.0 ** rng.uniform(lo, hi, size=shape)).astype(F32)


def special_row(cols):
    """one row of edge values for the plane producers: +-0, subnormals, 2^+-100, exact bf16 values, random"""
    v = [0.0, -0.0, 2.0 ** -149, -(2.0 ** -140), 2.0 ** -127 * 1.5, 2.0 ** 100, -(2.0 ** -100), 1.0, -3.0, 0.1]
    row = np.resize(np.array(v, F32), cols)
    return row


def sumsq_data(n, rng, overflow=False):
    """wide dynamic range, every 5th entry zero; `overflow`: one entry whose square overflows fp32"""
    x = spread(rng, n, -30, 30)
    x[::5] = 0
    if overflow:
        x[n // 2] = F32(3e19)
    return x
