"""CPU helpers of the GEMM kernel tests (test infrastructure only; no GPU, no kernels).

* The bf16 truncation split and the two plane layouts of include/coach_b200.h (core-tiled, header of
  cb200_gemm_desc; row-group interleaved, cb200_tgemm_desc.b_interleaved), in numpy.
* fp64 references of cb200_gemm and cb200_gemm_tiled written from the header's contract, not from the kernels:
  the contraction (``gemm_contract``, ``tiled_mode0``, ``tiled_mode1``) and the epilogue (``epilogue``), which is
  emulated in fp32 (the exact probes) or evaluated in fp64 (the accuracy checks).
* Exact-probe generators.  Operand values are integers times one power of two per operand, one operand sparse, and
  the budget sum_r |A_mr| |B_rn| < 2^23 units holds for every output, so every product and every partial sum in any
  order is exact in fp32: a kernel that issues the 3xBF16 product set correctly must return the exact result bit for
  bit, and one that drops or misplaces a product cannot.  Three kinds cover all six products between them:
    "a_bits": A dense with 17..23 significant bits (hi, mid and lo planes), B sparse in {-1, 0, +1}: a1b1 a2b1 a3b1
    "b_bits": the mirror image: a1b1 a1b2 a1b3
    "mid"   : both operands 9-bit odd integers (hi and mid planes, lo = 0), one of them sparse: a1b1 a1b2 a2b1 a2b2
  and "u8" (uint8 A in {0, 2^j}, B dense with 17..23 bits) the single-plane uint8 path.
"""
import numpy as np

BUDGET = 2.0 ** 23          # sum_r |a| |b| per output, in units of the product's unit
EXTRA = 2.0 ** 20           # |bias| and |pre-filled C| of the probes, same unit: the total stays below 2^24
ACT_NONE, ACT_RELU, ACT_TANH = 0, 1, 2


# ---- planes ---------------------------------------------------------------------------------------------------------
def split3(x):
    """fp32 -> (hi, mid, lo) as uint16 bf16 bit patterns: truncation split, x == hi + mid + lo"""
    x = np.ascontiguousarray(x, dtype=np.float32)
    hb = x.view(np.uint32) & np.uint32(0xffff0000)
    r1 = x - hb.view(np.float32)
    mb = r1.view(np.uint32) & np.uint32(0xffff0000)
    lb = (r1 - mb.view(np.float32)).view(np.uint32)
    return tuple((b >> np.uint32(16)).astype(np.uint16) for b in (hb, mb, lb))


def bf16_value(p):
    """uint16 bf16 bit patterns -> fp32"""
    return (np.asarray(p, dtype=np.uint32) << np.uint32(16)).view(np.float32)


def tiled_elem(r, c, cols):
    """element (r, c) of a [rows, cols] plane matrix in the 8x8 core-tiled format"""
    return ((r // 8) * (cols // 8) + c // 8) * 64 + (r % 8) * 8 + c % 8


def tiled_elem_il(r, c, cols, plane):
    """the same element of plane `plane` in the row-group interleaved format (row group | plane | column core | 64)"""
    return (((r // 8) * 3 + plane) * (cols // 8) + c // 8) * 64 + (r % 8) * 8 + c % 8


def _grid(rows, cols):
    return np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")


def pack_planes(x, nplanes=3, rows=None):
    """fp32 [rows, cols] -> uint16 [nplanes, rows * cols] core-tiled planes (nplanes 1: x must be exact in bf16).
    `rows`: pad the plane matrix to this many rows (zeros)"""
    x = np.asarray(x, dtype=np.float32)
    r, c = _grid(*x.shape)
    rows = x.shape[0] if rows is None else rows
    out = np.zeros((nplanes, rows * x.shape[1]), dtype=np.uint16)
    parts = split3(x)
    if nplanes == 1:
        assert not parts[1].any() and not parts[2].any(), "a single plane holds bf16-exact values only"
    for p in range(nplanes):
        out[p, tiled_elem(r, c, x.shape[1])] = parts[p]
    return out


def pack_planes_il(x):
    """fp32 [rows, cols] -> uint16 [3 * rows * cols] row-group interleaved planes"""
    x = np.asarray(x, dtype=np.float32)
    r, c = _grid(*x.shape)
    out = np.zeros(3 * x.size, dtype=np.uint16)
    for p, part in enumerate(split3(x)):
        out[tiled_elem_il(r, c, x.shape[1], p)] = part
    return out


def unpack_planes(buf, rows, cols, nplanes=3):
    """uint16 [nplanes, >= rows * cols] core-tiled planes -> the bit patterns [nplanes, rows, cols]"""
    r, c = _grid(rows, cols)
    return np.stack([np.asarray(buf[p])[tiled_elem(r, c, cols)] for p in range(nplanes)])


def plane_row(m, npix, batch):
    """plane row of result / operand row m (= b * npix + q -> q * batch + b when npix > 0)"""
    m = np.asarray(m)
    return (m % npix) * batch + m // npix if npix > 0 else m


def transpose_cores(x):
    """every 8x8 core of x [rows, cols] transposed in place (the mutant of a fragment read the wrong way round)"""
    r, c = x.shape
    return x.reshape(r // 8, 8, c // 8, 8).transpose(0, 3, 2, 1).reshape(r, c)


# ---- cb200_gemm -------------------------------------------------------------------------------------------------------
def gather_a(a_src, rowoff, coloff, rowinfo=None, colinfo=None, oh=0, ow=0, lut=None):
    """logical A [a_rows, a_cols] of cb200_gemm_desc: a_src[rowoff[m] + coloff[r]] (through the LUT if given), zero
    where the (rowinfo, colinfo) tap is outside the oh x ow window.  fp64."""
    v = np.asarray(a_src)[np.asarray(rowoff, np.int64)[:, None] + np.asarray(coloff, np.int64)[None, :]]
    v = (np.asarray(lut, np.float64)[v] if lut is not None else v).astype(np.float64)
    if rowinfo is not None:
        ri, ci = np.asarray(rowinfo, np.int64), np.asarray(colinfo, np.int64)
        y = (ri[:, None] >> 16) - (ci[None, :] >> 16)
        x = (ri[:, None] & 0xffff) - (ci[None, :] & 0xffff)
        v = np.where((y >= 0) & (y < oh) & (x >= 0) & (x < ow), v, 0.0)
    return v


def gemm_contract(A, B, transposed=False, ones_col=False):
    """sum_r A(m, r) B(r, n) (or A^T B, plus the row sum_m B[m, :] when ones_col) in fp64"""
    A, B = np.asarray(A, np.float64), np.asarray(B, np.float64)
    if not transposed:
        return A @ B
    out = A.T @ B
    return np.vstack([out, B.sum(0, keepdims=True)]) if ones_col else out


# ---- cb200_gemm_tiled -------------------------------------------------------------------------------------------------
def tiled_mode0(list_ptr, lst, A, W, batch, num_q, n):
    """C[q*B+b, :] = sum over the entries (a_pix, w_blk) of list q of A[a_pix*B+b, :] @ W[w_blk]
    (A [pixels*B, Ca], W [blocks*Ca, n] or [blocks, Ca, n])"""
    A = np.asarray(A)
    Ca = A.shape[1]
    W = np.asarray(W).reshape(-1, Ca, n)
    lst = np.asarray(lst).reshape(-1, 2)
    out = np.zeros((num_q * batch, n), dtype=np.result_type(A, W))
    for q in range(num_q):
        for a_pix, w_blk in lst[list_ptr[q]:list_ptr[q + 1]]:
            out[q * batch:(q + 1) * batch] += A[a_pix * batch:(a_pix + 1) * batch] @ W[w_blk]
    return out


def tiled_mode1(a_pix, A, G, batch, taps, num_q, bias_row=False):
    """C[t*Ca+c, :] = sum_q sum_b A[a_pix[t, q]*B+b, c] G[q*B+b, :]  (+ the row sum over all rows of G)"""
    A, G = np.asarray(A), np.asarray(G)
    Ca = A.shape[1]
    a_pix = np.asarray(a_pix).reshape(taps, num_q)
    out = np.zeros((taps * Ca + (1 if bias_row else 0), G.shape[1]), dtype=np.result_type(A, G))
    for t in range(taps):
        for q in range(num_q):
            out[t * Ca:(t + 1) * Ca] += A[a_pix[t, q] * batch:(a_pix[t, q] + 1) * batch].T @ G[q * batch:(q + 1) * batch]
    if bias_row:
        out[-1] = G[:num_q * batch].sum(0)
    return out


# ---- epilogue -------------------------------------------------------------------------------------------------------
def epilogue(P, dtype, div=0.0, scaled=None, bias=None, act=0, mask=None, mask_act=0, prev=None):
    """bias -> activation -> activation-derivative mask -> (+= prev) of the header's epilogue, on the contraction P.
    dtype float32: the kernels' fp32 operation order (the exact probes); float64: the exact value (accuracy checks).
    div / scaled: uint8 A with a declared divisor -- the rows flagged in `scaled` are divided by div first."""
    f = np.dtype(dtype).type
    v = np.asarray(P, np.float64).astype(dtype)
    if div:
        rows = np.ones(v.shape[0], bool) if scaled is None else np.asarray(scaled)
        v[rows] = v[rows] / f(div)
    if bias is not None:
        v = v + np.asarray(bias).astype(dtype)[None, :]
    if act == ACT_RELU:
        v = np.where(v > 0, v, f(0))
    elif act == ACT_TANH:
        v = np.tanh(v)
    if mask is not None and mask_act:
        y = np.asarray(mask).astype(dtype)
        v = v * (np.where(y > 0, f(1), f(0)) if mask_act == ACT_RELU else f(1) - y * y)
    if prev is not None:
        v = v + np.asarray(prev).astype(dtype)
    return v


# ---- exact probes ---------------------------------------------------------------------------------------------------
def _ternary(rng, shape, density):
    return (rng.rand(*shape) < density) * rng.choice([-1.0, 1.0], size=shape)


def _odd9(rng, shape):
    return rng.choice([-1.0, 1.0], size=shape) * (2 * rng.randint(128, 256, size=shape) + 1)


def _bits(rng, shape, bits):
    """random integers with exactly `bits` significant bits, random sign.  Bit 0 and bit bits - 9 are set: the mid
    plane then starts right below the hi plane and, for bits >= 17, the lo plane is never zero"""
    lo = 2 ** (bits - 1)
    v = rng.randint(lo, 2 * lo, size=shape) | 1 | (1 << max(bits - 9, 0))
    return rng.choice([-1.0, 1.0], size=shape) * v.astype(np.float64)


def probe_operands(kind, a_shape, b_shape, count, rng, a_sparse_mask=None, u8_max_exp=2):
    """Operands (A, B, unit_a, unit_b) of an exact probe.  `count(Aabs, Babs)` is the caller's contraction of two
    non-negative operands (per-output sum_r |a||b|); the sparse side's density is halved until the dense side can take
    >= 17 significant bits (9 for "mid") within BUDGET.  A and B are returned as integers (fp64); the operand values
    are A * unit_a, B * unit_b.  kind: "a_bits" | "b_bits" | "mid" | "u8" (A uint8 in {0, 2^j}, j <= u8_max_exp)."""
    density = 1.0
    dense_a = kind == "a_bits"
    for _ in range(40):
        if kind == "u8":
            S = (rng.rand(*a_shape) < density) * 2.0 ** rng.randint(0, u8_max_exp + 1, size=a_shape)
        elif kind == "mid":
            S = (rng.rand(*a_shape) < density) * _odd9(rng, a_shape)
        else:
            S = _ternary(rng, b_shape if dense_a else a_shape, density)
        ones = np.ones(a_shape if dense_a else b_shape)
        c = float(np.max(count(ones, np.abs(S)) if dense_a else count(np.abs(S), ones), initial=0.0))
        if kind == "mid":
            if c * 511 <= BUDGET:
                return S, _odd9(rng, b_shape), 2.0 ** -12, 2.0 ** -9
        else:
            bits = int(np.floor(np.log2(BUDGET / max(c, 1.0))))
            if bits >= 17:
                bits = min(bits, 23)
                D = _bits(rng, a_shape if dense_a else b_shape, bits)
                unit_d = 2.0 ** -(bits + 2)
                if kind == "u8":
                    return S, D, 1.0, unit_d
                return (D, S, unit_d, 2.0 ** -2) if dense_a else (S, D, 2.0 ** -2, unit_d)
        density /= 2
    raise AssertionError("no probe density meets the budget")


def probe_extra(rng, shape, unit):
    """bias / pre-filled C of a probe: integers below EXTRA in the product unit"""
    return rng.randint(-int(EXTRA), int(EXTRA) + 1, size=shape).astype(np.float64) * unit


def random_operand(dist, shape, rng):
    """accuracy data: "normal", "relu" (post-ReLU normal) or "spread" (magnitudes 2^U[-20, 20], random sign)"""
    if dist == "normal":
        return rng.randn(*shape)
    if dist == "relu":
        return np.maximum(rng.randn(*shape), 0.0)
    return rng.choice([-1.0, 1.0], size=shape) * 2.0 ** rng.uniform(-20, 20, size=shape)
