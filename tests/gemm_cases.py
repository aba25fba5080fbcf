"""Case tables and CPU problem builders of tests/test_gemm_kernels_gpu.py (numpy only; the host tests draw the same
probes).  A problem is a dict of host arrays: the operands as the entry point reads them, the descriptor fields, the
expected result (fp32 emulation for the exact probes, fp64 otherwise) and S = sum |A||B| + |bias| (+ |C before|) per
output, all in the row order of C."""
import numpy as np

import gemm_ref as gr

R_, T_ = gr.ACT_RELU, gr.ACT_TANH
EXACT_KINDS = ("a_bits", "b_bits", "mid")
RANDOM_KINDS = ("normal", "relu", "spread")

# ---- cb200_gemm: one row per case ------------------------------------------------------------------------------------
# M = output rows without the a_ones_col row, R = reduction length; kind f32 / u8 (raw integers, a_u8_div) / lut (uint8
# through the table, no divisor); layout: gather (random row / column-group offsets), info (+ rowinfo / colinfo tap
# masking), plain (rowoff = m * lda), lda (a_lda set: the skinny kernels); vec4 = a_vec4 hint.  bplanes / cplanes: None
# or the npix of the b_prow / c_prow remap (0 = plane row = row).  tune: cb200_tune switches for the call.
GEMM_CASES = [
    dict(id="tc32_N_f32_full_slice", M=129, R=1024, N=16, tr=0, kind="f32", layout="gather", bias=1, act=R_,
         rowmap=1, bplanes=0, cplanes=0, expect="tc<32,N,f32>"),
    dict(id="tc64_N_f32_split4", M=513, R=3136, N=48, tr=0, kind="f32", layout="info", splits=4, bias=1, act=T_,
         expect="tc<64,N,f32>+reduce_vec"),
    dict(id="tc32_T_f32_R1025_ones", M=128, R=1025, N=32, tr=1, kind="f32", layout="gather", ones=1, splits=2,
         mask=R_, expect="tc<32,T,f32>+reduce_vec"),
    dict(id="tc64_T_f32_split17_wide", M=64, R=3136, N=80, tr=1, kind="f32", layout="info", ones=1, splits=17,
         accumulate=1, bplanes=64, expect="tc<64,T,f32>+reduce_wide"),
    dict(id="tc64_N_u8_div255", M=128, R=1024, N=112, tr=0, kind="u8", div=255.0, layout="info", bias=1,
         cplanes=8, expect="tc<64,N,u8>"),
    dict(id="tc32_T_u8_div256_split2", M=128, R=1000, N=32, tr=1, kind="u8", div=256.0, layout="gather", ones=1,
         splits=2, expect="tc<32,T,u8>+reduce_vec"),
    dict(id="tc32_N_u8_div1_accumulate", M=65, R=36, N=16, tr=0, kind="u8", div=1.0, layout="gather", accumulate=1,
         mask=T_, expect="tc<32,N,u8>"),
    dict(id="tc64_T_u8_div255_tanh_mask", M=64, R=1024, N=64, tr=1, kind="u8", div=255.0, layout="info", ones=1,
         mask=T_, expect="tc<64,T,u8>"),
    dict(id="tc64_N_lut", M=127, R=28, N=64, tr=0, kind="lut", layout="gather", bias=1, act=R_,
         expect="tc<64,N,lut>"),
    dict(id="fast256x32_N", M=129, R=1000, N=16, tr=0, kind="f32", layout="info", splits=2, tune={"gemm_tc": 0},
         expect="fast<256,32,N>+reduce_vec"),
    dict(id="fast128x64_T_ones", M=128, R=1000, N=48, tr=1, kind="f32", layout="gather", ones=1,
         tune={"gemm_tc": 0}, expect="fast<128,64,T>"),
    dict(id="fast128x128_N", M=513, R=4, N=112, tr=0, kind="f32", layout="gather", bias=1, act=R_,
         tune={"gemm_tc": 0}, expect="fast<128,128,N>"),
    dict(id="fast256x32_T_n20", M=128, R=28, N=20, tr=1, kind="f32", layout="gather", rowmap=1,
         expect="fast<256,32,T>"),
    dict(id="fast128x64_N_n36", M=65, R=36, N=36, tr=0, kind="f32", layout="info", mask=R_,
         expect="fast<128,64,N>"),
    dict(id="fast128x128_T_n100", M=128, R=1025, N=100, tr=1, kind="f32", layout="info", splits=3,
         expect="fast<128,128,T>+reduce_vec"),
    dict(id="ffma128x32_N", M=128, R=36, N=16, tr=0, kind="f32", layout="info", vec4=0, bias=1,
         expect="ffma<128,32,N>"),
    dict(id="ffma128x32_T", M=127, R=1000, N=32, tr=1, kind="f32", layout="gather", vec4=0, accumulate=1,
         expect="ffma<128,32,T>"),
    dict(id="ffma128x64_N", M=129, R=1025, N=48, tr=0, kind="f32", layout="gather", vec4=0, splits=3,
         expect="ffma<128,64,N>+reduce_vec"),
    dict(id="ffma128x64_T", M=513, R=28, N=80, tr=1, kind="f32", layout="info", vec4=0, mask=R_,
         expect="ffma<128,64,T>"),
    dict(id="ffma32x32_N_scalar_reduce", M=63, R=100, N=7, tr=0, kind="f32", layout="gather", vec4=0, splits=3,
         bias=1, expect="ffma<32,32,N>+reduce_scalar"),
    dict(id="ffma32x32_T", M=64, R=3136, N=48, tr=1, kind="f32", layout="gather", vec4=0, act=T_,
         expect="ffma<32,32,T>"),
    dict(id="skinny_n", M=513, R=1000, N=6, tr=0, kind="f32", layout="lda", bias=1, expect="skinny_n"),
    dict(id="skinny_r", M=129, R=4, N=112, tr=0, kind="f32", layout="lda", act=R_, expect="skinny_r"),
    dict(id="skinny_tn_ones", M=64, R=1025, N=8, tr=1, kind="f32", layout="lda", ones=1, expect="skinny_tn"),
    dict(id="skinny_off_ffma", M=65, R=1000, N=6, tr=0, kind="f32", layout="lda", tune={"gemm_skinny": 0},
         expect="ffma<128,32,N>"),
]


def _pos(d, k, default=0):
    return d.get(k, default)


def gemm_slices(case):
    """(splits, reduction indices per slice) as cb200_gemm derives them"""
    R, s = case["R"], max(1, _pos(case, "splits", 1))
    rps = -(-R // s)
    rps = -(-rps // 16) * 16
    return -(-R // rps), rps


def gemm_gamma(case, dispatch):
    """error bound factor of the accuracy check: tensor cores (truncating fp32 accumulation per k16 step):
    (k16 steps per slice + splits + 8) 2^-23; fp32 FFMA chains (round to nearest): (terms per slice + splits + 8) 2^-24"""
    s, rps = gemm_slices(case)
    if dispatch.startswith("tc<"):
        return (rps // 16 + s + 8) * 2.0 ** -23
    return (min(rps, case["R"]) + s + 8) * 2.0 ** -24


def gemm_problem(case, kind, seed=0):
    rng = np.random.RandomState(seed)
    M, R, N, tr = case["M"], case["R"], case["N"], bool(case["tr"])
    ones = bool(_pos(case, "ones"))
    a_rows, a_cols = (R, M) if tr else (M, R)
    Mout = M + (1 if ones else 0)
    layout, u8 = case["layout"], case["kind"] in ("u8", "lut")
    div = float(_pos(case, "div", 0.0))
    p = dict(case=case, kind=kind, a_rows=a_rows, a_cols=a_cols, Mout=Mout, div=div)
    # tap masking of the gather layout: (i, j) per row, (a, b) per aligned group of 4 columns, window 4 x 4
    mask = np.ones((a_rows, a_cols), bool)
    rowinfo = colinfo = None
    if layout == "info":
        ij = rng.randint(0, 6, size=(a_rows, 2))
        ab = np.repeat(rng.randint(0, 3, size=(-(-a_cols // 4), 2)), 4, axis=0)[:a_cols]
        rowinfo = (ij[:, 0] << 16 | ij[:, 1]).astype(np.int32)
        colinfo = (ab[:, 0] << 16 | ab[:, 1]).astype(np.int32)
        y = ij[:, None, 0] - ab[None, :, 0]
        x = ij[:, None, 1] - ab[None, :, 1]
        mask = (y >= 0) & (y < 4) & (x >= 0) & (x < 4)
    p.update(rowinfo=rowinfo, colinfo=colinfo, oh=4, ow=4)

    def count(Aabs, Babs):
        return gr.gemm_contract(Aabs * mask, Babs, tr)

    if kind in RANDOM_KINDS:
        A = rng.randint(0, 256, size=(a_rows, a_cols)).astype(np.float64) if u8 else \
            gr.random_operand(kind, (a_rows, a_cols), rng)
        B = gr.random_operand(kind, (R, N), rng)
        ua = ub = 1.0
    else:
        A, B, ua, ub = gr.probe_operands(kind, (a_rows, a_cols), (R, N), count, rng)
    unit = ua * ub
    A = A * mask
    if u8:
        raw = A.astype(np.uint8)
        assert np.array_equal(raw, A)
        lut = (np.arange(256, dtype=np.float32) / np.float32(div)) if div else \
            np.arange(256, dtype=np.float32) * np.float32(2.0 ** -8)
        a_val = raw.astype(np.float64) if div else lut[raw].astype(np.float64)
    else:
        a_val = (A * ua).astype(np.float32).astype(np.float64)
        lut = None
        assert kind in RANDOM_KINDS or np.array_equal(a_val, A * ua)
    b_val = (B * ub).astype(np.float32)
    assert kind in RANDOM_KINDS or np.array_equal(b_val.astype(np.float64), B * ub)
    # operand memory: the logical A at table-driven offsets; masked-out entries hold garbage the kernel must not read
    if layout == "lda":
        lda = -(-a_cols // 4) * 4 + 4
        rowoff = (np.arange(a_rows) * lda).astype(np.int32)
        coloff = np.arange(a_cols).astype(np.int32)
        size = a_rows * lda
        p["a_lda"] = lda
    else:
        groups = -(-a_cols // 4)
        width = 4 * groups + 4
        rowoff = (rng.permutation(a_rows) * width).astype(np.int32)
        coloff = (rng.permutation(groups)[np.arange(a_cols) // 4] * 4 + np.arange(a_cols) % 4).astype(np.int32)
        size = a_rows * width
        p["a_lda"] = 0
    off = rowoff[:, None].astype(np.int64) + coloff[None, :]
    if u8:
        src = np.full(size, 255, np.uint8)
        src[off] = np.where(mask, raw, 255)
    else:
        src = np.full(size, 7.0 * (np.abs(a_val).max() + 1.0), np.float32)
        src[off] = np.where(mask, a_val, src[0]).astype(np.float32)
    p.update(a_src=src, lut=lut, rowoff=rowoff, coloff=coloff, b=b_val)
    assert np.array_equal(gr.gather_a(src, rowoff, coloff, rowinfo, colinfo, 4, 4,
                                      lut if (u8 and not div) else None), a_val)
    # epilogue inputs
    exact = kind not in RANDOM_KINDS
    scale = 1.0 if not exact else unit
    bias = mask_y = prev = rowmap = None
    if _pos(case, "bias"):
        bias = (gr.probe_extra(rng, N, unit) if exact else rng.randn(N)).astype(np.float32)
    mact = _pos(case, "mask")
    if mact == R_:
        mask_y = rng.choice([-1.0, 1.0], size=(Mout, N)).astype(np.float32)
    elif mact == T_:
        mask_y = rng.uniform(-1, 1, size=(Mout, N)).astype(np.float32)
    if _pos(case, "accumulate"):
        prev = (gr.probe_extra(rng, (Mout, N), unit) if exact else rng.randn(Mout, N)).astype(np.float32)
    rowmap = rng.permutation(Mout).astype(np.int32) if _pos(case, "rowmap") else np.arange(Mout, dtype=np.int32)
    p.update(bias=bias, act=_pos(case, "act"), mask_y=mask_y, mask_act=mact, prev=prev,
             rowmap=rowmap if _pos(case, "rowmap") else None)
    # expected result, rows in m order, then scattered through the row map
    P = gr.gemm_contract(a_val, b_val, tr, ones)
    Sabs = gr.gemm_contract(np.abs(a_val), np.abs(b_val), tr, ones)
    scaled = np.arange(Mout) < (a_cols if tr else Mout)          # the a_ones_col row is not divided
    mask_m = mask_y[rowmap] if mask_y is not None else None
    prev_m = prev[rowmap] if prev is not None else None
    args = dict(div=div if (u8 and div) else 0.0, scaled=scaled, bias=bias, act=p["act"], mask=mask_m,
                mask_act=mact, prev=prev_m)
    want = gr.epilogue(P, np.float32 if exact else np.float64, **args)
    if u8 and div:
        Sabs = np.where(scaled[:, None], Sabs / div, Sabs)
    Sabs = Sabs + (np.abs(bias)[None, :] if bias is not None else 0) + (np.abs(prev_m) if prev is not None else 0)
    out = np.zeros((Mout, N), want.dtype)
    S = np.zeros((Mout, N))
    out[rowmap] = want
    S[rowmap] = Sabs
    p.update(want=out, S=S, unit=scale, exact=exact, P=P)
    # outputs whose budget guarantees exact fp32 arithmetic (the a_ones_col row of a dense-B probe can exceed it)
    p["exact_rows"] = (S <= (2.0 ** 24 - 1) * unit).all(1) if exact else np.zeros(Mout, bool)
    return p


# ---- cb200_gemm_tiled ------------------------------------------------------------------------------------------------
def _lists(lengths, a_pixels, blocks, rng):
    return [[(int(rng.randint(a_pixels)), int(rng.randint(blocks))) for _ in range(k)] for k in lengths]


TILED_CASES = [
    # mode 0: B = 32 (a 128-row tile reaches 3 pixels further and past the last row of A), 32 chunks in one slice,
    # an empty tap list
    dict(id="m0_bn32_32chunks", mode=0, B=32, Ca=32, n=32, lengths=[32, 5, 0, 17, 32], a_pixels=6, blocks=7,
         bias=1, act=R_, cplanes=1, expect="tiled<32,N,3>"),
    # split count leaving the short lists without chunks in the last slices
    dict(id="m0_bn64_split3", mode=0, B=96, Ca=64, n=64, lengths=[6, 1, 0, 3], a_pixels=5, blocks=6, splits=3,
         mask=R_, rowmap=1, expect="tiled<64,N,3>+reduce_vec"),
    dict(id="m0_bn128_tanh_planes", mode=0, B=160, Ca=128, n=128, lengths=[4, 2, 3], a_pixels=4, blocks=5, splits=2,
         mask_planes=T_, cplanes=1, expect="tiled<128,N,3>+reduce_vec"),
    dict(id="m0_bn64_n192", mode=0, B=512, Ca=256, n=192, lengths=[2, 1], a_pixels=2, blocks=3, bias=1, act=T_,
         cplanes=1, expect="tiled<64,N,3>"),
    dict(id="m0_bn32_u8_div255", mode=0, B=32, Ca=64, n=32, lengths=[4, 0, 16], a_pixels=4, blocks=5, na=1,
         div=255.0, bias=1, expect="tiled<32,N,1>"),
    dict(id="m0_bn64_u8_div256", mode=0, B=96, Ca=128, n=64, lengths=[3, 8], a_pixels=3, blocks=4, na=1, div=256.0,
         splits=2, mask_planes=R_, expect="tiled<64,N,1>+reduce_vec"),
    dict(id="m0_bn128_u8_div1", mode=0, B=160, Ca=32, n=128, lengths=[9, 2], a_pixels=3, blocks=4, na=1, div=1.0,
         act=R_, cplanes=1, expect="tiled<128,N,1>"),
    # mode 1: tap tables with 1, 2, 3 stride classes and a non-uniform one (bulk copies)
    dict(id="m1_bn32_tma2", mode=1, B=64, Ca=32, n=32, taps=6, num_q=4, a_pixels=12, deltas=[2], bias_row=1,
         expect="tiled<32,T,3>/tma2"),
    dict(id="m1_bn64_tma3_split3", mode=1, B=32, Ca=32, n=64, taps=9, num_q=6, a_pixels=30, deltas=[1, 3],
         bias_row=1, splits=3, expect="tiled<64,T,3>/tma3+reduce_vec"),
    dict(id="m1_bn128_tma1_Ca256", mode=1, B=32, Ca=256, n=128, taps=2, num_q=8, a_pixels=10, deltas=[1],
         bias_row=1, splits=2, expect="tiled<128,T,3>/tma1+reduce_vec"),
    dict(id="m1_bn64_bulk_nonuniform", mode=1, B=32, Ca=64, n=64, taps=4, num_q=5, a_pixels=20, deltas=None,
         mask_planes=R_, expect="tiled<64,T,3>/bulk"),
    dict(id="m1_bn32_u8_div255_tma1", mode=1, B=32, Ca=64, n=32, taps=4, num_q=3, a_pixels=9, deltas=[2], na=1,
         div=255.0, expect="tiled<32,T,1>/tma1"),
    dict(id="m1_bn64_u8_div256_bias_row", mode=1, B=64, Ca=128, n=64, taps=1, num_q=16, a_pixels=16, deltas=[1],
         na=1, div=256.0, bias_row=1, splits=2, expect="tiled<64,T,1>/tma1+reduce_vec"),
    dict(id="m1_bn128_u8_div1_tma2", mode=1, B=32, Ca=32, n=128, taps=6, num_q=4, a_pixels=12, deltas=[1], na=1,
         div=1.0, rowmap=1, expect="tiled<128,T,1>/tma2"),
]


def _a_pix(case, rng):
    """tap table [taps, num_q]: inside every 128-row tile consecutive taps sit deltas[k % len] pixels apart at every
    output pixel (a_cols < 128: 128 / a_cols taps per tile); deltas None: a non-uniform stride"""
    taps, nq, Ca, npx = case["taps"], case["num_q"], case["Ca"], case["a_pixels"]
    per = max(1, 128 // Ca)
    t = np.zeros((taps, nq), np.int64)
    for tile in range(-(-taps // per)):
        t0, t1 = tile * per, min(taps, tile * per + per)
        if case["deltas"] is None:
            t[t0:t1] = rng.randint(0, npx, size=(t1 - t0, nq))
            continue
        delta = case["deltas"][tile % len(case["deltas"])]
        base = rng.randint(0, npx - (t1 - 1 - t0) * delta, size=nq)
        for k in range(t0, t1):
            t[k] = base + (k - t0) * delta
    assert 0 <= t.min() and t.max() < npx
    return t.astype(np.int32)


def tiled_slices(case):
    if case["mode"] == 0:
        total = max(case["lengths"]) * (case["Ca"] // 32)
    else:
        total = case["num_q"] * (case["B"] // 32)
    s = max(1, _pos(case, "splits", 1))
    cps = -(-total // s)
    return -(-total // cps), cps


def tiled_gamma(case):
    s, cps = tiled_slices(case)
    return (2 * cps + s + 8) * 2.0 ** -23


def tiled_problem(case, kind, seed=0):
    rng = np.random.RandomState(seed)
    B, Ca, n, mode = case["B"], case["Ca"], case["n"], case["mode"]
    na = _pos(case, "na", 3)
    div = float(_pos(case, "div", 0.0))
    p = dict(case=case, kind=kind, na=na, div=div)
    if mode == 0:
        lists = _lists(case["lengths"], case["a_pixels"], case["blocks"], rng)
        ptr = np.concatenate([[0], np.cumsum([len(l) for l in lists])]).astype(np.int32)
        flat = np.array([e for l in lists for e in l] or [(0, 0)], np.int32).reshape(-1, 2)
        num_q = len(lists)
        a_shape, b_shape = (case["a_pixels"] * B, Ca), (case["blocks"] * Ca, n)
        M = num_q * B

        def contract(A_, B_):
            return gr.tiled_mode0(ptr, flat, A_, B_, B, num_q, n)
        p.update(list_ptr=ptr, list=flat, num_q=num_q, max_list_len=max(case["lengths"]))
    else:
        a_pix = _a_pix(case, rng)
        taps, num_q = case["taps"], case["num_q"]
        a_shape, b_shape = (case["a_pixels"] * B, Ca), (num_q * B, n)
        M = taps * Ca + (1 if _pos(case, "bias_row") else 0)

        def contract(A_, B_, bias_row=False):
            return gr.tiled_mode1(a_pix, A_, B_, B, taps, num_q, bias_row)
        p.update(a_pix=a_pix, num_q=num_q, taps=taps)
    if kind in RANDOM_KINDS:
        A = rng.randint(0, 256, size=a_shape).astype(np.float64) if na == 1 else gr.random_operand(kind, a_shape, rng)
        Bm = gr.random_operand(kind, b_shape, rng)
        ua = ub = 1.0
    else:
        A, Bm, ua, ub = gr.probe_operands(kind, a_shape, b_shape, contract, rng)
    exact = kind not in RANDOM_KINDS
    unit = ua * ub
    a_val, b_val = (A * ua).astype(np.float32), (Bm * ub).astype(np.float32)
    assert kind in RANDOM_KINDS or (np.array_equal(a_val.astype(np.float64), A * ua) and
                                    np.array_equal(b_val.astype(np.float64), Bm * ub))
    p.update(A=a_val, Bm=b_val, M=M)
    bias = mask_y = None
    if _pos(case, "bias"):
        bias = (gr.probe_extra(rng, n, unit) if exact else rng.randn(n)).astype(np.float32)
    mact = _pos(case, "mask") or _pos(case, "mask_planes")
    if mact == R_:
        mask_y = rng.choice([-1.0, 1.0], size=(M, n)).astype(np.float32)
    elif mact == T_:
        mask_y = rng.uniform(-1, 1, size=(M, n)).astype(np.float32)
    rowmap = rng.permutation(M).astype(np.int32) if _pos(case, "rowmap") else None
    rows = rowmap if rowmap is not None else np.arange(M)
    # mask_y is indexed like C (through the row map), mask_planes like the result planes (row m)
    mask_c = None
    if mask_y is not None:
        mask_c = np.zeros_like(mask_y)
        mask_c[rows] = mask_y
    p.update(bias=bias, act=_pos(case, "act"), mask_m=mask_y, mask_c=mask_c, mask_act=mact, rowmap=rowmap)
    kw = dict(bias_row=True) if (mode == 1 and _pos(case, "bias_row")) else {}
    P = contract(a_val.astype(np.float64), b_val.astype(np.float64), **kw)
    Sabs = contract(np.abs(a_val).astype(np.float64), np.abs(b_val).astype(np.float64), **kw)
    scaled = np.arange(M) < (M - 1 if kw else M)                  # the bias row (sum of G) is not divided
    args = dict(div=div if na == 1 else 0.0, scaled=scaled, bias=bias, act=p["act"], mask=mask_y, mask_act=mact)
    want = gr.epilogue(P, np.float32 if exact else np.float64, **args)
    if na == 1:
        Sabs = np.where(scaled[:, None], Sabs / div, Sabs)
    Sabs = Sabs + (np.abs(bias)[None, :] if bias is not None else 0)
    out = np.zeros((M, n), want.dtype)
    S = np.zeros((M, n))
    out[rows] = want
    S[rows] = Sabs
    p.update(want=out, S=S, unit=unit if exact else 1.0, exact=exact, P=P, contract=contract)
    p["exact_rows"] = (S <= (2.0 ** 24 - 1) * unit).all(1) if exact else np.zeros(M, bool)
    return p
