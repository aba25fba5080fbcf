"""The GEMM kernels at the C ABI (pytest -m gpu): every row of tests/gemm_cases.py builds a cb200_gemm_desc /
cb200_tgemm_desc directly and runs

* exact probes (tests/gemm_ref.py): operands for which every product and partial sum is exact in fp32, so the result
  must equal the fp32 emulation of the header's contract bit for bit (tanh activations / masks: a few ulp);
* twins that issue the same products in the same order and must agree bit for bit: every call twice, B planes vs fp32
  B (cb200_gemm), interleaved vs planar B planes (tiled mode 0), bulk copies vs TMA boxes for A^T (tiled mode 1),
  c_planes vs the split of the fp32 result, planes-only vs planes + fp32 result;
* random data (normal, post-ReLU, magnitudes 2^[-20, 20]): |got - fp64| <= gamma * S with S = sum |A||B| + |bias|,
  gamma from the accumulation count (gemm_cases.*_gamma), and at most 4x the error of an fp32 CPU evaluation.
  The observed e / S is printed (pytest -rA);
* cb200_last_dispatch() of every call; the last test fails if a listed kernel variant was never run."""
import ctypes

import numpy as np
import pytest
import torch

import gemm_cases as gc
import gemm_ref as gr

pytestmark = pytest.mark.gpu

DISPATCHED = set()


def _lib():
    from coach_b200 import _lib
    return _lib, _lib.load()


class _Dev(object):
    """host arrays -> device tensors kept alive for one call"""

    def __init__(self):
        self.keep = []

    def __call__(self, x):
        if x is None:
            return None
        x = np.ascontiguousarray(x)
        t = torch.from_numpy(x.view(np.int16) if x.dtype == np.uint16 else x).cuda()
        self.keep.append(t)
        return t.data_ptr()

    def zeros(self, *shape, dtype=torch.float32):
        t = torch.zeros(*shape, dtype=dtype, device="cuda")
        self.keep.append(t)
        return t


def _ceil8(x):
    return -(-x // 8) * 8


def _planes_np(t):
    return t.cpu().numpy().view(np.uint16)


def run_gemm(p, b_planes=True, tune=None):
    L, lib = _lib()
    case, dv, d = p["case"], _Dev(), L.GemmDesc()
    N, Mout, R = case["N"], p["Mout"], case["R"]
    d.a_src, d.a_lut = dv(p["a_src"]), dv(p["lut"])
    d.a_rowoff, d.a_coloff = dv(p["rowoff"]), dv(p["coloff"])
    d.a_rowinfo, d.a_colinfo, d.a_oh, d.a_ow = dv(p["rowinfo"]), dv(p["colinfo"]), p["oh"], p["ow"]
    d.a_rows, d.a_cols, d.a_transposed = p["a_rows"], p["a_cols"], case["tr"]
    d.b, d.ldb, d.n = dv(p["b"]), N, N
    c = dv.zeros(Mout, N) if p["prev"] is None else torch.from_numpy(p["prev"].copy()).cuda()
    d.c, d.ldc = c.data_ptr(), N
    d.bias, d.act, d.mask_y, d.mask_act = dv(p["bias"]), p["act"], dv(p["mask_y"]), p["mask_act"]
    d.c_rowmap, d.accumulate = dv(p["rowmap"]), 1 if p["prev"] is not None else 0
    splits = case.get("splits", 1)
    d.splits = splits
    if splits > 1:
        d.workspace = dv.zeros(splits * Mout * N).data_ptr()
    d.a_vec4 = case.get("vec4", 1)
    assert not d.a_vec4 or p["a_cols"] % 4 == 0
    d.a_ones_col, d.a_u8_div = case.get("ones", 0), p["div"]
    if b_planes and case.get("bplanes") is not None:
        npix = case["bplanes"]
        rows = gr.plane_row(np.arange(R), npix, R // npix if npix else 0)
        bp = np.zeros_like(p["b"])
        bp[rows] = p["b"]
        d.b_planes, d.b_plane_stride = dv(gr.pack_planes(bp)), R * N
        d.b_prow_npix, d.b_prow_batch = npix, (R // npix if npix else 0)
    cpl = None
    if case.get("cplanes") is not None:
        npix = case["cplanes"]
        cpl = dv.zeros(3, _ceil8(Mout) * N, dtype=torch.int16)
        d.c_planes, d.c_plane_stride, d.c_plane_cols = cpl.data_ptr(), _ceil8(Mout) * N, N
        d.c_prow_npix, d.c_prow_batch = npix, (Mout // npix if npix else 0)
    d.a_lda = p["a_lda"]
    tune = dict(case.get("tune", {}), **(tune or {}))
    try:
        for k, v in tune.items():
            assert lib.cb200_tune(k.encode(), v) == 0
        L.check(lib.cb200_gemm(ctypes.byref(d), L.current_stream()))
        dispatch = lib.cb200_last_dispatch().decode()
    finally:
        for k in tune:
            lib.cb200_tune(k.encode(), 1)
    torch.cuda.synchronize()
    DISPATCHED.add(dispatch)
    return dict(c=c.cpu().numpy(), planes=_planes_np(cpl) if cpl is not None else None, dispatch=dispatch)


def run_tiled(p, interleaved=False, a_pix_host=True, c_null=False):
    L, lib = _lib()
    case, dv, d = p["case"], _Dev(), L.TGemmDesc()
    B, Ca, n, M, mode = case["B"], case["Ca"], case["n"], p["M"], case["mode"]
    d.mode, d.batch = mode, B
    a_rows = p["A"].shape[0]
    d.a_planes, d.a_plane_stride, d.a_cols = dv(gr.pack_planes(p["A"], p["na"])), a_rows * Ca, Ca
    d.a_num_planes, d.a_u8_div, d.a_rows = p["na"], p["div"], a_rows
    b_rows = p["Bm"].shape[0]
    if interleaved:
        d.b_planes, d.b_plane_stride, d.b_interleaved = dv(gr.pack_planes_il(p["Bm"])), 0, 1
    else:
        d.b_planes, d.b_plane_stride = dv(gr.pack_planes(p["Bm"])), b_rows * n
    d.n, d.b_rows = n, b_rows
    host = None
    if mode == 0:
        d.list_ptr, d.list, d.max_list_len, d.num_q = dv(p["list_ptr"]), dv(p["list"]), p["max_list_len"], p["num_q"]
    else:
        host = np.ascontiguousarray(p["a_pix"].reshape(-1), dtype=np.int32)
        d.a_pix, d.num_q, d.taps = dv(host), p["num_q"], p["taps"]
        d.bias_row = case.get("bias_row", 0)
        if a_pix_host:
            d.a_pix_host = host.ctypes.data
    c = None if c_null else dv.zeros(M, n)
    d.c, d.ldc = (None if c is None else c.data_ptr()), n
    d.bias, d.act, d.c_rowmap = dv(p["bias"]), p["act"], dv(p["rowmap"])
    if case.get("mask_planes"):
        mp = np.zeros((_ceil8(M), n), np.float32)
        mp[:M] = p["mask_m"]
        d.mask_planes, d.mask_plane_stride = dv(gr.pack_planes(mp)), _ceil8(M) * n
        d.mask_act, d.c_plane_cols = p["mask_act"], n
    elif p["mask_act"]:
        d.mask_y, d.mask_act = dv(p["mask_c"]), p["mask_act"]
    splits = case.get("splits", 1)
    d.splits = splits
    if splits > 1:
        d.workspace = dv.zeros(splits * M * n).data_ptr()
    cpl = None
    if case.get("cplanes") or c_null:
        cpl = dv.zeros(3, _ceil8(M) * n, dtype=torch.int16)
        d.c_planes, d.c_plane_stride, d.c_plane_cols = cpl.data_ptr(), _ceil8(M) * n, n
    L.check(lib.cb200_gemm_tiled(ctypes.byref(d), L.current_stream()))
    dispatch = lib.cb200_last_dispatch().decode()
    torch.cuda.synchronize()
    DISPATCHED.add(dispatch)
    return dict(c=None if c is None else c.cpu().numpy(), planes=_planes_np(cpl) if cpl is not None else None,
                dispatch=dispatch)


# ---- checks ---------------------------------------------------------------------------------------------------------
def check_exact(p, got, name):
    rows = p["exact_rows"]
    assert rows.sum() >= len(rows) - 1, "%s: the probe budget fails on %d rows" % (name, len(rows) - rows.sum())
    g, w = got[rows].astype(np.float64), p["want"][rows].astype(np.float64)
    tanh = p["act"] == gr.ACT_TANH or p["mask_act"] == gr.ACT_TANH
    if not tanh:
        bad = np.argwhere(g != w)
        assert bad.size == 0, "%s: %d of %d outputs differ from the exact result, first %s: got %r want %r" % (
            name, len(bad), g.size, bad[0], g[tuple(bad[0])], w[tuple(bad[0])])
        return
    # tanhf is not correctly rounded and 1 - y*y may be contracted into an FMA: a few ulp of the larger operand
    tol = 2.0 ** -21 * (np.abs(w) + p["S"][rows])
    err = np.abs(g - w)
    worst = np.argmax(err - tol)
    assert np.all(err <= tol), "%s: error %.3e above the ulp bound %.3e" % (name, err.flat[worst], tol.flat[worst])


def check_planes(p, got_c, planes, rows_out, npix=0, batch=0):
    """planes of the result == the truncation split of the fp32 result, at the plane row of every result row m"""
    n = got_c.shape[1]
    M = len(rows_out)
    pl = gr.unpack_planes(planes, _ceil8(M), n)
    prow = gr.plane_row(np.arange(M), npix, batch)
    for k, part in enumerate(gr.split3(got_c[rows_out])):
        assert np.array_equal(pl[k][prow], part), "plane %d differs from the split of the fp32 result" % k


def check_accuracy(name, p, got, gamma, cpu32, dispatch):
    want, S = p["want"].astype(np.float64), p["S"]
    e = np.abs(got.astype(np.float64) - want)
    ratio = np.where(S > 0, e / np.where(S > 0, S, 1.0), np.where(e > 0, np.inf, 0.0))
    e_cpu = np.abs(cpu32.astype(np.float64) - want).max()
    print("%-40s %-30s %-6s max e/S %.3e  p99.9 %.3e  gamma %.3e  (max e %.3e, fp32 CPU %.3e)" % (
        name, dispatch, p["kind"], ratio.max(), np.percentile(ratio, 99.9), gamma, e.max(), e_cpu))
    assert ratio.max() <= gamma, "%s: e/S %.3e above gamma %.3e" % (name, ratio.max(), gamma)
    assert e.max() <= 4 * e_cpu + 2e-6 * np.abs(want).max(), "%s: error %.3e vs fp32 CPU %.3e" % (name, e.max(), e_cpu)


def _gemm_cpu32(p):
    a = gr.gather_a(p["a_src"], p["rowoff"], p["coloff"], p["rowinfo"], p["colinfo"], p["oh"], p["ow"],
                    p["lut"] if p["lut"] is not None and not p["div"] else None).astype(np.float32)
    b = p["b"]
    P = a.T @ b if p["case"]["tr"] else a @ b
    if p["case"].get("ones"):
        P = np.vstack([P, b.sum(0, dtype=np.float32, keepdims=True)])
    rm = p["rowmap"] if p["rowmap"] is not None else np.arange(p["Mout"])
    Mout = p["Mout"]
    scaled = np.arange(Mout) < (p["a_cols"] if p["case"]["tr"] else Mout)
    v = gr.epilogue(P, np.float32, div=p["div"] if p["case"]["kind"] == "u8" else 0.0, scaled=scaled,
                    bias=p["bias"], act=p["act"], mask=None if p["mask_y"] is None else p["mask_y"][rm],
                    mask_act=p["mask_act"], prev=None if p["prev"] is None else p["prev"][rm])
    out = np.zeros_like(v)
    out[rm] = v
    return out


def _tiled_cpu32(p):
    case = p["case"]
    kw = dict(bias_row=True) if case["mode"] == 1 and case.get("bias_row") else {}
    P = p["contract"](p["A"], p["Bm"], **kw)
    M = p["M"]
    scaled = np.arange(M) < (M - 1 if kw else M)
    v = gr.epilogue(P, np.float32, div=p["div"] if p["na"] == 1 else 0.0, scaled=scaled, bias=p["bias"],
                    act=p["act"], mask=p["mask_m"], mask_act=p["mask_act"])
    rm = p["rowmap"] if p["rowmap"] is not None else np.arange(M)
    out = np.zeros_like(v)
    out[rm] = v
    return out


def _kinds(exact_u8):
    return ("u8",) if exact_u8 else gc.EXACT_KINDS


# ---- cb200_gemm -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", gc.GEMM_CASES, ids=[c["id"] for c in gc.GEMM_CASES])
def test_gemm(case):
    for kind in _kinds(case["kind"] in ("u8", "lut")):
        name = "%s/%s" % (case["id"], kind)
        p = gc.gemm_problem(case, kind, seed=1)
        r = run_gemm(p)
        assert r["dispatch"] == case["expect"], (name, r["dispatch"])
        check_exact(p, r["c"], name)
        again = run_gemm(p)
        assert np.array_equal(again["c"].view(np.uint32), r["c"].view(np.uint32)), "%s: not deterministic" % name
        if case.get("bplanes") is not None:
            fp32_b = run_gemm(p, b_planes=False)
            assert fp32_b["dispatch"] == r["dispatch"]
            assert np.array_equal(fp32_b["c"].view(np.uint32), r["c"].view(np.uint32)), \
                "%s: B planes and fp32 B differ" % name
        if r["planes"] is not None:
            npix = case["cplanes"]
            rm = p["rowmap"] if p["rowmap"] is not None else np.arange(p["Mout"])
            check_planes(p, r["c"], r["planes"], rm, npix, p["Mout"] // npix if npix else 0)
    for dist in gc.RANDOM_KINDS:
        p = gc.gemm_problem(case, dist, seed=2)
        r = run_gemm(p)
        check_accuracy(case["id"], p, r["c"], gc.gemm_gamma(case, r["dispatch"]), _gemm_cpu32(p), r["dispatch"])


def test_gemm_split_with_accumulate_adds_once():
    """splits > 1 with accumulate: the partial sums are reduced first, the pre-filled C is added once"""
    case = dict(id="tc_split_accumulate", M=128, R=2048, N=32, tr=0, kind="f32", layout="gather", splits=5,
                accumulate=1, bias=1)
    p = gc.gemm_problem(case, "b_bits", seed=3)
    r = run_gemm(p)
    assert r["dispatch"] == "tc<32,N,f32>+reduce_vec"
    check_exact(p, r["c"], case["id"])


# ---- cb200_gemm_tiled -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", gc.TILED_CASES, ids=[c["id"] for c in gc.TILED_CASES])
def test_gemm_tiled(case):
    from coach_b200.architectures import tiled as tl
    cat = case["mode"] == 0 and tl.b_interleaved(case["n"])
    for kind in _kinds(case.get("na", 3) == 1):
        name = "%s/%s" % (case["id"], kind)
        p = gc.tiled_problem(case, kind, seed=1)
        r = run_tiled(p)
        assert r["dispatch"] == case["expect"], (name, r["dispatch"])
        check_exact(p, r["c"], name)
        again = run_tiled(p)
        assert np.array_equal(again["c"].view(np.uint32), r["c"].view(np.uint32)), "%s: not deterministic" % name
        if cat:
            il = run_tiled(p, interleaved=True)
            kernel, _, rest = case["expect"].partition(">")
            assert il["dispatch"] == kernel + ",cat>" + rest, il["dispatch"]
            assert np.array_equal(il["c"].view(np.uint32), r["c"].view(np.uint32)), \
                "%s: interleaved and planar B planes differ" % name
        if case["mode"] == 1:
            bulk = run_tiled(p, a_pix_host=False)
            assert "/bulk" in bulk["dispatch"], bulk["dispatch"]
            assert np.array_equal(bulk["c"].view(np.uint32), r["c"].view(np.uint32)), \
                "%s: bulk copies and TMA boxes differ" % name
        if r["planes"] is not None:
            rm = p["rowmap"] if p["rowmap"] is not None else np.arange(p["M"])
            check_planes(p, r["c"], r["planes"], rm)
            if not p["mask_act"] or case.get("mask_planes"):
                only = run_tiled(p, c_null=True)
                assert np.array_equal(only["planes"], r["planes"]), "%s: planes-only call differs" % name
    for dist in gc.RANDOM_KINDS:
        p = gc.tiled_problem(case, dist, seed=2)
        r = run_tiled(p)
        check_accuracy(case["id"], p, r["c"], gc.tiled_gamma(case), _tiled_cpu32(p), r["dispatch"])


# ---- coverage -------------------------------------------------------------------------------------------------------
def _required():
    req = ["tc<%d,%s,%s>" % (w, t, k) for w in (32, 64) for t in "NT" for k in ("f32", "u8")] + ["tc<*,lut>"]
    req += ["tiled<%d,%s,%d>" % (w, t, na) for w in (32, 64, 128) for t in "NT" for na in (1, 3)]
    req += ["tiled<%d,N,%d,cat>" % (w, na) for w in (32, 64) for na in (1, 3)]
    req += ["/bulk", "/tma1", "/tma2", "/tma3"]
    req += ["fast<%s,%s>" % (c, t) for c in ("256,32", "128,64", "128,128") for t in "NT"]
    req += ["ffma<%s,%s>" % (c, t) for c in ("32,32", "128,32", "128,64") for t in "NT"]
    req += ["skinny_n", "skinny_r", "skinny_tn", "+reduce_wide", "+reduce_vec", "+reduce_scalar"]
    return req


def _hit(entry, seen):
    if entry.startswith("tc<*,"):
        return any(s.startswith("tc<") and (entry[5:] in s) for s in seen)
    if entry[0] in "/+":
        return any(entry in s for s in seen)
    return any(s == entry or s.startswith(entry + "/") or s.startswith(entry + "+") for s in seen)


def test_every_kernel_variant_was_run():
    """every kernel variant, A^T fetch mode and split reduction of the two GEMM entry points was dispatched by a case
    above (cases that did not run in this session are run now); a new variant must be added to this list and to the
    tables"""
    ran = set(DISPATCHED)
    if not all(_hit(e, ran) for e in _required()):
        for case in gc.GEMM_CASES:
            p = gc.gemm_problem(case, "u8" if case["kind"] in ("u8", "lut") else "normal", seed=2)
            run_gemm(p)
        for case in gc.TILED_CASES:
            p = gc.tiled_problem(case, "normal", seed=2)
            run_tiled(p)
            if case["mode"] == 0 and (case["n"] <= 64 or case["n"] % 128):
                run_tiled(p, interleaved=True)
            if case["mode"] == 1:
                run_tiled(p, a_pix_host=False)
    missing = [e for e in _required() if not _hit(e, DISPATCHED)]
    print("dispatched:", " ".join(sorted(DISPATCHED)))
    assert not missing, "kernel variants never run: %s" % missing
