"""CPU checks of the GEMM test helpers (tests/gemm_ref.py, tests/gemm_cases.py): the plane packing agrees with the
library's own reader, every exact probe the GPU suite draws keeps its exactness budget and exercises the planes it
claims, and the probes have the power to expose a kernel that drops one of the six 3xBF16 products or reads an 8x8
core the wrong way round."""
import numpy as np
import pytest
import torch

import gemm_cases as gc
import gemm_ref as gr


def _fp32_with_low_bits(rng, shape):
    return (rng.randn(*shape) * 2.0 ** rng.randint(-8, 8, size=shape)).astype(np.float32)


@pytest.mark.parametrize("interleaved", [False, True])
def test_packing_matches_planebuf(interleaved):
    from coach_b200.architectures import tiled as tl
    rng = np.random.RandomState(0)
    rows, cols = 40, 24
    x = _fp32_with_low_bits(rng, (rows, cols))
    buf = tl.PlaneBuf(rows, cols, "cpu", interleaved=interleaved)
    packed = gr.pack_planes_il(x) if interleaved else gr.pack_planes(x)
    buf.t.copy_(torch.from_numpy(packed.reshape(3, -1).view(np.int16)).view(torch.bfloat16))
    assert torch.equal(buf.to_dense(), torch.from_numpy(x))
    # the element formulas of the header, one element at a time
    r, c = 13, 17
    hi, mid, lo = gr.split3(x[r, c])
    flat = packed.reshape(-1)
    if interleaved:
        got = [flat[gr.tiled_elem_il(r, c, cols, p)] for p in range(3)]
    else:
        got = [flat[p * rows * cols + gr.tiled_elem(r, c, cols)] for p in range(3)]
    assert got == [hi, mid, lo]
    if not interleaved:
        assert np.array_equal(gr.unpack_planes(packed, rows, cols), np.stack(gr.split3(x)))


def test_split_is_exact_and_uses_all_planes():
    rng = np.random.RandomState(1)
    x = _fp32_with_low_bits(rng, (1000,))
    parts = [gr.bf16_value(p).astype(np.float64) for p in gr.split3(x)]
    assert np.array_equal(parts[0] + parts[1] + parts[2], x.astype(np.float64))
    assert (parts[2] != 0).mean() > 0.9


def _planes_nonzero(v):
    return [(gr.split3(np.asarray(v, np.float32))[k] & 0x7fff) != 0 for k in range(3)]


def _all_problems():
    for case in gc.GEMM_CASES:
        for kind in (("u8",) if case["kind"] in ("u8", "lut") else gc.EXACT_KINDS):
            p = gc.gemm_problem(case, kind, seed=1)
            a = gr.gather_a(p["a_src"], p["rowoff"], p["coloff"], p["rowinfo"], p["colinfo"], 4, 4,
                            p["lut"] if (p["lut"] is not None and not p["div"]) else None)
            yield case["id"], kind, p, a, p["b"].astype(np.float64)
    for case in gc.TILED_CASES:
        for kind in (("u8",) if case.get("na", 3) == 1 else gc.EXACT_KINDS):
            p = gc.tiled_problem(case, kind, seed=1)
            yield case["id"], kind, p, p["A"].astype(np.float64), p["Bm"].astype(np.float64)


def test_every_probe_meets_its_budget_and_uses_its_planes():
    n = 0
    for cid, kind, p, a, b in _all_problems():
        n += 1
        rows = p["exact_rows"]
        assert rows.sum() >= len(rows) - 1, (cid, kind)
        S = p["S"][rows] / p["unit"]
        assert S.max() < 2.0 ** 24, (cid, kind, np.log2(S.max()))
        # the products alone stay within 2^23 units (bias / pre-filled C take at most 2^21 more)
        dense, sparse = (a, b) if kind == "a_bits" else (b, a)
        if kind in ("a_bits", "b_bits", "u8"):
            nz = dense[dense != 0]
            lo = _planes_nonzero(nz)[2]
            assert lo.mean() >= 0.5, (cid, kind, lo.mean())
            if kind != "u8":
                assert set(np.unique(sparse)) <= {-1.0 / 4, 0.0, 1.0 / 4}, (cid, kind)
        else:
            for v in (a[a != 0], b[b != 0]):
                hi, mid, lo = _planes_nonzero(v)
                assert mid.all() and not lo.any(), (cid, kind)
    assert n > 60


PRODUCTS = [(0, 0), (0, 1), (1, 0), (1, 1), (0, 2), (2, 0)]        # (A plane, B plane) of the 3xBF16 product set


def _planes(x):
    return [gr.bf16_value(p).astype(np.float64) for p in gr.split3(np.asarray(x, np.float32))]


def _mutant(a, b, drop=None):
    pa, pb = _planes(a), _planes(b)
    return sum(pa[i] @ pb[j] for i, j in PRODUCTS if (i, j) != drop)


@pytest.mark.parametrize("drop", PRODUCTS, ids=["a%db%d" % (i + 1, j + 1) for i, j in PRODUCTS])
def test_probe_exposes_a_dropped_product(drop):
    """the kind that exercises the product: a1 b2 / a1 b3 -> b_bits, a2 b1 / a3 b1 -> a_bits, a2 b2 -> mid"""
    rng = np.random.RandomState(4)
    kind = {(0, 1): "b_bits", (0, 2): "b_bits", (1, 0): "a_bits", (2, 0): "a_bits", (1, 1): "mid"}.get(drop, "a_bits")
    A, B, ua, ub = gr.probe_operands(kind, (256, 1024), (1024, 64), lambda x, y: x @ y, rng)
    a, b = A * ua, B * ub
    exact = (a @ b).astype(np.float32)
    assert np.array_equal(_mutant(a, b).astype(np.float32), exact)         # the six products are exact
    differ = (_mutant(a, b, drop).astype(np.float32) != exact).mean()
    assert differ > 0.9, differ


@pytest.mark.parametrize("side", ["A", "B"])
def test_probe_exposes_a_transposed_core(side):
    rng = np.random.RandomState(5)
    for kind in gc.EXACT_KINDS:
        A, B, ua, ub = gr.probe_operands(kind, (128, 512), (512, 64), lambda x, y: x @ y, rng)
        a, b = A * ua, B * ub
        a2, b2 = (gr.transpose_cores(a), b) if side == "A" else (a, gr.transpose_cores(b))
        differ = ((a2 @ b2).astype(np.float32) != (a @ b).astype(np.float32)).mean()
        assert differ > 0.5, (kind, differ)


def test_u8_probe_is_exact_and_divides_once():
    rng = np.random.RandomState(6)
    A, B, ua, ub = gr.probe_operands("u8", (128, 1024), (1024, 32), lambda x, y: x @ y, rng)
    assert set(np.unique(A)) <= {0, 1, 2, 4} and (A @ np.abs(B * 1.0)).max() < 2 ** 23
    S = A @ B                                          # exact integers below 2^23
    for div in (1.0, 256.0, 255.0):
        want = gr.epilogue(S * ub, np.float32, div=div)
        assert np.array_equal(want, (S * ub).astype(np.float32) / np.float32(div))
    # dropping a b3 (the lo plane of B) changes most outputs
    pb = _planes(B * ub)
    assert ((A @ (pb[0] + pb[1])).astype(np.float32) != (S * ub).astype(np.float32)).mean() > 0.9


def test_tiled_references_agree_with_each_other():
    """mode 0 with one tap per pixel and mode 1 are the two halves of a dense layer on a flattened map:
    x @ w and x^T @ dy"""
    rng = np.random.RandomState(7)
    B, npix, C, N = 32, 3, 32, 64
    x, w, dy = rng.randn(B, npix * C), rng.randn(npix * C, N), rng.randn(B, N)
    A = x.reshape(B, npix, C).transpose(1, 0, 2).reshape(npix * B, C)
    ptr, lst = np.array([0, npix]), np.array([(q, q) for q in range(npix)])
    np.testing.assert_allclose(gr.tiled_mode0(ptr, lst, A, w, B, 1, N), x @ w, rtol=1e-12)
    dw = gr.tiled_mode1(np.arange(npix).reshape(npix, 1), A, dy, B, npix, 1, bias_row=True)
    np.testing.assert_allclose(dw[:-1], x.T @ dy, rtol=1e-12)
    np.testing.assert_allclose(dw[-1], dy.sum(0), rtol=1e-12)


def test_case_tables_are_consistent():
    ids = [c["id"] for c in gc.GEMM_CASES + gc.TILED_CASES]
    assert len(ids) == len(set(ids))
    for case in gc.TILED_CASES:
        s, cps = gc.tiled_slices(case)
        assert cps <= 32
    assert gc.tiled_slices(gc.TILED_CASES[0]) == (1, 32)            # the ABI maximum in one slice
    assert any(gc.gemm_slices(c) == (1, 1024) for c in gc.GEMM_CASES)
