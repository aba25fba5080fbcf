"""CPU checks of the host logic behind cb200_gemm_tiled: the tap lists, pixel tables, row maps and weight-block
orders that coach_b200/architectures/layers.py builds for the multi-tap tensor-core GEMMs are replayed here in numpy
(the contraction formulas of include/coach_b200.h) and compared with torch's convolution / its autograd on the CPU.
No kernel runs: descriptors are only built (prepare) and read back."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gemm_ref as gr
from coach_b200 import _lib
from coach_b200.architectures import tiled as tl
from coach_b200.architectures.layers import Conv2d, Dense, Workspace


def _tensor_at(op, ptr):
    for t in op.keep:
        if torch.is_tensor(t) and t.data_ptr() == ptr:
            return t
    raise KeyError(ptr)


def _mode0(op, A, W_blocks, B):
    """mode-0 contraction (gemm_ref.tiled_mode0) with the tap lists of a prepared call"""
    d = op.desc
    ptr = _tensor_at(op, d.list_ptr).numpy()
    lst = _tensor_at(op, d.list).numpy().reshape(-1, 2)
    out = gr.tiled_mode0(ptr, lst, A, W_blocks, B, d.num_q, d.n)
    if d.c_rowmap:
        rm = _tensor_at(op, d.c_rowmap).numpy()
        res = np.zeros_like(out)
        res[rm] = out
        return res
    return out


def _mode1(op, A, G, B):
    """mode-1 contraction (gemm_ref.tiled_mode1) with the pixel table of a prepared call"""
    d = op.desc
    out = gr.tiled_mode1(_tensor_at(op, d.a_pix).numpy(), A, G, B, d.taps, d.num_q)
    if d.c_rowmap:
        rm = _tensor_at(op, d.c_rowmap).numpy()
        res = np.zeros((int(rm.max()) + 1, d.n))
        res[rm[:out.shape[0]]] = out
        return res[:out.shape[0]] if res.shape[0] >= out.shape[0] else res
    return out


def _pm(t, B, npix, ch):
    """NHWC-flattened [B, npix*ch] -> plane-matrix order [npix*B, ch]"""
    return t.reshape(B, npix, ch).transpose(1, 0, 2).reshape(npix * B, ch)


def _ctx(B, npix_in, C, npix_out, N, dev, with_dx=True):
    wp = tl.PlaneBuf(8, 8, dev)
    return tl.PlaneCtx(x=tl.PlaneBuf(npix_in * B, C, dev, npix=npix_in), y=tl.PlaneBuf(npix_out * B, N, dev, npix=npix_out),
                       dy=tl.PlaneBuf(npix_out * B, N, dev, npix=npix_out),
                       dx=tl.PlaneBuf(npix_in * B, C, dev, npix=npix_in) if with_dx else None, w_ptr=wp.ptr,
                       w_stride=wp.stride), wp


@pytest.mark.parametrize("H,C,N,K,S", [(10, 32, 64, 4, 2), (7, 64, 32, 3, 1), (9, 32, 32, 3, 2)])
def test_conv_tap_lists_reproduce_convolution_and_its_gradients(H, C, N, K, S):
    lib, dev, B = _lib.load(), torch.device("cpu"), 32
    rng = np.random.RandomState(H)
    layer = Conv2d((H, H), C, N, K, S, None)
    OH = layer.OH
    x = rng.randn(B, H, H, C)
    w = rng.randn(K, K, C, N)
    dy = rng.randn(B, OH, OH, N)
    ctx, keep = _ctx(B, H * H, C, OH * OH, N, dev)
    flat = torch.zeros(K * K * C * N + N)
    y_t, dx_t = torch.zeros(B, OH * OH * N), torch.zeros(B, H * H * C)
    layer.prepare(lib, Workspace(dev), B, dev, torch.zeros(B, H * H * C), y_t, torch.zeros(K, K, C, N),
                  torch.zeros(N), flat[:K * K * C * N].view(K, K, C, N), flat[K * K * C * N:], torch.zeros_like(y_t),
                  dx_t, need_dx=True, prev_act=0, planes=ctx)
    assert layer.bwd_x is not None and layer.bwd_w.desc.bias_row == 1
    xt = torch.tensor(x).permute(0, 3, 1, 2).clone().requires_grad_(True)
    wt = torch.tensor(w).permute(3, 2, 0, 1).clone().requires_grad_(True)
    z = F.conv2d(xt, wt, stride=S)
    z.backward(torch.tensor(dy).permute(0, 3, 1, 2))
    A = _pm(x.reshape(B, -1), B, H * H, C)
    G = _pm(dy.reshape(B, -1), B, OH * OH, N)
    # forward: weight blocks = taps of the HWIO kernel, result rows mapped back to NHWC
    got_y = _mode0(layer.fwd, A, w.reshape(K * K, C, N), B).reshape(B, OH, OH, N)
    np.testing.assert_allclose(got_y, z.detach().permute(0, 2, 3, 1).numpy(), rtol=1e-9, atol=1e-9)
    # weight gradient
    got_dw = _mode1(layer.bwd_w, A, G, B).reshape(K, K, C, N)
    np.testing.assert_allclose(got_dw, wt.grad.permute(2, 3, 1, 0).numpy(), rtol=1e-9, atol=1e-9)
    # data gradient (gather form): weight blocks = per-tap transposed kernels as the permute table lays them out
    perm = layer.perm.numpy()
    wT = w.reshape(-1)[perm].reshape(K * K, N, C)
    got_dx = _mode0(layer.bwd_x, G, wT, B).reshape(B, H, H, C)
    np.testing.assert_allclose(got_dx, xt.grad.permute(0, 2, 3, 1).numpy(), rtol=1e-9, atol=1e-9)


def test_space_to_depth_first_layer_tables():
    """uint8 8x8/4 convolution as a 2x2/1 convolution over the space-to-depth(4) view: pixel table, permuted kernel
    rows and the row map of the weight gradient"""
    from coach_b200.architectures.network import make_u8_lut
    lib, dev, B = _lib.load(), torch.device("cpu"), 32
    H, C, N, K, S = 20, 4, 32, 8, 4
    rng = np.random.RandomState(1)
    layer = Conv2d((H, H), C, N, K, S, None)
    OH, Hs, Cs = layer.OH, H // S, S * S * C
    x = rng.randint(0, 256, (B, H, H, C)).astype(np.float64)
    w = rng.randn(K, K, C, N)
    dy = rng.randn(B, OH, OH, N)
    ctx, keep = _ctx(B, Hs * Hs, Cs, OH * OH, N, dev, with_dx=False)
    ctx.x = None
    flat = torch.zeros(K * K * C * N + N)
    y_t = torch.zeros(B, OH * OH * N)
    layer.prepare(lib, Workspace(dev), B, dev, torch.zeros(B, H, H, C, dtype=torch.uint8), y_t,
                  torch.zeros(K, K, C, N), torch.zeros(N), flat[:K * K * C * N].view(K, K, C, N),
                  flat[K * K * C * N:], torch.zeros_like(y_t), None, x_is_u8=True, lut=make_u8_lut(dev), need_dx=False,
                  planes=ctx)
    assert layer.s2d is not None and layer.fwd.desc.a_num_planes == 1 and layer.fwd.desc.a_u8_div == 255.0
    # the space-to-depth plane matrix exactly as cb200_u8_s2d_planes lays it out
    s2d = x.reshape(B, Hs, S, Hs, S, C).transpose(1, 3, 0, 2, 4, 5).reshape(Hs * Hs * B, Cs)
    w_s2d = w.reshape(-1)[layer.w_perm.numpy()].reshape(-1, Cs, N)
    xt = torch.tensor(x).permute(0, 3, 1, 2).clone()
    wt = torch.tensor(w).permute(3, 2, 0, 1).clone().requires_grad_(True)
    z = F.conv2d(xt, wt, stride=S)
    z.backward(torch.tensor(dy).permute(0, 3, 1, 2))
    got_y = _mode0(layer.fwd, s2d, w_s2d, B).reshape(B, OH, OH, N)
    np.testing.assert_allclose(got_y, z.detach().permute(0, 2, 3, 1).numpy(), rtol=1e-9, atol=1e-6)
    G = _pm(dy.reshape(B, -1), B, OH * OH, N)
    d = layer.bwd_w.desc
    rm = _tensor_at(layer.bwd_w, d.c_rowmap).numpy()
    assert rm[-1] == K * K * C                         # the bias row stays right behind the kernel gradient
    d.c_rowmap = None
    raw = _mode1(layer.bwd_w, s2d, G, B)               # rows (tap, (dy, dx, c)) ...
    got_dw = np.zeros((K * K * C, N))
    got_dw[rm[:-1]] = raw                              # ... scattered to the HWIO row order
    np.testing.assert_allclose(got_dw.reshape(K, K, C, N), wt.grad.permute(2, 3, 1, 0).numpy(), rtol=1e-9, atol=1e-6)


def test_dense_on_flattened_conv_map():
    """fc layer fed by a conv map: one tap per pixel forward / weight gradient, per-pixel transposed blocks backward"""
    lib, dev, B = _lib.load(), torch.device("cpu"), 32
    npix, C, N = 9, 64, 128
    K = npix * C
    rng = np.random.RandomState(2)
    x, w, dy = rng.randn(B, K), rng.randn(K, N), rng.randn(B, N)
    layer = Dense(K, N, None)
    ctx = tl.PlaneCtx(x=tl.PlaneBuf(npix * B, C, dev, npix=npix), y=tl.PlaneBuf(B, N, dev),
                      dy=tl.PlaneBuf(B, N, dev), dx=tl.PlaneBuf(npix * B, C, dev, npix=npix),
                      w_ptr=tl.PlaneBuf(8, 8, dev).ptr, w_stride=64)
    flat = torch.zeros(K * N + N)
    layer.prepare(lib, Workspace(dev), B, dev, torch.zeros(B, K), torch.zeros(B, N), torch.zeros(K, N), torch.zeros(N),
                  flat[:K * N].view(K, N), flat[K * N:], torch.zeros(B, N), torch.zeros(B, K), need_dx=True,
                  prev_act=0, planes=ctx)
    assert layer.tiled_x
    A = _pm(x, B, npix, C)
    np.testing.assert_allclose(_mode0(layer.fwd, A, w.reshape(npix, C, N), B), x @ w, rtol=1e-9, atol=1e-9)
    np.testing.assert_allclose(_mode1(layer.bwd_w, A, dy, B), x.T @ dy, rtol=1e-9, atol=1e-9)
    wT = w.reshape(-1)[layer.perm.numpy()].reshape(npix, N, C)
    # result rows (pixel, b) are mapped to the NHWC rows b * npix + pixel of the [B, npix * C] gradient
    np.testing.assert_allclose(_mode0(layer.bwd_x, dy, wT, B).reshape(B, K), dy @ w.T, rtol=1e-9, atol=1e-9)


def test_truncation_split_is_exact():
    """numpy restatement of csrc/nn_gemm.cuh split3 / nn_gemm_tc.cuh split8: hi = upper half-word of x, mid = upper
    half-word of the (exact) remainder, lo = upper half-word of the rest.  x == hi + mid + lo exactly whenever
    |x| >= 2^-110 (or x == 0); for smaller magnitudes `lo` is an fp32 denormal whose low half-word is cut, an absolute
    error below 2^-133"""
    rng = np.random.RandomState(0)
    bits = rng.randint(0, 2 ** 32, size=1 << 20, dtype=np.uint64).astype(np.uint32)
    special = np.array([0x00000000, 0x80000000, 0x00000001, 0x007fffff, 0x00800000, 0x7f7fffff, 0xff7fffff, 0x3f800000,
                        0x3f7fffff, 0x33800000], dtype=np.uint32)                  # zeros, denormals, extremes
    x = np.concatenate([bits, special]).view(np.float32)
    x = x[np.isfinite(x)]
    hi = (x.view(np.uint32) & np.uint32(0xffff0000)).view(np.float32)
    r1 = x - hi                                                                     # exact: at most 16 significant bits
    mid = (r1.view(np.uint32) & np.uint32(0xffff0000)).view(np.float32)
    lo = ((r1 - mid).view(np.uint32) & np.uint32(0xffff0000)).view(np.float32)      # what the kernels store
    rebuilt = (hi.astype(np.float64) + mid.astype(np.float64)) + lo.astype(np.float64)
    normal = (np.abs(x) >= 2.0 ** -110) | (x == 0)
    assert normal.sum() > 900000
    assert np.array_equal(rebuilt[normal], x[normal].astype(np.float64))
    assert np.array_equal(((hi + mid) + lo)[normal], x[normal])                     # also in fp32 arithmetic
    assert np.all(np.abs(rebuilt[~normal] - x[~normal].astype(np.float64)) < 2.0 ** -133)


def test_theta_planes_cover_the_tensor_core_layers_of_the_atari_network():
    """parameter planes: every kernel whose [rows, cols] form is a multiple of 8 both ways gets a segment at its own
    (8-aligned) offset of the flat buffer; the skinny Q head (512 x 6) stays fp32 only"""
    from coach_b200.architectures.q_network import QNetworkDef
    lib = _lib.load()
    net = QNetworkDef("cpu", (84, 84, 4), 6)
    tp = tl.ThetaPlanes(lib, net.store, net.store.theta)
    segs = {int(o): (int(r), int(c)) for o, r, c, _, _ in tp.segs.tolist()}
    shapes = sorted(segs.values())
    assert shapes == sorted([(256, 32), (512, 64), (576, 64), (3136, 512)])
    # narrow kernels (tile width <= 64) are row-group interleaved -- the second half of the plane buffer, 3 x their
    # offset -- and wide ones planar at their own offset; the regions are disjoint
    regions = []
    for o, r, c, po, il in tp.segs.tolist():
        assert bool(il) == tl.b_interleaved(int(c))
        if il:
            assert po == 3 * net.store.size + 3 * o
            regions.append((po, po + 3 * r * c))
        else:
            assert po == o
            regions += [(k * net.store.size + o, k * net.store.size + o + r * c) for k in range(3)]
    regions.sort()
    assert all(a[1] <= b[0] for a, b in zip(regions, regions[1:])) and regions[-1][1] <= tp.buf.numel()
    for name, (off, shape) in net.store.entries.items():
        assert off % 8 == 0, name
        if name.endswith("kernel"):
            assert tp.has(name) == (int(np.prod(shape[:-1])) % 8 == 0 and shape[-1] % 8 == 0), name
    head = [n for n in net.store.entries if n.endswith("kernel")][-1]
    assert not tp.has(head) and net.store.entries[head][1] == (512, 6)
    assert tp.stride == net.store.size and tp.max_elems == 3136 * 512


@pytest.mark.parametrize("tiles,total", [(324, 16), (196, 18), (16, 98), (4, 1296), (5, 784), (100, 16), (1600, 8)])
def test_split_choice_respects_the_accumulation_cap(tiles, total):
    """at most TILED_MAX_CHUNKS reduction chunks (40 accumulating MMAs) per launch slice, whatever the tile count"""
    s = tl.pick_splits_tiled(tiles, total)
    cps = -(-total // s)
    assert 1 <= s <= max(1, total) and cps <= tl.TILED_MAX_CHUNKS
