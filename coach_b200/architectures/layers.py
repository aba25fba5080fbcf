"""Layers of the learn-step networks as prepared gather-GEMM calls (include/coach_b200.h: cb200_gemm).

Mirrors the layer vocabulary of ``rl_coach/architectures/tensorflow_components/layers.py:108-183`` (Conv2d, Dense) and
the embedders' input rescale (``embedders/embedder.py:103-104``).  Data layout is TensorFlow's: activations NHWC,
conv kernels HWIO (= a row-major [KH*KW*Cin, N] matrix), dense kernels [in, out]; VALID padding
(``tf.layers.conv2d`` default).

Two execution forms, chosen per layer when it is prepared.  With operand planes (``planes=tiled.PlaneCtx``, batch a
multiple of 32, channel counts the tensor-core kernel supports) forward, weight gradient and data gradient are
multi-tap wgmma GEMMs on pre-split bf16 operands (``architectures/tiled.py``, cb200_gemm_tiled); the uint8 first
convolution runs on the space-to-depth view of the frames (``_prepare_s2d``).  Otherwise -- small batches, odd shapes,
the skinny Q head -- the gather-GEMM below.

Gather-GEMM: every contraction is ONE C-ABI call whose descriptor -- index tables included -- is built once per (layer,
batch size) and reused every step: forward, weight gradient (A^T * dZ with a fixed-order split reduction over the batch*pixels
axis; the bias gradient rides along as one extra output row when the bias gradient sits right behind the kernel
gradient in the flat buffer), data gradient (dense: dZ * W^T; conv: transposed convolution in gather form, one call
per stride-parity class, with the previous layer's activation derivative fused into the epilogue).
"""
import ctypes

import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.architectures import tiled as tl

ACT = {None: 0, "none": 0, "relu": 1, "tanh": 2}


def _dev_i32(a, device):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)


class Workspace(object):
    """One scratch buffer shared by all ops of a network (split-reduction partials, column sums)."""

    def __init__(self, device):
        self.device = device
        self.buf = torch.empty(1 << 20, dtype=torch.float32, device=device)
        self._side = None

    def side(self):
        """a second scratch buffer for the ops that may run on a side stream concurrently with the others of the
        network (the weight-gradient GEMMs and bias column sums, see SideStream)"""
        if self._side is None:
            self._side = Workspace(self.device)
        return self._side

    def require(self, nfloats):
        if self.buf.numel() < nfloats:
            self.buf = torch.empty(int(nfloats), dtype=torch.float32, device=self.device)

    def ptr(self):
        return self.buf.data_ptr()


class SideStream(object):
    """Fork / join of a second CUDA stream around a group of launches that only READ what the main stream has produced
    so far and whose results are needed later: the launches inside ``with side:`` go to the side stream (ordered after
    everything queued on the main stream at that point), ``side.join()`` makes the main stream wait for them.  Works
    eagerly and under CUDA-graph capture (the captured graph gets parallel branches).  The tiled GEMMs of one network
    leave SMs idle at their wave tails and during prologue / epilogue; two independent chains fill them."""

    def __init__(self, device):
        self.stream = torch.cuda.Stream(device=device)
        self._ctx, self._dirty = None, False

    def after(self, event):
        """the next ``with`` block is ordered after ``event`` instead of after everything queued on the current stream"""
        self._after = event
        return self

    def __enter__(self):
        ev = getattr(self, "_after", None)
        self._after = None
        if ev is None:
            ev = torch.cuda.Event()
            ev.record()
        self.stream.wait_event(ev)
        self._ctx = torch.cuda.stream(self.stream)
        self._ctx.__enter__()
        self._dirty = True
        return self

    def __exit__(self, *exc):
        self._ctx.__exit__(*exc)
        self._ctx = None

    def join(self):
        if self._dirty:
            ev = torch.cuda.Event()
            ev.record(self.stream)
            torch.cuda.current_stream().wait_event(ev)
            self._dirty = False


class _NoSide(object):
    def __enter__(self):
        return self

    def __exit__(self, *exc):
        return False

    def join(self):
        pass


NO_SIDE = _NoSide()


def _derive(layer, w):
    """a prepared layer is ready to run: its weight-derived operands are derived from the weights as they are now
    (layer.run_perms; after a later write of the weights ThetaPlanes.refresh runs it again).  Host-side tests prepare
    layers over CPU tensors only to inspect their tables: nothing is launched for them."""
    if w.is_cuda:
        layer.run_perms()


def _u8_div(lut, x_is_u8):
    return float(getattr(lut, "u8_div", 0.0)) if (x_is_u8 and lut is not None) else 0.0


class GemmOp(object):
    """A prepared cb200_gemm call.  Tensors referenced by the descriptor are kept alive here."""

    def __init__(self, lib, ws, **fields):
        self.lib = lib
        self.ws = ws
        self.keep = []
        self.desc = _lib.GemmDesc()
        self.splits = int(fields.pop("splits", 1))
        for k, v in fields.items():
            if torch.is_tensor(v):
                self.keep.append(v)
                v = v.data_ptr()
            setattr(self.desc, k, v)
        self.desc.splits = self.splits
        rows = self.desc.a_cols if self.desc.a_transposed else self.desc.a_rows
        if self.desc.a_ones_col:
            rows += 1
        if self.splits > 1:
            ws.require(self.splits * rows * self.desc.n)

    def run(self):
        if self.splits > 1:
            self.desc.workspace = self.ws.ptr()
        _lib.check(self.lib.cb200_gemm(ctypes.byref(self.desc), _lib.current_stream()))


def pick_splits(tiles, reduction, sm=132, min_chunk=128):
    """Split the reduction so that the grid has about two CTAs per SM, never below `min_chunk` per split."""
    # the tensor-core path never reduces more than TC_MAX_R terms in one launch (the error of its fp32 accumulation
    # grows with the accumulation count); the partial sums are then added in fp32 round-to-nearest by the
    # split-reduce kernel (csrc/nn_gemm_tc.cuh)
    need = (reduction + TC_MAX_R - 1) // TC_MAX_R
    if tiles >= sm:          # one full wave already: the extra reduction pass would cost more than it saves
        return int(max(1, need))
    s = max(1, (2 * sm + tiles - 1) // tiles)
    s = min(s, max(1, reduction // min_chunk))
    return int(max(s, need))


TC_MAX_R = 1024


def _tiles(M, N, fast=True):
    """CTA tiles of the kernel cb200_gemm will pick (csrc/nn.cu)."""
    if M <= 64:
        return ((M + 31) // 32) * ((N + 31) // 32)
    if fast and N % 4 == 0:
        if N % 16 == 0:
            # tensor-core kernel (nn_gemm_tc.cuh): 128 x 32 or 128 x 64 tiles -- one warpgroup holds the accumulators
            bn = 32 if N <= 32 else 64
            return ((M + 127) // 128) * ((N + bn - 1) // bn)
        if N <= 32:
            return ((M + 255) // 256) * ((N + 31) // 32)
        if N <= 64:
            return ((M + 127) // 128) * ((N + 63) // 64)
        return ((M + 127) // 128) * ((N + 127) // 128)
    bn = 32 if N <= 32 else 64
    return ((M + 127) // 128) * ((N + bn - 1) // bn)


def _bias_behind(dw, db, K, N):
    """the bias gradient is stored right behind the kernel gradient (flat ParamStore layout): one more GEMM row"""
    return dw is not None and db is not None and db.data_ptr() == dw.data_ptr() + K * N * 4


def _bias_rides_along(dw, db, K, N, skinny=False):
    """True when the bias gradient is stored right behind the kernel gradient (flat ParamStore layout)."""
    bm = 256 if N <= 32 else 128          # row tile of the kernel that will run; only use slack of the last tile
    if dw is None or db is None or db.data_ptr() != dw.data_ptr() + K * N * 4:
        return False
    if N <= 8 and skinny:                 # skinny weight-gradient kernel: the extra row is a block of its own
        return True
    return N % 4 == 0 and K % 4 == 0 and K + 1 > 64 and K % bm != 0


# =====================================================================================================================
class Dense(object):
    """y = act(x W + b), W [K, N] (layers.py:148-183)."""

    def __init__(self, in_features, out_features, activation=None):
        self.K, self.N = int(in_features), int(out_features)
        self.act = ACT[activation]
        self.param_shapes = [("kernel", (self.K, self.N)), ("bias", (self.N,))]
        self.in_shape = (self.K,)
        self.out_shape = (self.N,)

    def out_elems(self):
        return self.N

    def out_pixels(self):
        return 1

    def prepare(self, lib, ws, B, device, x, y, w, b, dw, db, dy, dx, x_is_u8=False, lut=None, need_dx=True,
                prev_act=0, dx_accumulate=False, planes=None):
        """x [B,K], y [B,N], dy [B,N] (gradient wrt the PRE-activation of this layer), dx [B,K] (gradient wrt the
        pre-activation of the previous layer: masked with prev_act' evaluated on x).  planes: tiled.PlaneCtx or None."""
        K, N = self.K, self.N
        self.lib, self.ws, self.w = lib, ws, w
        self.tiled_x = False
        self.db_args = None
        pl = planes
        if (pl is not None and pl.x is not None and not x_is_u8 and not dx_accumulate and B % 32 == 0 and pl.w_ptr and
                tl.width_ok(N) and tl.channels_ok(pl.x.cols) and pl.x.npix * pl.x.cols == K):
            self._prepare_tiled(lib, ws, B, device, x, y, w, b, dw, db, dy, dx, need_dx, prev_act, pl)
            return
        # operands without planes (uint8 / small / odd shapes): the register-staged paths of cb200_gemm; results
        # that feed plane consumers still get their planes written by the epilogue
        yp = dict(c_planes=pl.y.ptr, c_plane_stride=pl.y.stride, c_plane_cols=N) \
            if (pl is not None and pl.y is not None) else {}
        dxp = dict(c_planes=pl.dx.ptr, c_plane_stride=pl.dx.stride, c_plane_cols=K) \
            if (pl is not None and pl.dx is not None and pl.dx.npix == 1) else {}
        if need_dx and pl is not None and pl.dx is not None and pl.dx.npix != 1:
            # the producer of this gradient would have to write pixel-major planes of a flattened conv map, which only
            # the tiled data-gradient GEMM does: fail instead of leaving the consumer's planes stale
            raise NotImplementedError("Dense(%d -> %d) on a %d-pixel conv map has no tensor-core form (n must be 32 or a "
                                      "multiple of 64): its data gradient cannot feed the conv layer's operand planes"
                                      % (K, N, pl.dx.npix))
        rowoff = _dev_i32(np.arange(B) * K, device)
        coloff = _dev_i32(np.arange(K), device)
        vec = int(K % 4 == 0)
        common = dict(a_rowoff=rowoff, a_coloff=coloff, a_rows=B, a_cols=K, a_vec4=vec, a_src=x,
                      a_lut=lut if x_is_u8 else None, a_u8_div=_u8_div(lut, x_is_u8), a_lda=0 if x_is_u8 else K)
        self.fwd = GemmOp(lib, ws, a_transposed=0, b=w, ldb=N, n=N, c=y, ldc=N, bias=b, act=self.act,
                          splits=pick_splits(_tiles(B, N, vec), K), **common, **yp)
        self.bwd_w = None
        if dw is not None and dy is not None:
            ones = int(bool(vec) and _bias_rides_along(dw, db, K, N, skinny=not x_is_u8))
            self.bwd_w = GemmOp(lib, ws.side(), a_transposed=1, b=dy, ldb=N, n=N, c=dw, ldc=N, a_ones_col=ones,
                                splits=pick_splits(_tiles(K + ones, N, vec), B), **common)
            if not ones:
                self.db_args = (dy, B, N, db)
                ws.require(1024 * N)
        self.bwd_x = None
        if need_dx:
            self.wT = torch.empty((N, K), dtype=torch.float32, device=device)
            self.w = w
            ro = _dev_i32(np.arange(B) * N, device)
            co = _dev_i32(np.arange(N), device)
            self.bwd_x = GemmOp(lib, ws, a_src=dy, a_rowoff=ro, a_coloff=co, a_rows=B, a_cols=N, a_transposed=0,
                                a_vec4=int(N % 4 == 0), a_lda=N, b=self.wT, ldb=K, n=K, c=dx, ldc=K,
                                mask_y=x if prev_act else None, mask_act=prev_act,
                                accumulate=int(bool(dx_accumulate)),
                                splits=pick_splits(_tiles(B, K, N % 4 == 0), N), **dxp)

    def _prepare_tiled(self, lib, ws, B, device, x, y, w, b, dw, db, dy, dx, need_dx, prev_act, pl):
        """input available as planes [npix * B, Ca] (npix > 1: a flattened conv map, one tap per pixel)"""
        K, N = self.K, self.N
        xp = pl.x
        npix, Ca = xp.npix, xp.cols
        self.tiled_x = True
        self.fwd = tl.forward_op(lib, ws, B, device, xp, Ca, pl.w_ptr, pl.w_stride, N,
                                 [[(p, p) for p in range(npix)]], 1, y, N, b, self.act, None, pl.y)
        self.bwd_w = None
        if dw is not None and dy is not None:
            if pl.dy is not None:
                fused = _bias_behind(dw, db, K, N)        # bias gradient as one more row of the same GEMM
                self.bwd_w = tl.wgrad_op(lib, ws.side(), B, device, xp, Ca, pl.dy, N, np.arange(npix), npix, 1, dw,
                                         bias_row=int(fused))
                if not fused:
                    self.db_args = (dy, B, N, db)
                    ws.require(1024 * N)
            else:       # the gradient of this layer's output has no planes (written by a head kernel)
                vec = int(K % 4 == 0)
                ones = int(bool(vec) and _bias_rides_along(dw, db, K, N))
                self.bwd_w = GemmOp(lib, ws.side(), a_transposed=1, b=dy, ldb=N, n=N, c=dw, ldc=N, a_ones_col=ones,
                                    splits=pick_splits(_tiles(K + ones, N, vec), B),
                                    a_rowoff=_dev_i32(np.arange(B) * K, device), a_coloff=_dev_i32(np.arange(K), device),
                                    a_rows=B, a_cols=K, a_vec4=vec, a_src=x)
                if not ones:
                    self.db_args = (dy, B, N, db)
                    ws.require(1024 * N)
        self.bwd_x = None
        self.perm = None
        if need_dx:
            assert pl.dy is not None and tl.channels_ok(N) and tl.width_ok(Ca), "tiled data gradient: unsupported shape"
            # per-pixel transposed kernels: wT[p][n, c] = W[p * Ca + c, n]
            w_index = np.arange(K * N).reshape(npix, Ca, N)
            self.perm = _dev_i32(w_index.transpose(0, 2, 1).reshape(-1), device)
            self.wT = torch.empty(npix * N * Ca, dtype=torch.float32, device=device)
            self.wT_planes = tl.PlaneBuf(npix * N, Ca, device, interleaved=tl.b_interleaved(Ca))
            rowmap = None
            if npix > 1:
                qq, bb = np.meshgrid(np.arange(npix), np.arange(B), indexing="ij")
                rowmap = _dev_i32((bb * npix + qq).reshape(-1), device)
            self.bwd_x = tl.masked_forward_op(lib, ws, B, device, pl.dy, N, self.wT_planes, Ca,
                                              [[(0, q)] for q in range(npix)], npix, dx, Ca,
                                              x if prev_act else None, prev_act, rowmap, pl.dx, mask_planes=pl.x)
        _derive(self, w)

    def forward(self):
        self.fwd.run()

    def run_perms(self):
        """weight-derived operands of this layer: the per-pixel transposed kernels of the data-gradient GEMM (run when
        the layer is prepared and by ThetaPlanes.refresh after every write of the weights)"""
        if self.tiled_x and getattr(self, "perm", None) is not None:
            _lib.check(self.lib.cb200_permute_f32(self.w.data_ptr(), self.perm.data_ptr(), self.perm.numel(),
                                                  self.wT.data_ptr(), self.wT_planes.ptr, self.wT_planes.stride,
                                                  self.wT_planes.cols, _lib.current_stream()))

    def backward(self, weights=True, side=NO_SIDE):
        if weights:
            with side:        # weight / bias gradients only read dy and x: off the data-gradient chain
                self.bwd_w.run()
                if self.db_args is not None:
                    dy, B, N, db = self.db_args
                    _lib.check(self.lib.cb200_colsum(dy.data_ptr(), B, N, db.data_ptr(), self.ws.side().ptr(),
                                                     _lib.current_stream()))
        if self.bwd_x is not None:
            if not self.tiled_x:          # (the tiled form's transposed kernels are derived by run_perms)
                _lib.check(self.lib.cb200_transpose(self.w.data_ptr(), self.K, self.N, self.wT.data_ptr(), None, 0,
                                                    _lib.current_stream()))
            self.bwd_x.run()


# =====================================================================================================================
class Conv2d(object):
    """NHWC VALID convolution + bias + activation (layers.py:108-146: tf.layers.conv2d(filters, kernel, strides))."""

    def __init__(self, in_hw, in_channels, num_filters, kernel_size, strides, activation="relu"):
        self.H, self.W = int(in_hw[0]), int(in_hw[1])
        self.C, self.N = int(in_channels), int(num_filters)
        self.KH = self.KW = int(kernel_size)
        self.S = int(strides)
        self.OH = (self.H - self.KH) // self.S + 1
        self.OW = (self.W - self.KW) // self.S + 1
        self.K = self.KH * self.KW * self.C
        self.act = ACT[activation]
        self.param_shapes = [("kernel", (self.KH, self.KW, self.C, self.N)), ("bias", (self.N,))]
        self.in_shape = (self.H, self.W, self.C)
        self.out_shape = (self.OH, self.OW, self.N)

    def out_elems(self):
        return self.OH * self.OW * self.N

    def out_pixels(self):
        return self.OH * self.OW

    def prepare(self, lib, ws, B, device, x, y, w, b, dw, db, dy, dx, x_is_u8=False, lut=None, need_dx=True,
                prev_act=0, dx_accumulate=False, planes=None):
        assert not dx_accumulate, "accumulating data gradients is only wired for Dense layers"
        H, W, C, N, KH, KW, S, OH, OW, K = self.H, self.W, self.C, self.N, self.KH, self.KW, self.S, self.OH, \
            self.OW, self.K
        M = B * OH * OW
        self.lib, self.ws, self.w = lib, ws, w
        self.classes = []
        self.bwd_x = None
        self.db_args = None
        self.s2d = None
        pl = planes
        if (pl is not None and pl.x is not None and not x_is_u8 and B % 32 == 0 and pl.w_ptr and tl.width_ok(N) and
                tl.channels_ok(C) and pl.x.cols == C and pl.x.npix == H * W):
            self._prepare_tiled(lib, ws, B, device, x, y, w, b, dw, db, dy, dx, need_dx, prev_act, pl)
            return
        div = _u8_div(lut, x_is_u8)
        if isinstance(x, tl.PlaneBuf):
            assert (pl is not None and x_is_u8 and div > 0 and B % 32 == 0 and pl.y is not None and not need_dx), \
                "a space-to-depth input plane needs the tensor-core form of the layer"
        if (pl is not None and x_is_u8 and div > 0 and B % 32 == 0 and pl.y is not None and KH % S == 0 and
                KW % S == 0 and H % S == 0 and W % S == 0 and tl.channels_ok(S * S * C) and tl.width_ok(N) and
                not need_dx and _lib.tune_default("conv_s2d", 1)):
            self._prepare_s2d(lib, ws, B, device, x, y, w, b, dw, db, dy, pl, div)
            return
        # no input planes (the uint8 frames of the first layer): register-staged cb200_gemm; the output planes are
        # written by its epilogue (plane row = pixel * B + b), the weight gradient reads dY's planes as its B operand
        yp = dict(c_planes=pl.y.ptr, c_plane_stride=pl.y.stride, c_plane_cols=N, c_prow_npix=OH * OW,
                  c_prow_batch=B) if (pl is not None and pl.y is not None) else {}
        gp = dict(b_planes=pl.dy.ptr, b_plane_stride=pl.dy.stride, b_prow_npix=OH * OW, b_prow_batch=B) \
            if (pl is not None and pl.dy is not None) else {}
        wp = dict(b_planes=pl.w_ptr, b_plane_stride=pl.w_stride) \
            if (pl is not None and pl.w_ptr and K % 8 == 0 and pl.w_stride > 0) else {}
        bb, oy, ox = np.meshgrid(np.arange(B), np.arange(OH), np.arange(OW), indexing="ij")
        rowoff = (((bb * H + oy * S) * W + ox * S) * C).reshape(-1)
        ky, kx, cc = np.meshgrid(np.arange(KH), np.arange(KW), np.arange(C), indexing="ij")
        coloff = ((ky * W + kx) * C + cc).reshape(-1)
        assert rowoff.max() + coloff.max() < 2 ** 31
        vec = int(C % 4 == 0)          # (kx, c) runs are contiguous: groups of 4 channels never straddle a pixel
        common = dict(a_rowoff=_dev_i32(rowoff, device), a_coloff=_dev_i32(coloff, device), a_rows=M, a_cols=K,
                      a_src=x, a_lut=lut if x_is_u8 else None, a_vec4=vec, a_u8_div=_u8_div(lut, x_is_u8))
        self.fwd = GemmOp(lib, ws, a_transposed=0, b=w, ldb=N, n=N, c=y, ldc=N, bias=b, act=self.act,
                          splits=pick_splits(_tiles(M, N, vec), K), **common, **yp, **wp)
        self.bwd_w = None
        if dw is not None and dy is not None:
            ones = int(bool(vec) and _bias_rides_along(dw, db, K, N))
            self.bwd_w = GemmOp(lib, ws.side(), a_transposed=1, b=dy, ldb=N, n=N, c=dw, ldc=N, a_ones_col=ones,
                                splits=pick_splits(_tiles(K + ones, N, vec), M, min_chunk=512), **common, **gp)
            if not ones:
                self.db_args = (dy, M, N, db)
                ws.require(1024 * N)
        if not need_dx:
            return
        # transposed convolution, gather form, one GEMM per stride-parity class of input pixels
        w_index = np.arange(KH * KW * C * N).reshape(KH, KW, C, N)
        for py in range(S):
            for px in range(S):
                IH = (H - py + S - 1) // S
                IW = (W - px + S - 1) // S
                TA = (KH - py + S - 1) // S
                TB = (KW - px + S - 1) // S
                if IH <= 0 or IW <= 0 or TA <= 0 or TB <= 0:
                    continue
                b_, i_, j_ = np.meshgrid(np.arange(B), np.arange(IH), np.arange(IW), indexing="ij")
                ro = (((b_ * OH + i_) * OW + j_) * N).reshape(-1)
                rinfo = ((i_ << 16) | j_).reshape(-1)
                rowmap = ((b_ * H + (S * i_ + py)) * W + (S * j_ + px)).reshape(-1)
                a_, t_, n_ = np.meshgrid(np.arange(TA), np.arange(TB), np.arange(N), indexing="ij")
                co = (-(a_ * OW + t_) * N + n_).reshape(-1)
                cinfo = ((a_ << 16) | t_).reshape(-1)
                # B_class[(a, t, n), c] = W[S*a + py, S*t + px, c, n]
                perm = w_index[S * a_ + py, S * t_ + px, :, n_]          # [TA, TB, N, C]
                perm = perm.reshape(-1)
                wt = torch.empty((TA * TB * N, C), dtype=torch.float32, device=device)
                op = GemmOp(lib, ws, a_src=dy, a_rowoff=_dev_i32(ro, device), a_coloff=_dev_i32(co, device),
                            a_rowinfo=_dev_i32(rinfo, device), a_colinfo=_dev_i32(cinfo, device), a_oh=OH, a_ow=OW,
                            a_rows=B * IH * IW, a_cols=TA * TB * N, a_transposed=0, a_vec4=int(N % 4 == 0),
                            b=wt, ldb=C, n=C, c=dx, ldc=C,
                            mask_y=x if prev_act else None, mask_act=prev_act, c_rowmap=_dev_i32(rowmap, device),
                            splits=pick_splits(_tiles(B * IH * IW, C, N % 4 == 0), TA * TB * N))
                self.classes.append((op, wt, _dev_i32(perm, device)))

    def _prepare_s2d(self, lib, ws, B, device, x, y, w, b, dw, db, dy, pl, div):
        """uint8 frames, kernel size a multiple of the stride: the space-to-depth(S) view of the input (one exact
        bf16 plane, cb200_u8_s2d_planes) turns the layer into a (K/S) x (K/S) stride-1 convolution over S*S*C
        channels -- a multi-tap tensor-core GEMM like every other layer, with 3 products instead of 6."""
        H, W, C, N, KH, KW, S, OH, OW = self.H, self.W, self.C, self.N, self.KH, self.KW, self.S, self.OH, self.OW
        Hs, Ws, Cs, TH, TW = H // S, W // S, S * S * C, KH // S, KW // S
        T, nq = TH * TW, OH * OW
        if isinstance(x, tl.PlaneBuf):
            # the replay's fused gather already delivered the space-to-depth plane (cb200_per_sample_gather_s2d)
            assert x.nplanes == 1 and x.rows == Hs * Ws * B and x.cols == Cs, "s2d plane geometry"
            self.s2d = (None, x, B)
        else:
            self.s2d = (x, tl.PlaneBuf(Hs * Ws * B, Cs, device, npix=Hs * Ws, nplanes=1), B)
        # rows of the s2d kernel matrix: (tap (ty, tx), (dy, dx, c)) <- original row (ky, kx, c) = (S ty + dy, ...)
        ty, tx, dy_, dx_, cc = np.meshgrid(np.arange(TH), np.arange(TW), np.arange(S), np.arange(S), np.arange(C),
                                           indexing="ij")
        orig_row = (((S * ty + dy_) * KW + (S * tx + dx_)) * C + cc).reshape(-1)            # [T * Cs]
        self.w_s2d = torch.empty(T * Cs * N, dtype=torch.float32, device=device)
        self.w_s2d_planes = tl.PlaneBuf(T * Cs, N, device, interleaved=tl.b_interleaved(N))
        self.w_perm = _dev_i32((orig_row[:, None] * N + np.arange(N)[None, :]).reshape(-1), device)
        pix_in = np.zeros((T, nq), dtype=np.int64)
        for t in range(T):
            oy, ox = np.meshgrid(np.arange(OH), np.arange(OW), indexing="ij")
            pix_in[t] = ((oy + t // TW) * Ws + (ox + t % TW)).reshape(-1)
        qq, bb = np.meshgrid(np.arange(nq), np.arange(B), indexing="ij")
        rowmap_out = _dev_i32((bb * nq + qq).reshape(-1), device)
        xp = self.s2d[1]
        self.fwd = tl.forward_op(lib, ws, B, device, xp, Cs, self.w_s2d_planes.ptr, self.w_s2d_planes.stride, N,
                                 [[(int(pix_in[t, q]), t) for t in range(T)] for q in range(nq)], nq, y, N, b,
                                 self.act, rowmap_out, pl.y, w_rows=T * Cs, a_u8_div=div)
        self.fwd.keep.append(self.w_s2d_planes)
        self.bwd_w = None
        if dw is not None and dy is not None:
            assert pl.dy is not None, "s2d conv weight gradient needs the planes of dY"
            fused = _bias_behind(dw, db, T * Cs, N)
            self.bwd_w = tl.wgrad_op(lib, ws.side(), B, device, xp, Cs, pl.dy, N, pix_in, T, nq, dw, a_u8_div=div,
                                     c_rowmap=_dev_i32(np.concatenate([orig_row, [T * Cs]]), device),
                                     bias_row=int(fused))
            if not fused:
                self.db_args = (dy, B * nq, N, db)
                ws.require(1024 * N)
        _derive(self, w)

    def _prepare_tiled(self, lib, ws, B, device, x, y, w, b, dw, db, dy, dx, need_dx, prev_act, pl):
        """input available as planes [H * W * B, C]: forward, weight gradient and data gradient as multi-tap GEMMs"""
        H, W, C, N, KH, KW, S, OH, OW = self.H, self.W, self.C, self.N, self.KH, self.KW, self.S, self.OH, self.OW
        T, nq = KH * KW, OH * OW
        taps = [(ky, kx) for ky in range(KH) for kx in range(KW)]
        pix_in = np.zeros((T, nq), dtype=np.int64)                  # input pixel under tap t at output pixel q
        for t, (ky, kx) in enumerate(taps):
            oy, ox = np.meshgrid(np.arange(OH), np.arange(OW), indexing="ij")
            pix_in[t] = ((oy * S + ky) * W + (ox * S + kx)).reshape(-1)
        qq, bb = np.meshgrid(np.arange(nq), np.arange(B), indexing="ij")
        rowmap_out = _dev_i32((bb * nq + qq).reshape(-1), device)   # plane row q * B + b -> NHWC row b * nq + q
        self.fwd = tl.forward_op(lib, ws, B, device, pl.x, C, pl.w_ptr, pl.w_stride, N,
                                 [[(int(pix_in[t, q]), t) for t in range(T)] for q in range(nq)], nq, y, N, b,
                                 self.act, rowmap_out, pl.y)
        self.bwd_w = None
        if dw is not None and dy is not None:
            assert pl.dy is not None, "tiled conv weight gradient needs the planes of dY"
            fused = _bias_behind(dw, db, T * C, N)
            self.bwd_w = tl.wgrad_op(lib, ws.side(), B, device, pl.x, C, pl.dy, N, pix_in, T, nq, dw, bias_row=int(fused))
            if not fused:
                self.db_args = (dy, B * nq, N, db)
                ws.require(1024 * N)
        if not need_dx:
            return
        assert pl.dy is not None and tl.channels_ok(N) and tl.width_ok(C), "tiled data gradient: unsupported shape"
        # gather form over INPUT pixels: only the taps whose output pixel exists are listed
        lists = []
        for iy in range(H):
            for ix in range(W):
                ent = []
                for t, (ky, kx) in enumerate(taps):
                    dy_, dx_ = iy - ky, ix - kx
                    if dy_ % S == 0 and dx_ % S == 0 and 0 <= dy_ // S < OH and 0 <= dx_ // S < OW:
                        ent.append(((dy_ // S) * OW + dx_ // S, t))
                lists.append(ent)
        # per-tap transposed kernels wT[t][n, c] = W[ky, kx, c, n]
        w_index = np.arange(T * C * N).reshape(T, C, N)
        self.perm = _dev_i32(w_index.transpose(0, 2, 1).reshape(-1), device)
        self.wT = torch.empty(T * N * C, dtype=torch.float32, device=device)
        self.wT_planes = tl.PlaneBuf(T * N, C, device, interleaved=tl.b_interleaved(C))
        npix = H * W
        qq, bb = np.meshgrid(np.arange(npix), np.arange(B), indexing="ij")
        rowmap_in = _dev_i32((bb * npix + qq).reshape(-1), device)
        self.bwd_x = tl.masked_forward_op(lib, ws, B, device, pl.dy, N, self.wT_planes, C, lists, npix, dx, C,
                                          x if prev_act else None, prev_act, rowmap_in, pl.dx, mask_planes=pl.x)
        _derive(self, w)

    def forward(self):
        if self.s2d is not None:
            st = _lib.current_stream()
            x, xp, B = self.s2d
            if x is not None:
                _lib.check(self.lib.cb200_u8_s2d_planes(x.data_ptr(), B, self.H, self.W, self.C, self.S, xp.ptr, st))
        self.fwd.run()

    def run_perms(self):
        """weight-derived operands of this layer: the space-to-depth kernel (forward) and the per-tap transposed
        kernels of the data-gradient GEMM (run when the layer is prepared and by ThetaPlanes.refresh after every write
        of the weights)"""
        st = _lib.current_stream()
        if self.s2d is not None:
            _lib.check(self.lib.cb200_permute_f32(self.w.data_ptr(), self.w_perm.data_ptr(), self.w_perm.numel(),
                                                  self.w_s2d.data_ptr(), self.w_s2d_planes.ptr,
                                                  self.w_s2d_planes.stride, self.w_s2d_planes.cols, st))
        if self.bwd_x is not None:
            _lib.check(self.lib.cb200_permute_f32(self.w.data_ptr(), self.perm.data_ptr(), self.perm.numel(),
                                                  self.wT.data_ptr(), self.wT_planes.ptr, self.wT_planes.stride,
                                                  self.wT_planes.cols, st))

    def backward(self, weights=True, side=NO_SIDE):
        if weights:
            with side:        # weight / bias gradients only read dy and x: off the data-gradient chain
                self.bwd_w.run()
                if self.db_args is not None:
                    dy, M, N, db = self.db_args
                    _lib.check(self.lib.cb200_colsum(dy.data_ptr(), M, N, db.data_ptr(), self.ws.side().ptr(),
                                                     _lib.current_stream()))
        st = _lib.current_stream()
        for op, wt, perm in self.classes:
            _lib.check(self.lib.cb200_permute_f32(self.w.data_ptr(), perm.data_ptr(), perm.numel(), wt.data_ptr(),
                                                  None, 0, 0, st))
            op.run()
        if self.bwd_x is not None:
            self.bwd_x.run()
