"""Pre-split operand planes and the multi-tap tensor-core GEMM calls (include/coach_b200.h: cb200_gemm_tiled).

The tensor-core path of the learn step computes fp32 products as 3 x BF16 operand splits.  Splitting inside every GEMM
costs more than the GEMM, so every tensor that feeds a GEMM is kept, next to its fp32 form, as three bf16 "planes" in
the 8x8 core-tiled format of csrc/nn_gemm.cuh (``tiled_elem``): activations / gradients as [pixel * batch + b, channel]
matrices written by the producing GEMM's epilogue, parameters re-derived from theta after every write of it
(``ThetaPlanes.refresh``), per-tap transposed kernels by the permute kernel.  ``build_*`` below turn a layer geometry
into the tap lists of cb200_gemm_tiled:

  conv forward   C[q*B + b, n]      = sum_taps    X[pix_in(q, tap)*B + b, :] W_tap          (mode 0)
  conv dX        dX[q_in*B + b, c]  = sum_valid   dY[pix_out(q_in, tap)*B + b, :] W_tap^T    (mode 0, gather form)
  conv dW        dW[tap*C + c, n]   = sum_q sum_b X[pix_in(q, tap)*B + b, c] dY[q*B + b, n]  (mode 1)

Dense layers are the one-pixel case; a dense layer on a flattened conv map has one tap per pixel.
Reference semantics: rl_coach/architectures/tensorflow_components/layers.py:108-183 (+ tf.gradients).
"""
import ctypes
import os

import numpy as np
import torch

from coach_b200 import _lib


def _dev_i32(a, device):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int32)).to(device)


def b_interleaved(n):
    """B operands of the N <= 64 tile width (cb200_gemm_tiled: bn = 32 / 64) use row-group interleaved planes: one
    TMA box then delivers [b1 | b2 | b3] as ONE operand (csrc/nn_gemm_tiled.cuh, kCat)"""
    return bool(_lib.tune_default("gemm_cat", 1)) and (n <= 64 or n % 128 != 0)


class PlaneBuf(object):
    """bf16 hi / mid / lo planes of a [rows, cols] matrix (rows = npix * batch) in the core-tiled format.
    interleaved: (row group | plane | column core | 64) instead of three planes `rows * cols` apart -- the layout of
    the B operands of the narrow GEMMs (``b_interleaved``); its plane stride is passed to the library as -1."""

    def __init__(self, rows, cols, device, npix=1, nplanes=3, interleaved=False):
        assert rows % 8 == 0 and cols % 8 == 0, (rows, cols)
        self.rows, self.cols, self.npix, self.nplanes = int(rows), int(cols), int(npix), int(nplanes)
        self.interleaved = bool(interleaved)
        assert not self.interleaved or self.nplanes == 3
        self.t = torch.zeros((self.nplanes, self.rows * self.cols), dtype=torch.bfloat16, device=device)

    @property
    def ptr(self):
        return self.t.data_ptr()

    @property
    def stride(self):
        return -1 if self.interleaved else self.rows * self.cols

    def view_rows(self, lo, n, npix=1):
        """rows [lo, lo + n) as a plane matrix of their own (same memory, same plane stride); lo, n multiples of 8"""
        assert lo % 8 == 0 and n % 8 == 0 and 0 <= lo and lo + n <= self.rows
        return PlaneView(self, lo, n, npix)

    def load(self, lib, m):
        """planes <- split of an fp32 [rows, cols] matrix (tests, host-written inputs)"""
        m = m.contiguous().view(self.rows, self.cols).float()
        seg = torch.tensor([[0, self.rows, self.cols, 0, int(self.interleaved)]], dtype=torch.int64, device=m.device)
        _lib.check(lib.cb200_split_planes(m.data_ptr(), self.ptr, 0 if self.interleaved else self.stride, seg.data_ptr(), 1,
                                          self.rows * self.cols, _lib.current_stream()))
        torch.cuda.current_stream().synchronize()      # m / seg are temporaries
        return self

    def to_dense(self):
        """fp32 [rows, cols] reconstruction hi + mid + lo (tests)"""
        if self.interleaved:
            p = self.t.reshape(self.rows // 8, 3, self.cols // 8, 8, 8).float()
            v = (p[:, 0] + p[:, 1]) + p[:, 2]
            return v.permute(0, 2, 1, 3).reshape(self.rows, self.cols)
        v = self.t[0].float()
        if self.nplanes == 3:
            v = (v + self.t[1].float()) + self.t[2].float()
        v = v.view(self.rows // 8, self.cols // 8, 8, 8).permute(0, 2, 1, 3)
        return v.reshape(self.rows, self.cols)


class PlaneView(object):
    """A run of 8-row groups of a PlaneBuf: in the core-tiled format whole row groups are contiguous inside a plane,
    so the view is the parent's memory at an element offset, with the PARENT's plane stride."""

    def __init__(self, parent, lo, n, npix=1):
        self.parent, self.lo = parent, int(lo)
        self.rows, self.cols, self.npix, self.nplanes = int(n), parent.cols, int(npix), parent.nplanes
        self.interleaved = parent.interleaved
        self.t = parent.t                      # keeps the storage alive

    @property
    def ptr(self):
        return self.parent.ptr + 2 * self.lo * self.cols * (3 if self.interleaved else 1)

    @property
    def stride(self):
        return self.parent.stride

    def to_dense(self):
        return self.parent.to_dense()[self.lo:self.lo + self.rows]


def channels_ok(c):
    """a_cols constraint of cb200_gemm_tiled"""
    return c in (32, 64, 128) or (c > 128 and c % 128 == 0)


def width_ok(n):
    """n constraint of cb200_gemm_tiled"""
    return n == 32 or (n > 0 and n % 64 == 0)


class ThetaPlanes(object):
    """Planes of every 2-D-able kernel of a flat parameter buffer, at the kernels' own element offsets.  ``refresh``
    re-derives all of them from the current fp32 values in one launch; whoever writes theta (Adam, target network
    copies, polyak, checkpoint loads) calls it right after the write."""

    def __init__(self, lib, store, theta):
        self.lib, self.store, self.theta = lib, store, theta
        # further kernels over theta that run with the refresh: transposed / permuted kernels of the data-gradient
        # GEMMs, the space-to-depth kernel of the first convolution
        self.derived = []
        # one buffer of 6 * size elements.  Planar kernels: plane p of the tensor at `off` sits at p * size + off
        # (first half).  Row-group interleaved kernels (narrow B operands, ``b_interleaved``): [3 off, 3 off + 3 rows
        # cols) of the second half.
        self.buf = torch.zeros(6 * store.size, dtype=torch.bfloat16, device=theta.device)
        self.planes = self.buf[:3 * store.size].view(3, store.size)
        self.planes_il = self.buf[3 * store.size:]
        segs, self.max_elems = [], 0
        self.layout = {}
        for name, (off, shape) in store.entries.items():
            if not name.endswith("kernel") or len(shape) < 2:
                continue
            rows, cols = int(np.prod(shape[:-1])), int(shape[-1])
            if rows % 8 or cols % 8 or off % 8:
                continue
            il = b_interleaved(cols)
            segs.append((off, rows, cols, 3 * store.size + 3 * off if il else off, int(il)))
            self.layout[off] = il
            self.max_elems = max(self.max_elems, rows * cols)
        self.names = set(n for n in store.entries)
        self.segs = torch.tensor(segs, dtype=torch.int64, device=theta.device) if segs else None
        self.eligible = {s[0] for s in segs}

    def has(self, name):
        return self.store.entries[name][0] in self.eligible

    def interleaved(self, name):
        return bool(self.layout.get(self.store.entries[name][0], False))

    def ptr(self, name):
        off = self.store.entries[name][0]
        if self.layout.get(off, False):
            return self.planes_il.data_ptr() + 2 * 3 * off
        return self.planes.data_ptr() + 2 * off

    def stride_of(self, name):
        return -1 if self.interleaved(name) else self.store.size

    @property
    def stride(self):
        return self.store.size

    def refresh(self):
        for fn in self.derived:
            fn()
        if self.segs is not None:
            _lib.check(self.lib.cb200_split_planes(self.theta.data_ptr(), self.planes.data_ptr(), self.stride,
                                                   self.segs.data_ptr(), self.segs.shape[0], self.max_elems,
                                                   _lib.current_stream()))


class PlaneCtx(object):
    """What one layer needs to run on pre-split operands."""

    def __init__(self, x=None, y=None, dy=None, dx=None, w_ptr=0, w_stride=0):
        self.x, self.y, self.dy, self.dx = x, y, dy, dx       # PlaneBuf or None
        # planes of this layer's kernel inside ThetaPlanes; w_stride -1 = row-group interleaved (``b_interleaved``)
        self.w_ptr, self.w_stride = w_ptr, w_stride


TILED_MAX_CHUNKS = int(os.environ.get("CB200_TILED_MAX_CHUNKS", "20"))
SPLIT_WAVES = int(os.environ.get("CB200_SPLIT_WAVES", "2"))     # CTAs per SM a split-reduction launch aims for


def pick_splits_tiled(tiles, total_chunks, sm=132):
    """reduction slices of a tiled GEMM: at most TILED_MAX_CHUNKS chunks (40 accumulating k16 steps) per slice -- the
    error of the tensor-core fp32 accumulation grows with the accumulation count (tests/test_learn_gpu.py holds every
    gradient of the B = 512 step within 1e-5) -- and more slices when the tile count alone does not fill the
    machine (132 SMs on an H100 SXM)"""
    need = (total_chunks + TILED_MAX_CHUNKS - 1) // TILED_MAX_CHUNKS
    if tiles >= sm:
        return int(max(1, need))
    s = max(1, (SPLIT_WAVES * sm + tiles - 1) // tiles)
    s = min(s, max(1, total_chunks // 4))
    return int(max(s, need))


class TGemmOp(object):
    """A prepared cb200_gemm_tiled call.  ``macs`` = multiply-accumulates of the contraction, ``nprod`` = bf16 tensor-core
    products issued per multiply (6: 3xBF16 split of both operands, 3: exact uint8 A)."""

    trace = None          # bench.py: a list -> (op, start event, end event) is appended around every launch

    def __init__(self, lib, ws, **fields):
        self.lib, self.ws = lib, ws
        self.macs = int(fields.pop("macs", 0))
        self.tag = fields.pop("tag", "")
        self.keep = []
        self.desc = _lib.TGemmDesc()
        for k, v in fields.items():
            if torch.is_tensor(v):
                self.keep.append(v)
                v = v.data_ptr()
            elif isinstance(v, (PlaneBuf, PlaneView)):
                self.keep.append(v)
                v = v.ptr
            setattr(self.desc, k, v)
        d = self.desc
        rows = d.num_q * d.batch if d.mode == 0 else d.taps * d.a_cols + (1 if d.bias_row else 0)
        if d.splits > 1:
            ws.require(d.splits * rows * d.n)

    @property
    def nprod(self):
        return 3 if self.desc.a_num_planes == 1 else 6

    def run(self):
        if self.desc.splits > 1:
            self.desc.workspace = self.ws.ptr()
        if TGemmOp.trace is not None:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            _lib.check(self.lib.cb200_gemm_tiled(ctypes.byref(self.desc), _lib.current_stream()))
            e1.record()
            TGemmOp.trace.append((self, e0, e1))
            return
        _lib.check(self.lib.cb200_gemm_tiled(ctypes.byref(self.desc), _lib.current_stream()))


def _tiles0(num_q, B, n):
    bn = 32 if n <= 32 else (128 if n % 128 == 0 else 64)
    return num_q * ((B + 127) // 128) * ((n + bn - 1) // bn)


def _tiles1(rows, n):
    bn = 32 if n <= 32 else (128 if n % 128 == 0 else 64)
    return ((rows + 127) // 128) * ((n + bn - 1) // bn)


def forward_op(lib, ws, B, device, x, Ca, w_ptr, w_stride, N, lists, num_q, c, ldc, bias, act, rowmap, y_planes,
               w_rows=None, **extra):
    """mode 0 with explicit per-pixel tap lists: `lists[q]` = [(a_pix, w_blk), ...]"""
    ptr = np.zeros(num_q + 1, dtype=np.int64)
    flat = []
    for q in range(num_q):
        flat.extend(lists[q])
        ptr[q + 1] = len(flat)
    max_len = int(np.max(np.diff(ptr))) if num_q else 0
    flat = np.asarray(flat, dtype=np.int32).reshape(-1, 2) if flat else np.zeros((1, 2), dtype=np.int32)
    total = max_len * (Ca // 32)
    extra.setdefault("macs", int(ptr[-1]) * Ca * B * N)
    il = int(w_stride == -1)
    assert not il or b_interleaved(N), "interleaved B planes only for the narrow tile widths"
    return TGemmOp(lib, ws, mode=0, batch=B, a_planes=x, a_plane_stride=x.stride, a_cols=Ca, b_planes=w_ptr,
                   b_plane_stride=0 if il else w_stride, b_interleaved=il, n=N, list_ptr=_dev_i32(ptr, device), list=_dev_i32(flat, device),
                   max_list_len=max_len, num_q=num_q, taps=0, c=c, ldc=ldc, bias=bias, act=act, a_rows=x.rows,
                   b_rows=int(w_rows if w_rows is not None else (int(flat[:, 1].max()) + 1) * Ca),
                   c_rowmap=rowmap, splits=pick_splits_tiled(_tiles0(num_q, B, N), total),
                   c_planes=y_planes if y_planes is not None else None,
                   c_plane_stride=y_planes.stride if y_planes is not None else 0,
                   c_plane_cols=N if y_planes is not None else 0, a_num_planes=x.nplanes, **extra)


def masked_forward_op(lib, ws, B, device, x, Ca, w_buf, N, lists, num_q, c, ldc, mask_y, mask_act, rowmap, y_planes,
                      mask_planes=None):
    """data-gradient flavour: no bias / activation, previous layer's activation derivative in the epilogue -- read
    from the activation's planes when they exist (``mask_planes``, same geometry as the result), else from fp32"""
    op = forward_op(lib, ws, B, device, x, Ca, w_buf.ptr, w_buf.stride, N, lists, num_q, c, ldc, None, 0, rowmap,
                    y_planes, w_rows=w_buf.rows)
    op.keep.append(w_buf)
    if mask_act and mask_planes is not None and mask_planes.nplanes == 3 and mask_planes.cols == N:
        op.keep.append(mask_planes)
        op.desc.mask_planes = mask_planes.ptr
        op.desc.mask_plane_stride = mask_planes.stride
        op.desc.mask_act = mask_act
        op.desc.c_plane_cols = N
    elif mask_y is not None and mask_act:
        op.keep.append(mask_y)
        op.desc.mask_y = mask_y.data_ptr()
        op.desc.mask_act = mask_act
    return op


def wgrad_op(lib, ws, B, device, x, Ca, g, N, a_pix, taps, num_q, dw, **extra):
    """mode 1: dw [taps * Ca, N] row-major fp32"""
    total = num_q * (B // 32)
    extra.setdefault("macs", taps * Ca * N * num_q * B)
    host = np.ascontiguousarray(np.asarray(a_pix).reshape(-1), dtype=np.int32)
    op = TGemmOp(lib, ws, mode=1, batch=B, a_planes=x, a_plane_stride=x.stride, a_cols=Ca, b_planes=g,
                 b_plane_stride=g.stride, n=N, a_pix=_dev_i32(host, device), num_q=num_q,
                 taps=taps, max_list_len=0, c=dw, ldc=N, act=0, a_rows=x.rows, b_rows=g.rows,
                 splits=pick_splits_tiled(_tiles1(taps * Ca, N), total), a_num_planes=x.nplanes, **extra)
    if _lib.tune_default("wgrad_tma", 1):
        # host copy of the tap table: lets the library fetch the A^T operand of a chunk with one TMA box
        op.keep.append(host)
        op.desc.a_pix_host = host.ctypes.data
    return op
