"""Flat-buffer networks for the learn step.

``ParamStore`` keeps ALL trainable tensors of one network in a single fp32 buffer (plus same-shaped gradient and Adam
slot buffers), in TensorFlow variable-creation order -- embedders (sorted by input name) -> middleware -> head ->
``gradients_from_head_*_rescalers`` scalar (general_network.py:244-349, SURVEY.md Q15) -- so that per-tensor
comparisons with the reference line up, the optimizer / clipping / polyak / NCCL all-reduce are ONE launch each over
the flat buffer, and a target network is just a second ``theta``.

``Sequential`` wires a chain of layers (coach_b200/architectures/layers.py) to persistent activation / gradient
buffers for one batch size; an "instance" binds the chain to one parameter buffer and one input tensor.
"""
from collections import OrderedDict

import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.architectures import tiled as tl
from coach_b200.architectures.layers import ACT, Workspace


class ParamStore(object):
    def __init__(self, device):
        self.device = torch.device(device)
        self.entries = OrderedDict()      # name -> (offset, shape)
        self.size = 0
        self.theta = None
        self.glorot_fans = {}             # kernel name -> (fan_in, fan_out) when it is not the tensor's own
        self.initial_values = {}          # rescaler name -> initial value (default 1.0)
        self.normalized_columns = {}      # kernel name -> [(first column, columns, std)]: normalized_columns_initializer

    def add(self, name, shape):
        if self.theta is not None:
            raise RuntimeError("ParamStore is finalised")
        n = int(np.prod(shape)) if len(shape) else 1
        # keep every tensor 32-byte aligned inside the flat buffer (vector loads in the kernels; 16-byte aligned
        # core-matrix rows in the bf16 planes that shadow the buffer, architectures/tiled.py)
        self.size = (self.size + 7) // 8 * 8
        self.entries[name] = (self.size, tuple(shape))
        self.size += n
        return name

    def finalize(self):
        self.size = (self.size + 7) // 8 * 8
        z = lambda: torch.zeros(self.size, dtype=torch.float32, device=self.device)   # noqa: E731
        self.theta, self.grad, self.m, self.v = z(), z(), z(), z()
        return self

    def view(self, buf, name):
        off, shape = self.entries[name]
        n = int(np.prod(shape)) if len(shape) else 1
        return buf[off:off + n].view(shape if len(shape) else (1,))

    def new_buffer(self):
        return torch.zeros(self.size, dtype=torch.float32, device=self.device)

    def num_params(self):
        return sum(int(np.prod(s)) if len(s) else 1 for _, s in self.entries.values())

    # -- initialisation (TF defaults: glorot-uniform kernels, zero biases; head.py:93 xavier) ------------------------
    def init_glorot(self, generator=None):
        for name, (off, shape) in self.entries.items():
            v = self.view(self.theta, name)
            if name.endswith("kernel"):
                if len(shape) == 4:
                    rf = shape[0] * shape[1]
                    fan_in, fan_out = rf * shape[2], rf * shape[3]
                else:
                    fan_in, fan_out = shape[0], shape[1]
                fan_in, fan_out = self.glorot_fans.get(name, (fan_in, fan_out))
                limit = float(np.sqrt(6.0 / (fan_in + fan_out)))
                cpu = (torch.rand(shape, generator=generator, dtype=torch.float32) * 2 - 1) * limit
                for c0, n, std in self.normalized_columns.get(name, ()):   # head.py:28-33: randn scaled to a column
                    w = torch.randn((shape[0], n), generator=generator, dtype=torch.float32)    # norm of std
                    cpu[:, c0:c0 + n] = w * (std / torch.sqrt((w * w).sum(dim=0, keepdim=True)))
                v.copy_(cpu)
            elif name.endswith("rescalers"):
                v.fill_(self.initial_values.get(name, 1.0))
            else:
                v.zero_()

    def load_named(self, tensors: dict, buf=None):
        buf = self.theta if buf is None else buf
        for name, t in tensors.items():
            self.view(buf, name).copy_(torch.as_tensor(t, dtype=torch.float32).reshape(self.entries[name][1] or (1,)))

    def export_named(self, buf=None):
        buf = self.theta if buf is None else buf
        return OrderedDict((name, self.view(buf, name).detach().cpu().numpy().copy()) for name in self.entries)


class Sequential(object):
    """layers: list of layer objects; params registered as '<prefix>/<i>_<LayerType>/<kernel|bias>'."""

    def __init__(self, layers, store, prefix):
        self.layers = layers
        self.store = store
        self.names = []
        for i, layer in enumerate(layers):
            base = "%s/%s_%d" % (prefix, type(layer).__name__, i)
            self.names.append([store.add(base + "/" + pname, shape) for pname, shape in layer.param_shapes])

    def instantiate(self, lib, ws, B, x, theta, grad=None, x_is_u8=False, lut=None, need_input_grad=False,
                    input_act=0, train=False, dx_in=None, dx_accumulate=False, theta_planes=None, x_planes=None,
                    last_planes=False, dz_planes_map=None):
        """need_input_grad: also produce the gradient wrt the (pre-activation of the) input, masked by
        ``input_act``' evaluated on x; it is written (or, with dx_accumulate, added) to ``dx_in``.
        x_planes: operand planes of the input (a PlaneBuf written by whoever produces x); last_planes: the last
        layer's output / pre-activation gradient carry planes too (their consumers / producers are tiled GEMMs of
        another chain); dz_planes_map {layer index: planes}: use these planes for that layer's pre-activation gradient
        (several chains sharing one plane matrix so that ONE GEMM can contract over all of them)."""
        return SequentialInstance(self, lib, ws, B, x, theta, grad, x_is_u8, lut, need_input_grad, input_act, train,
                                  dx_in, dx_accumulate, theta_planes, x_planes, last_planes, dz_planes_map)


class SequentialInstance(object):
    """Binds a Sequential to (batch size, input tensor, parameter buffer).  ``train=True`` also allocates the
    pre-activation gradient buffers and prepares the backward ops (gradients land in ``grad``)."""

    def __init__(self, seq, lib, ws, B, x, theta, grad, x_is_u8, lut, need_input_grad, input_act, train,
                 dx_in=None, dx_accumulate=False, theta_planes=None, x_planes=None, last_planes=False,
                 dz_planes_map=None):
        import copy
        self.seq, self.B = seq, B
        dev = theta.device
        store = seq.store
        self.layers = [copy.copy(l) for l in seq.layers]
        self.acts, self.dzs = [], []
        self.x = x
        self.dx_in = dx_in
        prev, prev_act = x, input_act
        if need_input_grad and dx_in is None:
            self.dx_in = torch.empty((B, int(np.prod(self.layers[0].in_shape))), dtype=torch.float32, device=dev)
        for i, layer in enumerate(self.layers):
            y = torch.empty((B, layer.out_elems()), dtype=torch.float32, device=dev)
            dz = torch.empty_like(y) if train else None
            self.acts.append(y)
            self.dzs.append(dz)
        # theta_planes (tiled.ThetaPlanes): run on pre-split bf16 operands.  Hidden activations / pre-activation
        # gradients are produced by GEMM epilogues only and consumed by GEMMs, so they carry planes [pixels * B,
        # channels]; the last layer's output and gradient are touched by head kernels and stay plain fp32.
        self.act_planes = [None] * len(self.layers)
        self.dz_planes = [None] * len(self.layers)
        if theta_planes is not None and B % 32 == 0:
            for i, layer in enumerate(self.layers if last_planes else self.layers[:-1]):
                npix, ch = layer.out_pixels(), layer.N
                if ch % 8 == 0:
                    self.act_planes[i] = tl.PlaneBuf(npix * B, ch, dev, npix=npix)
                    if train:
                        self.dz_planes[i] = (dz_planes_map or {}).get(i) or tl.PlaneBuf(npix * B, ch, dev, npix=npix)
        for i, layer in enumerate(self.layers):
            wname, bname = seq.names[i]
            w, b = store.view(theta, wname), store.view(theta, bname)
            dw = store.view(grad, wname) if train else None
            db = store.view(grad, bname) if train else None
            first = i == 0
            dx = (self.dx_in if first else self.dzs[i - 1]) if train else None
            need_dx = train and (not first or need_input_grad)
            ctx = None
            if theta_planes is not None and B % 32 == 0:
                ctx = tl.PlaneCtx(x=x_planes if first else self.act_planes[i - 1], y=self.act_planes[i],
                                  dy=self.dz_planes[i], dx=None if first else self.dz_planes[i - 1],
                                  w_ptr=theta_planes.ptr(wname) if theta_planes.has(wname) else 0,
                                  w_stride=theta_planes.stride_of(wname) if theta_planes.has(wname) else 0)
            if train:
                layer.prepare(lib, ws, B, dev, prev, self.acts[i], w, b, dw, db, self.dzs[i], dx,
                              x_is_u8=(x_is_u8 and first), lut=lut, need_dx=need_dx, prev_act=prev_act,
                              dx_accumulate=(dx_accumulate and first), planes=ctx)
            else:
                self._prepare_fwd_only(layer, lib, ws, B, dev, prev, self.acts[i], w, b, x_is_u8 and first, lut, ctx)
            for attr in ("fwd", "bwd_w", "bwd_x"):
                op = getattr(layer, attr, None)
                if isinstance(op, tl.TGemmOp):
                    op.tag = "%s_%d.%s" % (type(layer).__name__, i, attr)
            prev, prev_act = self.acts[i], layer.act
        # Forward-only instances (target networks): a hidden activation whose consumer reads its planes needs no fp32
        # copy -- the epilogue is bound by write bandwidth, and the fp32 result is 40 % of what it writes.
        def tiled(op):
            return isinstance(op, tl.TGemmOp)

        for i in range(len(self.layers) - 1):
            op, nxt = getattr(self.layers[i], "fwd", None), self.layers[i + 1]
            if not (tiled(op) and op.desc.c_planes and tiled(getattr(nxt, "fwd", None)) and
                    nxt.fwd.desc.a_num_planes == 3):
                continue
            # the next layer reads this activation as planes in its forward; in training it must also do so in its
            # weight gradient and take the derivative mask of its data gradient from the planes
            bw, bx = getattr(nxt, "bwd_w", None), getattr(nxt, "bwd_x", None)
            if train and not (tiled(bw) and (bx is None or (tiled(bx) and not bx.desc.mask_y))):
                continue
            op.desc.c = None
            self.acts[i] = None                  # not produced: fail loudly if anything asks for it
        if train:
            # pre-activation gradients: dz[i] is written by layer i+1's data-gradient GEMM and read by layer i's
            # weight / data gradients; when both read planes (and the bias gradient rides in the GEMM), no fp32 copy
            for i in range(len(self.layers) - 1):
                cur, nxt = self.layers[i], self.layers[i + 1]
                prod = getattr(nxt, "bwd_x", None)
                bw, bx = getattr(cur, "bwd_w", None), getattr(cur, "bwd_x", None)
                if tiled(prod) and prod.desc.c_planes and tiled(bw) and bw.desc.bias_row and \
                        getattr(cur, "db_args", None) is None and (bx is None or tiled(bx)):
                    prod.desc.c = None
                    self.dzs[i] = None
        self.out = self.acts[-1]
        self.d_out = self.dzs[-1]
        self.train = train

    @staticmethod
    def _prepare_fwd_only(layer, lib, ws, B, dev, x, y, w, b, x_is_u8, lut, ctx=None):
        # reuse prepare() with dummy gradient tensors but drop the backward ops: forward descriptors are identical
        layer.prepare(lib, ws, B, dev, x, y, w, b, None, None, None, None, x_is_u8=x_is_u8, lut=lut, need_dx=False,
                      planes=ctx)

    def forward(self, upto=None):
        """upto: run only the first ``upto`` layers (the caller computes the rest itself, e.g. a fused head kernel)"""
        for layer in (self.layers if upto is None else self.layers[:upto]):
            layer.forward()
        return self.out

    def backward(self, weights=True, layers=None, side=None):
        """weights=False: data gradients only (d(out)/d(input), e.g. dQ/da through the critic).  layers=(lo, hi): only
        layers lo <= i < hi, last first (e.g. everything below a head the caller differentiates itself)."""
        lo, hi = (0, len(self.layers)) if layers is None else layers
        for i in reversed(range(lo, hi)):
            if side is not None:
                self.layers[i].backward(weights, side=side)
            else:
                self.layers[i].backward(weights)


def make_u8_lut(device, rescale=255.0, offset=0.0):
    """lut[v] = float32(v) / rescale - offset, the embedder's input normalisation (embedder.py:103-104) evaluated in
    fp32 exactly like TensorFlow would (true division, not a reciprocal multiply)."""
    v = torch.arange(256, dtype=torch.float32)
    lut = ((v / np.float32(rescale)) - np.float32(offset)).to(device)
    # with no offset the table is exactly v / rescale: declared to the GEMM (cb200_gemm_desc.a_u8_div) so that the
    # tensor-core path can contract the raw integers exactly and divide once
    lut.u8_div = float(rescale) if offset == 0.0 else 0.0
    return lut
