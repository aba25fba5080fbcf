"""Q-value networks (DQN / DDQN / dueling) as flat-buffer device networks.

Structure and variable order follow the TF graph of the reference:
  embedder  -- image: Conv2d(32,8,4) Conv2d(64,4,2) Conv2d(64,3,1), ReLU, flatten (image_embedder.py:62-67, Medium);
               vector: Dense(256) ReLU (vector_embedder.py:58-61, Medium); input / 255 for images (embedder.py:103)
  middleware-- Dense(512) ReLU (fc_middleware.py:66-69, Medium); MiddlewareScheme.Empty = no layer at all, the heads
               read the flattened embedder output (fc_middleware.py:58-59; presets/Atari_Dueling_DDQN_with_PER_OpenAI.py:17:
               the dueling towers sit directly on the 3136-wide conv map, 3,293,863 trainable parameters)
  head      -- QHead: Dense(num_actions) (q_head.py:52-54);
               DuelingQHead: V: Dense(512) ReLU, Dense(1); A: Dense(512) ReLU, Dense(num_actions);
               Q = V + (A - mean_a A) (dueling_q_head.py:33-47)
  + one scalar ``gradients_from_head_0-0_rescalers`` variable (general_network.py:312-315; gradient identically 0)

With ``value_head`` the heads are the actor-critic pair VHead + PolicyHead (actor_critic_agent.py:66-70) as ONE
Dense(1 + num_actions): column 0 is V, columns 1..num_actions the policy logits.
"""
import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.architectures import tiled as tl
from coach_b200.architectures.layers import Conv2d, Dense, Workspace
from coach_b200.architectures.network import ParamStore, Sequential, make_u8_lut


class QNetworkDef(object):
    """Parameter layout + layer chain; instances bind it to buffers (see QNetworkInstance)."""

    def __init__(self, device, observation_shape, num_actions, dueling=False, embedder="auto", middleware_units=512,
                 head_copies=1, head_grad_rescale=1.0, embedder_scheme=None, value_head=False, gaussian_policy=False):
        """embedder_scheme: the input embedder's layers (InputEmbedderParameters.scheme as a list): for images a list of
        base_parameters.Conv2d specs, for vectors a list of base_parameters.Dense specs; None is the Medium embedder
        above (image_embedder.py:62-67 / vector_embedder.py:58-61).
        middleware_units: width of one FC middleware layer, a tuple of widths, or None / () for MiddlewareScheme.Empty.
        head_copies > 1 (Bootstrapped DQN, bootstrapped_dqn_agent.py:26-30): ``head_copies`` QHeads of ``num_actions``
        outputs on the same features, as ONE Dense(head_copies * num_actions) whose column block [k A, (k + 1) A) is
        head k; each block is Glorot-initialised with the fans of its own [F, A] layer, and there is one
        ``gradients_from_head_0-<k>_rescalers`` scalar per copy, initialised to ``head_grad_rescale``
        (general_network.py:304-325).
        value_head (ActorCritic): VHead Dense(1) + PolicyHead Dense(num_actions) as ONE Dense(1 + num_actions); column 0
        is initialised as normalized_columns_initializer(1.0) (v_head.py:44-47, head.py:28-33), the policy block
        Glorot-uniform with the fans of its own [F, num_actions] layer; one ``gradients_from_head_{0,1}-0_rescalers``
        scalar per head.
        gaussian_policy (with value_head, continuous actions; policy_head.py:102-152 with ContinuousEntropy): the
        num_actions = 2 D policy columns are fc_mean (columns 1..D, Glorot-uniform with the fans of its own [F, D]
        layer) and fc_std (columns D+1..2D, normalized_columns_initializer(0.01))."""
        self.value_head = bool(value_head)
        self.gaussian_policy = bool(gaussian_policy)
        if self.gaussian_policy and not (self.value_head and num_actions % 2 == 0):
            raise ValueError("gaussian_policy takes value_head and an even number of policy columns (mean | std)")
        if self.value_head and (dueling or head_copies != 1):
            raise NotImplementedError("the actor-critic head takes neither a dueling head nor head copies")
        self.head_copies = int(head_copies)
        self.head_grad_rescale = float(head_grad_rescale)
        if self.head_copies > 1 and dueling:
            raise NotImplementedError("head copies are implemented for the plain QHead only")
        if middleware_units is None:
            middleware_units = ()
        elif isinstance(middleware_units, int):
            middleware_units = (middleware_units,)
        self.middleware_units = tuple(int(u) for u in middleware_units)
        self.device = torch.device(device)
        self.obs_shape = tuple(observation_shape)
        self.num_actions = int(num_actions)
        self.dueling = bool(dueling)
        self.store = ParamStore(self.device)
        self.is_image = len(self.obs_shape) == 3
        layers = []
        if self.is_image:
            convs = ((32, 8, 4), (64, 4, 2), (64, 3, 1)) if embedder_scheme is None else \
                tuple((int(c.num_filters), int(c.kernel_size), int(c.strides)) for c in embedder_scheme)
            h, w, c = self.obs_shape
            for (n, k, s) in convs:
                conv = Conv2d((h, w), c, n, k, s, "relu")
                layers.append(conv)
                h, w, c = conv.OH, conv.OW, n
            flat = h * w * c
        else:
            flat = self.obs_shape[0]
            for u in ((256,) if embedder_scheme is None else tuple(int(d.units) for d in embedder_scheme)):
                layers.append(Dense(flat, u, "relu"))
                flat = u
        for u in self.middleware_units:
            layers.append(Dense(flat, u, "relu"))
            flat = u
        middleware_units = flat                 # width of what the head reads
        if not self.dueling:
            layers.append(Dense(middleware_units, self.head_copies * self.num_actions + self.value_head, None))
            self.trunk = Sequential(layers, self.store, "main/online/network_0")
            self.v_tower = self.a_tower = None
            kernel = self.trunk.names[-1][0]
            if self.gaussian_policy:
                D = self.num_actions // 2
                self.store.glorot_fans[kernel] = (middleware_units, D)
                self.store.normalized_columns[kernel] = [(0, 1, 1.0), (1 + D, D, 0.01)]
            elif self.head_copies > 1 or self.value_head:
                self.store.glorot_fans[kernel] = (middleware_units, self.num_actions)
            if self.value_head and not self.gaussian_policy:
                self.store.normalized_columns[kernel] = [(0, 1, 1.0)]
        else:
            self.trunk = Sequential(layers, self.store, "main/online/network_0")
            self.v_tower = Sequential([Dense(middleware_units, 512, "relu"), Dense(512, 1, None)], self.store,
                                      "main/online/network_0/dueling_q_values_head_0/state_value")
            self.a_tower = Sequential([Dense(middleware_units, 512, "relu"), Dense(512, self.num_actions, None)],
                                      self.store, "main/online/network_0/dueling_q_values_head_0/action_advantage")
        if self.value_head:
            for k in range(2):
                self.store.add("main/online/network_0/gradients_from_head_%d-0_rescalers" % k, ())
        elif self.head_copies == 1:
            self.store.add("main/online/network_0/gradients_from_head_0-0_rescalers", ())
        else:
            for k in range(self.head_copies):
                name = self.store.add("main/online/network_0/gradients_from_head_0-%d_rescalers" % k, ())
                self.store.initial_values[name] = self.head_grad_rescale
        self.store.finalize()
        self.lut = make_u8_lut(self.device) if self.is_image else None

    def instantiate(self, lib, ws, B, x, theta, grad=None, train=False):
        return QNetworkInstance(self, lib, ws, B, x, theta, grad, train)


class QNetworkInstance(object):
    def __init__(self, net, lib, ws, B, x, theta, grad, train):
        self.net, self.lib, self.B = net, lib, B
        dev = net.device
        x_is_u8 = isinstance(x, tl.PlaneBuf) or x.dtype == torch.uint8      # PlaneBuf: s2d plane of the uint8 frames
        # Large batches run the trunk on pre-split bf16 operands (architectures/tiled.py).  Whoever writes theta --
        # Adam, a target network copy, polyak, a checkpoint load -- calls theta_planes.refresh() right after the write.
        # (CB200_GEMM_TILED=0 keeps every layer on the gather-GEMM of cb200_gemm: A/B runs, bench.py --no-tc)
        self.theta_planes = tl.ThetaPlanes(lib, net.store, theta) \
            if (B >= 128 and B % 32 == 0 and _lib.tune_default("gemm_tiled", 1)) else None
        # dueling towers directly on a conv map (MiddlewareScheme.Empty, the Atari dueling-DDQN preset): the towers'
        # first layers are the two largest GEMMs of the network, so they run on the conv map's operand planes too
        last = net.trunk.layers[-1]
        self.towers_on_planes = bool(net.dueling and self.theta_planes is not None and not net.middleware_units and
                                     net.is_image and tl.channels_ok(last.N) and tl.width_ok(last.N))
        self.trunk = net.trunk.instantiate(lib, ws, B, x, theta, grad, x_is_u8=x_is_u8, lut=net.lut, train=train,
                                           theta_planes=self.theta_planes, last_planes=self.towers_on_planes)
        self.towers_dx = None
        if not net.dueling:
            self.q = self.trunk.out
            self.dq = self.trunk.d_out
        else:
            h = self.trunk.out                  # what the head reads (post-ReLU): middleware or embedder output
            dh = self.trunk.d_out               # gradient wrt its pre-activation
            self.q = torch.empty((B, net.num_actions), dtype=torch.float32, device=dev)
            self.dq = torch.empty_like(self.q) if train else None
            if self.towers_on_planes:
                self._towers_on_conv_map(lib, ws, B, h, dh, theta, grad, train)
            else:
                self.v = net.v_tower.instantiate(lib, ws, B, h, theta, grad, need_input_grad=train, input_act=1,
                                                 train=train, dx_in=dh, dx_accumulate=False)
                self.a = net.a_tower.instantiate(lib, ws, B, h, theta, grad, need_input_grad=train, input_act=1,
                                                 train=train, dx_in=dh, dx_accumulate=True)
        if self.theta_planes is not None:
            # kernels derived from the weights (per-tap transposed kernels of the data-gradient GEMMs, the
            # space-to-depth kernel of the first convolution) are re-derived together with the planes
            for sq in [self.trunk] + ([self.v, self.a] if net.dueling else []):
                self.theta_planes.derived += [layer.run_perms for layer in sq.layers]
            if self.towers_dx is not None:
                self.theta_planes.derived.append(self._towers_perm)

    def _towers_on_conv_map(self, lib, ws, B, h, dh, theta, grad, train):
        """V / A towers as tiled GEMMs on the planes of the last conv map [npix * B, C].  Forward and weight gradients
        are per tower; the data gradient into the conv map is ONE multi-tap GEMM over both towers: their
        pre-activation gradients are the two "pixels" of one [2B, 512] plane matrix, the per-pixel transposed kernels
        of both towers one weight stack, and every conv pixel's tap list has one entry per tower -- so the sum
        dV W_v^T + dA W_a^T is accumulated in the tensor-core accumulators instead of by a second, accumulating pass."""
        net, dev = self.net, self.net.device
        xp = self.trunk.act_planes[-1]
        npix, C = xp.npix, xp.cols
        H1 = net.v_tower.layers[0].N                                   # 512
        comb = tl.PlaneBuf(2 * B, H1, dev, npix=2) if train else None
        maps = [({0: comb.view_rows(t * B, B)} if train else None) for t in range(2)]
        self.v = net.v_tower.instantiate(lib, ws, B, h, theta, grad, input_act=1, train=train,
                                         theta_planes=self.theta_planes, x_planes=xp, dz_planes_map=maps[0])
        self.a = net.a_tower.instantiate(lib, ws, B, h, theta, grad, input_act=1, train=train,
                                         theta_planes=self.theta_planes, x_planes=xp, dz_planes_map=maps[1])
        assert self.v.layers[0].tiled_x and self.a.layers[0].tiled_x
        if not train:
            return
        store = net.store
        K = npix * C
        w_index = np.arange(K * H1).reshape(npix, C, H1)
        perm = torch.from_numpy(np.ascontiguousarray(w_index.transpose(0, 2, 1).reshape(-1), dtype=np.int32)).to(dev)
        wT = torch.empty(2 * npix * H1 * C, dtype=torch.float32, device=dev)
        wT_planes = tl.PlaneBuf(2 * npix * H1, C, dev, interleaved=tl.b_interleaved(C))
        w_src = [store.view(theta, seq.names[0][0]) for seq in (net.v_tower, net.a_tower)]
        qq, bb = np.meshgrid(np.arange(npix), np.arange(B), indexing="ij")
        rowmap = torch.from_numpy(np.ascontiguousarray((bb * npix + qq).reshape(-1), dtype=np.int32)).to(dev)
        op = tl.masked_forward_op(lib, ws, B, dev, comb, H1, wT_planes, C,
                                  [[(0, q), (1, npix + q)] for q in range(npix)], npix, dh, C, h, 1, rowmap,
                                  self.trunk.dz_planes[-1], mask_planes=xp)
        op.tag = "DuelingTowers.bwd_x"
        self.towers_dx = (op, perm, wT, wT_planes, w_src, npix * H1)

    def _towers_perm(self):
        op, perm, wT, wT_planes, w_src, half = self.towers_dx
        st = _lib.current_stream()
        for t, w in enumerate(w_src):
            pv = wT_planes.view_rows(t * half, half)
            _lib.check(self.lib.cb200_permute_f32(w.data_ptr(), perm.data_ptr(), perm.numel(),
                                                  wT.data_ptr() + 4 * t * perm.numel(), pv.ptr, pv.stride, pv.cols, st))

    def forward(self):
        self.trunk.forward()
        if self.net.dueling:
            self.v.forward()
            self.a.forward()
            _lib.check(self.lib.cb200_dueling_combine_fwd(self.v.out.data_ptr(), self.a.out.data_ptr(), self.B,
                                                          self.net.num_actions, self.q.data_ptr(),
                                                          _lib.current_stream()))
        return self.q

    # ---- a head computed by one of the agents' fused head kernels --------------------------------------------------------
    def feature_head(self):
        """the head is one Dense on a 256- or 512-wide ReLU feature layer whose fp32 activations are kept: what every
        fused head kernel reads"""
        if self.net.dueling or len(self.trunk.layers) < 2:
            return False
        head = self.trunk.layers[-1]
        return (type(head).__name__ == "Dense" and head.K in (256, 512) and self.trunk.acts[-2] is not None and
                self.trunk.layers[-2].act == 1)

    def head_fusable(self):
        """plain Dense(num_actions) head of <= 8 actions (cb200_dqn_head_fused)"""
        return self.feature_head() and self.trunk.layers[-1].N <= 8

    def ensemble_fusable(self):
        """head copies of <= 8 actions each (cb200_ensemble_head_fused)"""
        return (self.feature_head() and self.net.num_actions <= 8 and
                self.trunk.layers[-1].N == self.net.head_copies * self.net.num_actions)

    def bind_head_grads(self, d):
        """points a fused head descriptor's gradient outputs at this training instance: dh (dL/d of the feature layer's
        pre-activation, fp32 and / or its operand planes) and the head layer's dw / db in the gradient buffer"""
        store = self.net.store
        wname, bname = self.net.trunk.names[-1]
        dz, pl = self.trunk.dzs[-2], self.trunk.dz_planes[-2]
        d.dh = dz.data_ptr() if dz is not None else None
        if pl is not None:
            d.dh_planes, d.dh_plane_stride = pl.ptr, pl.stride
        d.dw, d.db = store.view(store.grad, wname).data_ptr(), store.view(store.grad, bname).data_ptr()

    def forward_features(self):
        """everything below the head: the feature layer's post-ReLU output is ``features``"""
        self.trunk.forward(upto=len(self.trunk.layers) - 1)
        return self.trunk.acts[-2]

    def backward_features(self, side=None):
        """expects the gradient w.r.t. the feature layer's pre-activation in trunk.dzs[-2] (/ its planes).
        side: a layers.SideStream for the weight-gradient launches (they leave the data-gradient chain)"""
        self.trunk.backward(layers=(0, len(self.trunk.layers) - 1), side=side)

    def backward(self, side=None):
        """expects d(loss)/dq in self.dq; leaves all parameter gradients in the grad buffer"""
        if self.net.dueling:
            _lib.check(self.lib.cb200_dueling_combine_bwd(self.dq.data_ptr(), self.B, self.net.num_actions,
                                                          self.v.d_out.data_ptr(), self.a.d_out.data_ptr(),
                                                          _lib.current_stream()))
            self.v.backward(side=side)      # writes d(middleware pre-activation)
            self.a.backward(side=side)      # accumulates into it
            if self.towers_dx is not None:
                self.towers_dx[0].run()     # both towers' data gradients into the conv map, one GEMM
        self.trunk.backward(side=side)
