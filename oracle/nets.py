"""torch-CPU fp32 restatement of the TensorFlow-1.x graph semantics of the learn step.  TEST INFRASTRUCTURE ONLY.

**Parity unpinned**: TensorFlow (tensorflow>=1.9,<=1.14, setup.py:69,73) cannot be installed here and the reference
holds no unit test of any loss, gradient or optimizer step (SURVEY.md section 8c).  What is restated, and from where:

  embedders   rl_coach/architectures/tensorflow_components/embedders/embedder.py:95-124 (x / 255, conv/dense stack)
              image_embedder.py:62-67 (Conv2d(32,8,4),(64,4,2),(64,3,1), VALID, NHWC, ReLU), vector_embedder.py:58-61
  middleware  middlewares/fc_middleware.py:66-69 (Dense(512) ReLU)
  heads       heads/q_head.py:52-54, heads/dueling_q_head.py:33-47, heads/head.py:165-177 (weighted loss, mean over
              the batch of the per-sample sum)
  losses      tf.losses.huber_loss(delta=1) / tf.losses.mean_squared_error, Reduction.NONE (q_head.py:44-47)
  gradients   tf.gradients(total_loss, weights) + tf.global_norm + tf.clip_by_global_norm (architecture.py:193-240)
  optimizer   tf.train.AdamOptimizer, kernel form of tensorflow/core/kernels/training_ops.cc ApplyAdam:
              alpha = lr*sqrt(1-b2^t)/(1-b1^t); m += (g-m)(1-b1); v += (g^2-v)(1-b2); var -= m*alpha/(sqrt(v)+eps)
  target      architecture.py:598-607 set_weights: rate*new + (1-rate)*old on host fp32
  DQN step    agents/dqn_agent.py:81-113, agents/ddqn_agent.py:42-43 (fp64 scalar target math on fp32 Q-values)

Parameters are exchanged as {name: ndarray} dicts in TF layout (conv kernels HWIO, dense kernels [in, out]).  All
functions take a ``dtype`` so that the same code gives an fp64 "ground truth" to measure both implementations against.
"""
from collections import OrderedDict

import numpy as np
import torch
import torch.nn.functional as F


def _t(a, dtype):
    return torch.as_tensor(np.asarray(a)).to(dtype)


def huber(pred, label, delta=1.0):
    """tf.losses.huber_loss element-wise (Reduction.NONE)."""
    err = pred - label
    abs_err = err.abs()
    quad = torch.clamp(abs_err, max=delta)
    lin = abs_err - quad
    return 0.5 * quad * quad + delta * lin


class QNetOracle(object):
    """Functional Q-network; ``params`` is an OrderedDict name -> tensor in creation order."""

    def __init__(self, observation_shape, num_actions, dueling=False, dtype=torch.float32, middleware=True):
        """middleware=False: MiddlewareScheme.Empty (fc_middleware.py:58-59), the head reads the embedder output"""
        self.middleware = middleware
        self.obs_shape = tuple(observation_shape)
        self.A = num_actions
        self.dueling = dueling
        self.dtype = dtype
        self.is_image = len(self.obs_shape) == 3

    def forward(self, params, x, kink=None):
        """x: uint8 [B,H,W,C] (image) or float [B,K].  Returns Q [B,A].

        kink (optional): {"masks": [bool tensor per ReLU, in the order the ReLUs are evaluated, this function's layout],
        "tol": t}.  A ReLU is not differentiable at 0: where a pre-activation lies within rounding noise of zero
        (|z| <= t * max|z|) both 0 and 1 are valid fp32 derivatives, and two correct implementations that sum in
        different orders can land on different sides.  There -- and only there -- the given mask (the implementation
        under test's) replaces this evaluation's own; "flipped" counts those elements, "hard" the disagreements
        elsewhere (genuine errors, which the caller asserts to be zero)."""
        p = list(params.values())
        k = 0
        h = torch.as_tensor(x).to(self.dtype)
        relu_i = [0]

        def relu(z):
            i = relu_i[0]
            relu_i[0] += 1
            if kink is None or i >= len(kink["masks"]) or kink["masks"][i] is None:
                return F.relu(z)
            own = z > 0
            other = kink["masks"][i].to(torch.bool).reshape(z.shape)
            near = z.detach().abs() <= kink["tol"] * z.detach().abs().max()
            m = torch.where(near, other, own)
            kink["flipped"] = kink.get("flipped", 0) + int((m != own).sum())
            kink["hard"] = kink.get("hard", 0) + int(((other != own) & ~near).sum())
            return z * m.to(z.dtype)

        if self.is_image:
            h = h / 255.0                                   # embedder.py:103 (true division)
            h = h.permute(0, 3, 1, 2)                       # NHWC -> NCHW for torch
            for stride in (4, 2, 1):
                w, b = p[k], p[k + 1]
                k += 2
                h = relu(F.conv2d(h, w.permute(3, 2, 0, 1), b, stride=stride))       # HWIO -> OIHW, VALID
            h = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)                         # flatten in NHWC order
        else:
            h = relu(h @ p[k] + p[k + 1])
            k += 2
        if self.middleware:
            h = relu(h @ p[k] + p[k + 1])                   # middleware Dense(512)
            k += 2
        if not self.dueling:
            return h @ p[k] + p[k + 1]
        v = relu(h @ p[k] + p[k + 1]) @ p[k + 2] + p[k + 3]
        a = relu(h @ p[k + 4] + p[k + 5]) @ p[k + 6] + p[k + 7]
        return v + (a - a.mean(dim=1, keepdim=True))

    def cast(self, named):
        return OrderedDict((n, _t(v, self.dtype)) for n, v in named.items())


def q_head_loss(q, targets, weights, huber_loss=True):
    """head.py:165-177: mean_b( w_b * sum_a l(target, q) ) with loss_weight 1."""
    l = huber(q, targets) if huber_loss else (q - targets) ** 2
    per_sample = l.sum(dim=1)
    if weights is not None:
        per_sample = weights * per_sample
    return per_sample.mean()


def dqn_targets(q_next, q_select, q_online, actions, rewards, game_overs, discount):
    """dqn_agent.py:92-103, the Python loop verbatim in spirit: fp64 scalar math on fp32 network outputs."""
    q_next = np.asarray(q_next)
    q_online = np.asarray(q_online)
    sel = np.argmax(np.asarray(q_select), 1)
    targets = q_online.copy()
    td = np.zeros(len(actions), dtype=np.float64)
    for i in range(len(actions)):
        new_target = rewards[i] + (1.0 - game_overs[i]) * discount * q_next[i][sel[i]]
        td[i] = np.abs(new_target - targets[i, actions[i]])
        targets[i, actions[i]] = new_target
    return targets, td


class AdamTF(object):
    """TF-1.x Adam on a list of tensors (same dtype as the params)."""

    def __init__(self, params, lr, beta1=0.9, beta2=0.99, eps=1e-4, dtype=torch.float32):
        self.lr, self.b1, self.b2, self.eps = lr, beta1, beta2, eps
        self.dtype = dtype
        npd = np.float32 if dtype == torch.float32 else np.float64
        self.npd = npd
        self.b1p, self.b2p = npd(beta1), npd(beta2)
        self.m = [torch.zeros_like(p) for p in params]
        self.v = [torch.zeros_like(p) for p in params]

    def step(self, params, grads):
        npd = self.npd
        alpha = npd(self.lr) * np.sqrt(npd(1) - self.b2p) / (npd(1) - self.b1p)
        out = []
        for i, (p, g) in enumerate(zip(params, grads)):
            self.m[i] = self.m[i] + (g - self.m[i]) * float(npd(1) - npd(self.b1))
            self.v[i] = self.v[i] + (g * g - self.v[i]) * float(npd(1) - npd(self.b2))
            # torch's vectorised fp32 sqrt on the CPU is not always correctly rounded (about 0.6 % of random inputs
            # are one ulp off); numpy's is, like the kernels' __fsqrt_rn (tests/test_learn_ref_host.py)
            sq = torch.from_numpy(np.sqrt(self.v[i].detach().numpy()))
            out.append(p - (self.m[i] * float(alpha)) / (sq + float(npd(self.eps))))
        self.b1p = npd(self.b1p * npd(self.b1))
        self.b2p = npd(self.b2p * npd(self.b2))
        return out


def dqn_learn_step(net, online, target, opt, batch, discount, huber_loss=True, double_dqn=False, clip=None,
                   world_scale=1.0, kink=None):
    """One learn_from_batch step.  batch: dict with states, next_states, actions, rewards, game_overs, weights (or None).
    Returns dict(loss, grads (named), grad_norm, td_errors, targets, new_params (named), q_online).
    kink: ReLU masks of the implementation under test for the differentiated forward pass (QNetOracle.forward)."""
    names = list(online.keys())
    params = [online[n].clone().requires_grad_(True) for n in names]
    pd = OrderedDict(zip(names, params))
    with torch.no_grad():
        q_next = net.forward(target, batch["next_states"])
        q_online_ng = net.forward(online, batch["states"])
        q_select = net.forward(online, batch["next_states"]) if double_dqn else q_next
    targets, td = dqn_targets(q_next.numpy(), q_select.numpy(), q_online_ng.numpy(), batch["actions"], batch["rewards"],
                              batch["game_overs"], discount)
    w = batch.get("weights")
    wt = _t(np.asarray(w, dtype=np.float64), net.dtype) if w is not None else None
    q = net.forward(pd, batch["states"], kink=kink)
    loss = q_head_loss(q, _t(targets, net.dtype), wt, huber_loss)
    grads = torch.autograd.grad(loss, params, allow_unused=True)
    grads = [g if g is not None else torch.zeros_like(p) for g, p in zip(grads, params)]
    gnorm = torch.sqrt(sum((g * g).sum() for g in grads))
    if clip:
        scale = clip / max(float(gnorm), clip)
        grads = [g * scale for g in grads]
    grads = [g * world_scale for g in grads] if world_scale != 1.0 else grads
    new_params = opt.step([p.detach() for p in params], grads)
    return dict(loss=float(loss.detach()), grads=OrderedDict(zip(names, [g.detach() for g in grads])),
                grad_norm=float(gnorm), td_errors=td, targets=targets,
                new_params=OrderedDict(zip(names, new_params)), q_online=q_online_ng.numpy(),
                q_next=q_next.numpy())


def polyak(target, online, rate, dtype=np.float32):
    """architecture.py:598-607 in numpy fp32: rate * new + (1 - rate) * old."""
    out = OrderedDict()
    for n in target:
        out[n] = dtype(rate) * np.asarray(online[n], dtype=dtype) + dtype(1 - rate) * np.asarray(target[n],
                                                                                                dtype=dtype)
    return out
