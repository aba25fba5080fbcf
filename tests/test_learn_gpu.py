"""GPU parity tests of the learn step (pytest -m gpu): CUDA kernels vs the torch-CPU oracle (oracle/nets.py).

Tolerance (north_star: "losses/gradients within 1e-5 rtol fp32"): every tensor is compared with
``|got - want| <= 1e-5 * max|want| + 1e-5 * |want|`` -- 1e-5 relative to the tensor's scale plus 1e-5 element-wise --
because two fp32 evaluations with different summation orders cannot agree to 1e-5 *element-wise* on entries that are
the result of cancellation.  In addition the CUDA result must be at least as close to an fp64 evaluation of the same
graph as the fp32 oracle is (factor 4 slack), which is the meaningful statement of "same result within fp32".
"""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import nets as on     # noqa: E402  (checker only)


def close(got, want, rtol=1e-5, name="", atol=0.0):
    got, want = np.asarray(got, dtype=np.float64), np.asarray(want, dtype=np.float64)
    scale = np.abs(want).max() if want.size else 0.0
    err = np.abs(got - want)
    tol = rtol * scale + rtol * np.abs(want) + atol
    assert np.all(err <= tol), "%s: max err %.3e (scale %.3e, allowed %.3e)" % (name, err.max(), scale, tol.min())


def _lib():
    from coach_b200 import _lib
    return _lib, _lib.load()


def _pixel_major(t, B, npix, ch):
    """NHWC-flattened [B, npix * ch] -> plane-matrix order [npix * B, ch]"""
    return t.reshape(B, npix, ch).permute(1, 0, 2).reshape(npix * B, ch)


def _check_planes(buf, t, B):
    """the planes a GEMM epilogue wrote for `t` reconstruct it exactly: hi + mid + lo == t bit for bit"""
    want = _pixel_major(t, B, buf.npix, buf.cols)
    assert torch.equal(buf.to_dense(), want), "planes do not reconstruct the fp32 output"


# ---- gather-GEMM primitive ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,K,N,act", [(512, 3136, 512, "relu"), (512, 512, 6, None), (32, 4, 256, "relu"),
                                       (64, 17, 64, "tanh"), (100, 23, 400, "relu"), (1, 5, 3, None),
                                       (512, 512, 512, "relu"), (128, 512, 64, None), (96, 64, 128, "tanh"),
                                       (64, 256, 32, "relu")])
@pytest.mark.parametrize("planes", [False, True])
def test_dense_forward_backward(B, K, N, act, planes):
    from coach_b200.architectures import tiled as tl
    from coach_b200.architectures.layers import Dense, Workspace
    L, lib = _lib()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(B * 7 + K)
    x = torch.randn(B, K, generator=g)
    w = torch.randn(K, N, generator=g) / np.sqrt(K)
    b = torch.randn(N, generator=g) * 0.1
    dy = torch.randn(B, N, generator=g)
    xd, wd, bd, dyd = x.to(dev), w.to(dev), b.to(dev), dy.to(dev)
    y = torch.empty(B, N, device=dev)
    flat = torch.empty(K * N + N, device=dev)          # bias gradient right behind the kernel gradient (ParamStore)
    dw, db, dx = flat[:K * N].view(K, N), flat[K * N:], torch.empty(B, K, device=dev)
    ws = Workspace(dev)
    layer = Dense(K, N, act)
    ctx = None
    if planes:          # pre-split operands (tiled bf16 planes next to every fp32 buffer): cb200_gemm_tiled
        if B % 32 or K % 8 or N % 8:
            pytest.skip("shape has no plane form")
        wp = tl.PlaneBuf(K, N, dev, interleaved=tl.b_interleaved(N)).load(lib, wd)
        ctx = tl.PlaneCtx(x=tl.PlaneBuf(B, K, dev).load(lib, xd), y=tl.PlaneBuf(B, N, dev),
                          dy=tl.PlaneBuf(B, N, dev).load(lib, dyd), dx=tl.PlaneBuf(B, K, dev), w_ptr=wp.ptr,
                          w_stride=wp.stride)
    layer.prepare(lib, ws, B, dev, xd, y, wd, bd, dw, db, dyd, dx, need_dx=True, prev_act=1,   # relu'(x) mask on dx
                  planes=ctx)
    if planes and tl.width_ok(N) and tl.channels_ok(K):
        assert layer.tiled_x
    layer.forward()
    layer.backward()
    torch.cuda.synchronize()
    if planes:
        _check_planes(ctx.y, y, B), _check_planes(ctx.dx, dx, B)
    x64, w64, b64, dy64 = x.double(), w.double(), b.double(), dy.double()
    f = {"relu": torch.relu, "tanh": torch.tanh, None: lambda t: t}[act]
    close(y.cpu(), f(x64 @ w64 + b64), name="y")
    close(dw.cpu(), x64.t() @ dy64, name="dw")
    close(db.cpu(), dy64.sum(0), name="db")
    close(dx.cpu(), (dy64 @ w64.t()) * (x64 > 0), name="dx")


@pytest.mark.parametrize("B,H,C,N,K,S,u8", [(8, 84, 4, 32, 8, 4, True), (8, 20, 32, 64, 4, 2, False),
                                            (8, 9, 64, 64, 3, 1, False), (3, 11, 3, 5, 3, 2, False),
                                            (2, 10, 2, 7, 4, 3, False), (32, 84, 4, 32, 8, 4, True),
                                            (160, 20, 32, 64, 4, 2, False), (64, 9, 64, 64, 3, 1, False),
                                            (32, 7, 128, 32, 3, 2, False),
                                            # the three conv layers of the Atari network at the BENCHMARKED batch size
                                            (512, 84, 4, 32, 8, 4, True), (512, 20, 32, 64, 4, 2, False),
                                            (512, 9, 64, 64, 3, 1, False)])
@pytest.mark.parametrize("planes", [False, True])
def test_conv_forward_backward(B, H, C, N, K, S, u8, planes):
    if B >= 512 and not planes:
        pytest.skip("B = 512 runs on the plane path (the plane-less form is covered at the smaller batch sizes)")
    from coach_b200.architectures import tiled as tl
    from coach_b200.architectures.layers import Conv2d, Workspace
    from coach_b200.architectures.network import make_u8_lut
    import torch.nn.functional as F
    L, lib = _lib()
    dev = torch.device("cuda")
    g = torch.Generator().manual_seed(H * 31 + C)
    layer = Conv2d((H, H), C, N, K, S, "relu")
    OH = layer.OH
    if u8:
        x = torch.randint(0, 256, (B, H, H, C), generator=g, dtype=torch.uint8)
        xf = x.double() / 255.0
    else:
        x = torch.relu(torch.randn(B, H, H, C, generator=g))
        xf = x.double()
    w = torch.randn(K, K, C, N, generator=g) / np.sqrt(K * K * C)
    b = torch.randn(N, generator=g) * 0.1
    dy = torch.randn(B, OH, OH, N, generator=g)
    xd, wd, bd, dyd = x.to(dev), w.to(dev), b.to(dev), dy.to(dev)
    y = torch.empty(B, OH * OH * N, device=dev)
    flat = torch.empty(K * K * C * N + N, device=dev)  # bias gradient right behind the kernel gradient (ParamStore)
    dw, db = flat[:K * K * C * N].view(K, K, C, N), flat[K * K * C * N:]
    dx = torch.empty(B, H * H * C, device=dev)
    ws = Workspace(dev)
    ctx = None
    if planes:
        if B % 32 or C % 4 or N % 8:
            pytest.skip("shape has no plane form")
        wp = tl.PlaneBuf(K * K * C, N, dev, interleaved=tl.b_interleaved(N)).load(lib, wd)
        xp = None if u8 else tl.PlaneBuf(H * H * B, C, dev, npix=H * H).load(lib, _pixel_major(xd, B, H * H, C))
        ctx = tl.PlaneCtx(x=xp, y=tl.PlaneBuf(OH * OH * B, N, dev, npix=OH * OH),
                          dy=tl.PlaneBuf(OH * OH * B, N, dev, npix=OH * OH).load(lib, _pixel_major(dyd, B, OH * OH, N)),
                          dx=None if u8 else tl.PlaneBuf(H * H * B, C, dev, npix=H * H), w_ptr=wp.ptr,
                          w_stride=wp.stride)
    layer.prepare(lib, ws, B, dev, xd, y, wd, bd, dw, db, dyd, dx, x_is_u8=u8, lut=make_u8_lut(dev) if u8 else None,
                  need_dx=not u8, prev_act=0 if u8 else 1, planes=ctx)
    if planes and not u8:
        assert layer.bwd_x is not None                      # the multi-tap tensor-core path was taken
    layer.forward()
    layer.backward()
    torch.cuda.synchronize()
    if planes:
        _check_planes(ctx.y, y, B)
        if not u8:
            _check_planes(ctx.dx, dx, B)
    xt = xf.permute(0, 3, 1, 2).clone().requires_grad_(True)
    wt = w.double().permute(3, 2, 0, 1).clone().requires_grad_(True)
    bt = b.double().clone().requires_grad_(True)
    z = F.conv2d(xt, wt, bt, stride=S)
    close(y.cpu().view(B, OH, OH, N), torch.relu(z).permute(0, 2, 3, 1).detach(), name="y")
    # gradient wrt the pre-activation z with upstream dy
    z.backward(dy.double().permute(0, 3, 1, 2))
    close(dw.cpu(), wt.grad.permute(2, 3, 1, 0), name="dw")
    close(db.cpu(), bt.grad, name="db")
    if not u8:
        want_dx = xt.grad.permute(0, 2, 3, 1) * (xf > 0)
        close(dx.cpu().view(B, H, H, C), want_dx, name="dx")


# ---- element-wise kernels ------------------------------------------------------------------------------------------
def test_adam_polyak_clip_match_numpy_fp32():
    L, lib = _lib()
    dev = torch.device("cuda")
    n = 100003
    rng = np.random.RandomState(0)
    theta = rng.randn(n).astype(np.float32)
    g = (rng.randn(n) * 0.01).astype(np.float32)
    th, m, v = torch.from_numpy(theta).to(dev), torch.zeros(n, device=dev), torch.zeros(n, device=dev)
    gd = torch.from_numpy(g).to(dev)
    opt = on.AdamTF([torch.from_numpy(theta)], 2.5e-4, 0.9, 0.99, 1e-4)
    cur = [torch.from_numpy(theta)]
    b1p, b2p = np.float32(0.9), np.float32(0.99)
    for step in range(3):
        L.check(lib.cb200_adam_tf(th.data_ptr(), m.data_ptr(), v.data_ptr(), gd.data_ptr(), n, 2.5e-4, 0.9, 0.99, 1e-4,
                                  float(b1p), float(b2p), None))
        b1p, b2p = np.float32(b1p * np.float32(0.9)), np.float32(b2p * np.float32(0.99))
        cur = opt.step(cur, [torch.from_numpy(g)])
        np.testing.assert_allclose(th.cpu().numpy(), cur[0].numpy(), rtol=2e-6, atol=1e-7)
    # polyak: exact fp32 arithmetic
    tgt = rng.randn(n).astype(np.float32)
    td = torch.from_numpy(tgt).to(dev)
    L.check(lib.cb200_polyak(td.data_ptr(), th.data_ptr(), n, 0.005, None))
    want = np.float32(0.005) * th.cpu().numpy() + np.float32(1 - 0.005) * tgt
    np.testing.assert_array_equal(td.cpu().numpy(), want)
    L.check(lib.cb200_polyak(td.data_ptr(), th.data_ptr(), n, 1.0, None))
    np.testing.assert_array_equal(td.cpu().numpy(), th.cpu().numpy())
    # global norm + clip
    ss = torch.zeros(1, device=dev)
    wsb = torch.empty(2048, device=dev)
    L.check(lib.cb200_sumsq(gd.data_ptr(), n, ss.data_ptr(), wsb.data_ptr(), None))
    np.testing.assert_allclose(ss.item(), np.sum(g.astype(np.float64) ** 2), rtol=1e-6)
    g2 = gd.clone()
    L.check(lib.cb200_clip_by_global_norm(g2.data_ptr(), n, ss.data_ptr(), 0.5, None))
    norm = np.sqrt(np.sum(g.astype(np.float64) ** 2))
    np.testing.assert_allclose(g2.cpu().numpy(), g * (0.5 / max(norm, 0.5)), rtol=1e-6)


def test_td_targets_match_python_loop():
    L, lib = _lib()
    dev = torch.device("cuda")
    rng = np.random.RandomState(1)
    B, A = 512, 6
    qn = rng.randn(B, A).astype(np.float32)
    qs = rng.randn(B, A).astype(np.float32)
    qs[3, 2] = qs[3, 4] = qs[3].max() + 1          # tie: first maximum wins
    qo = rng.randn(B, A).astype(np.float32)
    act = rng.randint(0, A, B).astype(np.int64)
    rew = rng.randint(-1, 2, B).astype(np.float64)
    done = (rng.rand(B) < 0.2)
    want_t, want_e = on.dqn_targets(qn, qs, qo, act, rew, done, 0.99)
    out_t = torch.empty(B, A, device=dev)
    out_e = torch.empty(B, dtype=torch.float64, device=dev)
    keep = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (qn, qs, qo, act, rew, done.astype(np.uint8))]
    L.check(lib.cb200_dqn_td_targets(keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), keep[3].data_ptr(),
                                     keep[4].data_ptr(), keep[5].data_ptr(), 0.99, B, A,
                                     out_t.data_ptr(), out_e.data_ptr(), None))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(out_t.cpu().numpy(), want_t)       # bit-exact: same fp64 operations, one rounding
    np.testing.assert_array_equal(out_e.cpu().numpy(), want_e)


# ---- whole learn step ----------------------------------------------------------------------------------------------
def _make_agent(obs_shape, A, B, dueling, double, per, clip=None, huber=True, seed=0, middleware=True):
    from coach_b200.agents.dqn_agent import DQNAgent, DDQNAgent, DQNAgentParameters
    from coach_b200.memories.memory import MemoryGranularity
    from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplayParameters
    from coach_b200.schedules import LinearSchedule
    ap = DQNAgentParameters()
    if per:
        ap.memory = PrioritizedExperienceReplayParameters()
        ap.memory.beta = LinearSchedule(0.4, 1, 1000)
    ap.memory.max_size = (MemoryGranularity.Transitions, 1024)
    net = ap.network_wrappers["main"]
    net.batch_size = B
    net.replace_mse_with_huber_loss = huber
    net.clip_gradients = clip
    if dueling:
        net.heads_parameters = ["DuelingQHead"]
    if not middleware:
        from coach_b200.base_parameters import MiddlewareScheme
        net.middleware_parameters.scheme = MiddlewareScheme.Empty
    cls = DDQNAgent if double else DQNAgent
    return cls(ap, observation_shape=obs_shape, num_actions=A, seed=seed)


def _device_relu_masks(agent):
    """[y > 0] of every ReLU of the differentiated forward pass (online network on s), in the oracle's evaluation order
    and tensor layout (conv maps [B, C, H, W], dense [B, K])"""
    inst = agent.networks["main"].online_s
    nd = agent.net_def
    B = agent.batch_size

    def of(seq_inst, i):
        layer = seq_inst.layers[i]
        pb = seq_inst.act_planes[i]
        if pb is not None:
            d = pb.to_dense() > 0                                        # [npix * B, C], rows pixel * B + b
            if pb.npix == 1:
                return d.cpu()
            return d.reshape(layer.OH, layer.OW, B, layer.N).permute(2, 3, 0, 1).contiguous().cpu()
        a = seq_inst.acts[i] > 0                                         # fp32 [B, npix * C] NHWC
        if hasattr(layer, "OH"):
            return a.reshape(B, layer.OH, layer.OW, layer.N).permute(0, 3, 1, 2).contiguous().cpu()
        return a.cpu()

    n_relu_trunk = len(inst.trunk.layers) - (0 if nd.dueling else 1)
    masks = [of(inst.trunk, i) for i in range(n_relu_trunk)]
    if nd.dueling:
        masks += [of(inst.v, 0), of(inst.a, 0)]
    return masks


@pytest.mark.parametrize("cfg", [
    dict(obs=(4,), A=2, B=32, dueling=False, double=False, per=False, huber=False, clip=None),       # CartPole_DQN
    dict(obs=(84, 84, 4), A=6, B=16, dueling=False, double=False, per=True, huber=True, clip=None),  # Atari DQN + PER
    dict(obs=(84, 84, 4), A=6, B=8, dueling=True, double=True, per=True, huber=True, clip=10.0),     # dueling DDQN + PER
    dict(obs=(84, 84, 4), A=6, B=128, dueling=False, double=True, per=True, huber=True, clip=None),  # bf16-plane path
    # BASELINE config 5 (presets/Atari_Dueling_DDQN_with_PER_OpenAI.py:17-19): towers on the conv map, clip-norm 10
    dict(obs=(84, 84, 4), A=6, B=8, dueling=True, double=True, per=True, huber=True, clip=10.0, middleware=False),
    dict(obs=(84, 84, 4), A=6, B=128, dueling=True, double=True, per=True, huber=True, clip=10.0, middleware=False),
    # the BENCHMARKED batch size, whole step: BASELINE config 2 (DQN + PER), DDQN, and config 5
    dict(obs=(84, 84, 4), A=6, B=512, dueling=False, double=False, per=True, huber=True, clip=None),
    dict(obs=(84, 84, 4), A=6, B=512, dueling=False, double=True, per=True, huber=True, clip=None),
    dict(obs=(84, 84, 4), A=6, B=512, dueling=True, double=True, per=True, huber=True, clip=10.0, middleware=False),
], ids=lambda c: "%s%s%s_B%d%s" % ("dueling_" if c["dueling"] else "", "ddqn" if c["double"] else "dqn",
                                   "_per" if c["per"] else "", c["B"], "" if c.get("middleware", True) else "_nomw"))
def test_dqn_learn_step_matches_oracle(cfg):
    import random
    torch.manual_seed(0)
    mw = cfg.get("middleware", True)
    agent = _make_agent(cfg["obs"], cfg["A"], cfg["B"], cfg["dueling"], cfg["double"], cfg["per"], cfg["clip"],
                        cfg["huber"], middleware=mw)
    if not mw and cfg["dueling"] and len(cfg["obs"]) == 3:
        assert agent.net_def.store.num_params() - 1 == 3293863          # SURVEY section 8d, config 5
        assert agent.networks["main"].online_s.towers_on_planes == (cfg["B"] >= 128)
    B, A = cfg["B"], cfg["A"]
    rng = np.random.RandomState(3)
    n = max(256, 2 * B)
    if len(cfg["obs"]) == 3:
        s = rng.randint(0, 256, (n,) + cfg["obs"]).astype(np.uint8)
        s2 = rng.randint(0, 256, (n,) + cfg["obs"]).astype(np.uint8)
    else:
        s = rng.uniform(-1, 1, (n,) + cfg["obs"]).astype(np.float32)
        s2 = rng.uniform(-1, 1, (n,) + cfg["obs"]).astype(np.float32)
    a = rng.randint(0, A, n).astype(np.int64)
    r = rng.randint(-1, 2, n).astype(np.float64)
    done = (rng.rand(n) < 0.1).astype(np.uint8)
    agent.memory.store_columns({"state:observation": s, "next_state:observation": s2, "action": a, "reward": r,
                                "game_over": done})
    if cfg["per"]:
        agent.memory.update_priorities(np.arange(n), np.abs(rng.randn(n)))
    store = agent.net_def.store
    # make target != online so that the test can tell them apart
    net = agent.networks["main"]
    net.theta_target.copy_(store.theta * 0.9 + 0.01)
    net.target_changed()                     # a direct write to the target parameters: re-derive their operand planes
    oracle32 = on.QNetOracle(cfg["obs"], A, cfg["dueling"], torch.float32, middleware=mw)
    oracle64 = on.QNetOracle(cfg["obs"], A, cfg["dueling"], torch.float64, middleware=mw)
    results = {}
    fp64_clause = []          # tensors for which the 1e-5 rule was replaced by the fp64-distance clause
    for step in range(2):
        online_named = store.export_named()
        target_named = store.export_named(net.theta_target)
        random.seed(10 + step)
        np.random.seed(10 + step)
        batch = agent.sample_batch()
        if step == 0:
            opt32 = on.AdamTF([torch.from_numpy(v) for v in online_named.values()], 2.5e-4, 0.9, 0.99, 1e-4)
        loss, losses, gnorm = agent.learn_from_batch(batch)
        torch.cuda.synchronize()
        # (read after the step: on the fused input path the frames reach the network as operand planes and the uint8
        # columns are gathered on demand from the drawn slots)
        for k in ("state:observation", "next_state:observation"):
            batch.column(k)
        cols = {k: v.cpu().numpy() for k, v in batch.columns.items()}
        ob = dict(states=cols["state:observation"], next_states=cols["next_state:observation"],
                  actions=cols["action"], rewards=cols["reward"], game_overs=cols["game_over"].astype(bool),
                  weights=cols["weight32"] if cfg["per"] else None)
        # ReLU kink rule: where a pre-activation is within 1e-5 of zero (relative to the layer's scale) either
        # derivative is a valid fp32 result; there the oracle takes the device's choice (and nowhere else: "hard"
        # disagreements are failures).  One flipped element out of 1.6 M moves a conv weight gradient -- a sum of
        # 25,000 cancelling terms -- by 1e-3, so without the rule the comparison is a coin toss at batch 512.
        masks = _device_relu_masks(agent)
        k32, k64 = dict(masks=masks, tol=1e-5), dict(masks=masks, tol=1e-5)
        ref = on.dqn_learn_step(oracle32, oracle32.cast(online_named), oracle32.cast(target_named), opt32, ob, 0.99,
                                cfg["huber"], cfg["double"], cfg["clip"], kink=k32)
        opt64 = on.AdamTF([torch.from_numpy(v).double() for v in online_named.values()], 2.5e-4, 0.9, 0.99, 1e-4,
                          dtype=torch.float64)
        ref64 = on.dqn_learn_step(oracle64, oracle64.cast(online_named), oracle64.cast(target_named), opt64, ob, 0.99,
                                  cfg["huber"], cfg["double"], cfg["clip"], kink=k64)
        assert k32.get("hard", 0) == 0 and k64.get("hard", 0) == 0, "ReLU masks differ away from the kink"
        print("[relu-kink] step %d: %d element(s) within 1e-5 of zero took the device's derivative" %
              (step, k64.get("flipped", 0)))
        close(net.online_s.q.cpu().numpy(), ref["q_online"], name="q_online")
        close(agent.targets.cpu().numpy(), ref["targets"], name="targets")
        close(agent.td_err.cpu().numpy(), ref["td_errors"], name="td_errors")
        close(loss, ref["loss"], name="loss")
        close(gnorm, ref["grad_norm"], name="grad_norm")
        got_grads = store.export_named(store.grad)
        for name in ref["grads"]:
            want = ref["grads"][name].numpy()
            # distance to the fp64 evaluation of the same graph: ours, and the fp32 oracle's own
            e_ours = np.abs(got_grads[name] - ref64["grads"][name].numpy()).max()
            e_orc = np.abs(want - ref64["grads"][name].numpy()).max()
            try:
                close(got_grads[name], want, name="grad " + name)
            except AssertionError as exc:
                # A weight gradient is a sum over batch x pixels of terms of either sign (51200 for conv1 at B = 128):
                # two fp32 evaluations differ by the rounding noise of that ill-conditioned sum, which can exceed
                # 1e-5 of the result.  The 1e-5 rule is then replaced by: at least as close to the fp64 value as
                # the fp32 oracle itself is.
                assert e_ours <= e_orc, "%s; vs fp64: ours %.3e, fp32 oracle %.3e" % (exc, e_ours, e_orc)
                fp64_clause.append("step %d grad %s (vs fp64: ours %.2e, fp32 oracle %.2e)" % (step, name, e_ours, e_orc))
            # always: closer to (or as close as) the fp32 oracle is to the fp64 evaluation, with slack 4
            assert e_ours <= 4 * e_orc + 2e-6 * (np.abs(want).max() + 1e-30), (name, e_ours, e_orc)
        got_params = store.export_named()
        for name in ref["new_params"]:
            want = ref["new_params"][name].numpy()
            try:
                close(got_params[name], want, name="param " + name)
            except AssertionError as exc:
                # Adam normalises the gradient, so the relative rounding noise of an ill-conditioned gradient sum
                # (see above) shows up unchanged in the first steps of a parameter: same fp64 clause
                w64 = ref64["new_params"][name].numpy()
                e_ours, e_orc = np.abs(got_params[name] - w64).max(), np.abs(want - w64).max()
                assert e_ours <= 2 * e_orc, "%s; vs fp64: ours %.3e, fp32 oracle %.3e" % (exc, e_ours, e_orc)
                fp64_clause.append("step %d param %s (vs fp64: ours %.2e, fp32 oracle %.2e)" % (step, name, e_ours, e_orc))
        results[step] = loss
    # which tensors needed the fp64 clause instead of 1e-5 (printed with pytest -s / -rA)
    print("[fp64-clause] %s: %s" % (cfg, "; ".join(fp64_clause) if fp64_clause else "none"))
    # PER priorities were updated with the pre-update TD errors of the last batch (value_optimization_agent.py:74-80)
    if cfg["per"]:
        from oracle import memory as om
        idx = cols["idx"]
        leaves = agent.memory.sum_tree.cpu().numpy()[agent.memory.power_of_2_size - 1:]
        td = agent.td_err.cpu().numpy()
        last = {int(i): k for k, i in enumerate(idx)}       # last writer wins
        for i, k in last.items():
            assert leaves[i] == (td[k] + 1e-6) ** 0.6


def test_target_network_cadence_and_polyak():
    from coach_b200.base_parameters import TrainingSteps
    agent = _make_agent((4,), 2, 8, False, False, False)
    agent.ap.algorithm.num_steps_between_copying_online_weights_to_target = TrainingSteps(3)
    agent.ap.algorithm.num_consecutive_playing_steps.num_steps = 1
    rng = np.random.RandomState(0)
    n = 64
    agent.memory.store_columns({"state:observation": rng.randn(n, 4).astype(np.float32),
                                "next_state:observation": rng.randn(n, 4).astype(np.float32),
                                "action": rng.randint(0, 2, n).astype(np.int64), "reward": rng.randn(n),
                                "game_over": np.zeros(n, np.uint8)})
    net = agent.networks["main"]
    synced = []
    for step in range(7):
        agent.total_steps_counter += 1
        agent.train()
        synced.append(bool(torch.equal(net.theta, net.theta_target)))
    assert synced == [False, False, True, False, False, True, False]


def test_dqn_graph_replay_matches_eager(monkeypatch):
    """the CUDA-graph replay of the learn step (agents/dqn_agent.py) is bit-identical to the eager launch sequence"""
    import random
    results = []
    for graph in (0, 1):
        monkeypatch.setenv("CB200_DQN_GRAPH", str(graph))
        torch.manual_seed(0)
        agent = _make_agent((84, 84, 4), 6, 128, False, True, True, None, True, seed=5)
        assert agent.use_graph == bool(graph)
        rng = np.random.RandomState(3)
        n = 512
        agent.memory.store_columns({
            "state:observation": rng.randint(0, 256, (n, 84, 84, 4)).astype(np.uint8),
            "next_state:observation": rng.randint(0, 256, (n, 84, 84, 4)).astype(np.uint8),
            "action": rng.randint(0, 6, n).astype(np.int64), "reward": rng.randint(-1, 2, n).astype(np.float64),
            "game_over": (rng.rand(n) < 0.1).astype(np.uint8)})
        agent.memory.update_priorities(np.arange(n), np.abs(rng.randn(n)))
        losses = []
        for step in range(6):                       # 2 eager steps, capture, 3 replays
            random.seed(20 + step)
            np.random.seed(20 + step)
            batch = agent.sample_batch()
            loss, _, _ = agent.learn_from_batch(batch)
            losses.append(loss)
        torch.cuda.synchronize()
        if graph:
            assert agent._graphs is not None and agent.graph_kernel_launches > 0
        store = agent.net_def.store
        results.append((losses, store.theta.clone(), agent.memory.sum_tree.clone()))
    assert results[0][0] == results[1][0]
    assert torch.equal(results[0][1], results[1][1])
    assert torch.equal(results[0][2], results[1][2])


@pytest.mark.parametrize("E", [16, 128])
def test_acting_path_batched_q_values_and_e_greedy(E):
    """DQNAgent.choose_actions: the batched online-network forward equals the oracle's Q-values and the actions are the
    epsilon-greedy policy's on those values (the policy itself is pinned to the reference in tests/test_acting.py)"""
    from coach_b200.exploration_policies.e_greedy import BatchedEGreedy
    from coach_b200.schedules import ConstantSchedule
    agent = _make_agent((84, 84, 4), 6, 128, False, False, True)
    rng = np.random.RandomState(E)
    states = rng.randint(0, 256, (E, 84, 84, 4)).astype(np.uint8)
    np.random.seed(3)
    pol = BatchedEGreedy(6, E, ConstantSchedule(0.25), 0.05)
    actions, q = agent.choose_actions(states, pol)
    oracle = on.QNetOracle((84, 84, 4), 6, False, torch.float64)
    want = oracle.forward(oracle.cast(agent.net_def.store.export_named()), states).numpy()
    close(q, want, name="acting Q-values")
    np.random.seed(3)
    pol2 = BatchedEGreedy(6, E, ConstantSchedule(0.25), 0.05)
    want_actions, _ = pol2.get_actions(q)
    np.testing.assert_array_equal(actions, want_actions)
    greedy = ~(np.array([a != int(np.argmax(q[e])) for e, a in enumerate(actions)]))
    assert greedy.mean() > 0.5                      # epsilon 0.25: most actions are the arg-max
    # the weights change -> so do the acting Q-values (the acting network reads the live parameters)
    agent.net_def.store.theta.mul_(1.01)
    agent.networks["main"].online_changed()
    q2 = agent.get_all_q_values_for_states(states).cpu().numpy()
    assert np.abs(q2 - q).max() > 0
