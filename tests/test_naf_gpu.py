"""NAF on the GPU.

  cb200_naf_head at the C ABI, A in {1, 2, 3, 6, 17, 32} x B in {1, 31, 32, 256, 4096}:
    exact probes (u = mu: adv = 0, Q = V, zero d_l / d_zmu; l = 0 (L = I) with dyadic d: adv = -|d|^2 / 2 bit for bit),
    random data against fp64 -- d_zv bit for bit given the kernel's Q, every other output within gamma_n S where S is
    the same expression evaluated on absolute values (the observed e / S is printed) --, canaries after every output,
    repeat calls with identical bits, acting mode leaving the gradient buffers alone, argument errors, and a final
    check that both instantiations ran;
  cb200_clip_by_value against numpy (+-clip, +-inf, NaN);
  NAFAgent learn steps against oracle/naf.py (three steps from desynchronised targets, clipping active and inactive),
  graph replay against eager steps, the train() driver, acting, checkpoints and two ranks.
Reads tests/golden/naf.npz only through the host-pinned oracle and exploration policy."""
import ctypes
import functools
import os
import random
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from oracle import naf as onaf         # noqa: E402  (checker only)
from oracle.actor_critic import make_adam
from oracle.nets import polyak
from oracle.rl_math import ac_td_targets
from test_learn_gpu import close           # noqa: E402

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
RAN = set()
GUARD = 64
CANARY = 0x7FA5A5A5


def gamma(n):
    return n * U32 / (1.0 - n * U32)


def _lib():
    from coach_b200 import _lib as L
    return L, L.load()


class Outs(object):
    """fp32 device outputs, each followed by GUARD canary elements"""

    def __init__(self):
        self.t = {}

    def add(self, name, n):
        full = torch.empty(n + GUARD, dtype=torch.float32, device="cuda")
        full.view(torch.int32).fill_(CANARY)
        self.t[name] = (full, n)
        return full.data_ptr()

    def numpy(self):
        torch.cuda.synchronize()
        out = {}
        for k, (full, n) in self.t.items():
            tail = full[n:].view(torch.int32).cpu().numpy()
            assert (tail == np.int32(CANARY)).all(), "%s: write past its end" % k
            out[k] = full[:n].cpu().numpy()
        return out


def run_head(d, huber=False, train=True, grad_canaries=False):
    """d: dict of numpy inputs (z_v [B], z_mu [B, A], l [B, nl], scale [A], u [B, A], y [B]).  Returns the outputs."""
    L, lib = _lib()
    B, A = d["z_mu"].shape
    nl = A * (A + 1) // 2
    keep = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).cuda() for k, v in d.items()}
    o = Outs()
    desc = L.NafHeadDesc()
    desc.z_v, desc.z_mu, desc.l, desc.scale = (keep[k].data_ptr() for k in ("z_v", "z_mu", "l", "scale"))
    desc.huber, desc.batch, desc.n_actions, desc.ld_mu, desc.ld_l, desc.ld_actions = int(huber), B, A, A, nl, A
    desc.mu, desc.q = o.add("mu", B * A), o.add("q", B)
    if train or grad_canaries:
        desc.loss, desc.d_zv, desc.d_zmu, desc.d_l, desc.adv = (o.add("loss", 1), o.add("d_zv", B),
                                                                 o.add("d_zmu", B * A), o.add("d_l", B * nl),
                                                                 o.add("adv", B))
    if train:
        desc.actions, desc.targets = keep["u"].data_ptr(), keep["y"].data_ptr()
    L.check(lib.cb200_naf_head(ctypes.byref(desc), L.current_stream()))
    RAN.add(train)
    r = o.numpy()
    r["mu"] = r["mu"].reshape(B, A)
    for k, shape in (("d_zmu", (B, A)), ("d_l", (B, nl))):
        if k in r:
            r[k] = r[k].reshape(shape)
    return r


def random_data(A, B, seed=0):
    rng = np.random.RandomState(seed + 1000 * A + B)
    nl = A * (A + 1) // 2
    f = np.float32
    return dict(z_v=(rng.randn(B) * 3).astype(f), z_mu=(rng.randn(B, A) * 1.5).astype(f),
                l=(rng.randn(B, nl) * 0.7).astype(f), scale=rng.uniform(0.5, 3.0, A).astype(f),
                u=rng.uniform(-3, 3, (B, A)).astype(f), y=(rng.randn(B) * 4).astype(f))


def ref64(d, q_kernel, huber):
    """fp64 evaluation of the head and, for the bounds, the same expressions on absolute values.  dL/dQ is the fp32
    expression on the kernel's Q (checked bit for bit separately)."""
    B, A = d["z_mu"].shape
    f64 = lambda k: np.asarray(d[k], np.float64)      # noqa: E731
    zv, zmu, lv, scale, u, y = (f64(k) for k in ("z_v", "z_mu", "l", "scale", "u", "y"))
    t = np.tanh(zmu)
    mu = t * scale
    dd = u - mu
    Lm = np.zeros((B, A, A))
    i = 0
    for c in range(A):
        Lm[:, c, c] = np.exp(lv[:, i])
        Lm[:, c + 1:, c] = lv[:, i + 1:i + A - c]
        i += A - c
    w = np.einsum("brc,br->bc", Lm, dd)
    adv = -0.5 * (w * w).sum(1)
    q = zv + adv
    dq = dq32(q_kernel, d["y"], huber, B).astype(np.float64)
    lw = np.einsum("brc,bc->br", Lm, w)
    d_zmu = dq[:, None] * lw * scale * (1 - t * t)
    G = -dd[:, :, None] * w[:, None, :] * dq[:, None, None]             # dQ/dL[r, c] times dL/dQ
    for c in range(A):
        G[:, c, c] *= Lm[:, c, c]
    d_l = np.concatenate([G[:, c:, c] for c in range(A)], axis=1)
    # absolute-value versions: |d| through |u| + |mu| (the subtraction's operands)
    aL, ad = np.abs(Lm), np.abs(u) + np.abs(mu)
    aw = np.einsum("brc,br->bc", aL, ad)
    S_adv = 0.5 * (aw * aw).sum(1)
    S_q = np.abs(zv) + S_adv
    S_dzmu = np.abs(dq)[:, None] * np.einsum("brc,bc->br", aL, aw) * scale * (1 + t * t)
    SG = ad[:, :, None] * aw[:, None, :] * np.abs(dq)[:, None, None]
    for c in range(A):
        SG[:, c, c] *= aL[:, c, c]
    S_dl = np.concatenate([SG[:, c:, c] for c in range(A)], axis=1)
    return dict(mu=mu, q=q, adv=adv, d_zmu=d_zmu, d_l=d_l, S_q=S_q, S_adv=S_adv, S_dzmu=S_dzmu, S_dl=S_dl,
                S_mu=np.abs(mu))


def loss_terms32(q, y, huber):
    e = (np.asarray(q, np.float32) - np.asarray(y, np.float32)).astype(np.float32)
    if huber:
        ae = np.abs(e)
        qq = np.minimum(ae, np.float32(1))
        return (np.float32(0.5) * qq * qq + (ae - qq)).astype(np.float32), \
            np.where(ae <= 1, e, np.sign(e)).astype(np.float32)
    return (e * e).astype(np.float32), (np.float32(2) * e).astype(np.float32)


def dq32(q, y, huber, B):
    _, g = loss_terms32(q, y, huber)
    return (np.float32(1.0) / np.float32(B) * g).astype(np.float32)


def check(name, got, ref, S, n, report):
    got, ref, S = (np.asarray(x, np.float64) for x in (got, ref, S))
    err = np.abs(got - ref)
    bound = gamma(n) * S
    bad = err > bound
    assert not bad.any(), "%s: %d elements beyond gamma_%d S, worst err %.3e bound %.3e" % (
        name, bad.sum(), n, err[bad].max(), bound[bad][np.argmax(err[bad])])
    report.append("%-6s n=%-3d max e/S = %.2e (gamma_n = %.2e)" % (name, n, float((err / np.maximum(S, 1e-300)).max()),
                                                                    gamma(n)))


CASES = [(A, B) for A in (1, 2, 3, 6, 17, 32) for B in (1, 31, 32, 256, 4096)]


@pytest.mark.parametrize("A,B", CASES)
@pytest.mark.parametrize("huber", [False, True])
def test_naf_head_random_against_fp64(A, B, huber):
    d = random_data(A, B)
    r = run_head(d, huber)
    ref = ref64(d, r["q"], huber)
    # dL/dQ: the fp32 expression on the kernel's Q, bit for bit
    np.testing.assert_array_equal(r["d_zv"].view(np.uint32), dq32(r["q"], d["y"], huber, B).view(np.uint32))
    report = []
    check("mu", r["mu"], ref["mu"], ref["S_mu"], 6, report)                   # tanhf (2 ulp) and the scale
    check("q", r["q"], ref["q"], ref["S_q"], 2 * A + 16, report)
    check("adv", r["adv"], ref["adv"], ref["S_adv"], 2 * A + 16, report)
    check("d_zmu", r["d_zmu"], ref["d_zmu"], ref["S_dzmu"], 3 * A + 16, report)
    check("d_l", r["d_l"], ref["d_l"], ref["S_dl"], 2 * A + 16, report)
    lt, _ = loss_terms32(r["q"], d["y"], huber)
    lsum = lt.astype(np.float64).sum()
    check("loss", r["loss"], [lsum / B], [lsum / B], int(np.log2(max(B, 2))) + B // 256 + 4, report)
    print("A=%d B=%d huber=%d: %s" % (A, B, huber, "; ".join(report)))
    again = run_head(d, huber)
    for k in r:
        np.testing.assert_array_equal(r[k].view(np.uint32), again[k].view(np.uint32), err_msg="repeat: " + k)


@pytest.mark.parametrize("A,B", CASES)
def test_naf_head_exact_probes(A, B):
    d = random_data(A, B, seed=7)
    # u = mu (the acting mode's own mu): d = 0, adv = 0, Q = V, no gradient into mu or l
    act = run_head(d, train=False)
    np.testing.assert_array_equal(act["q"].view(np.uint32), d["z_v"].view(np.uint32))
    d["u"] = act["mu"]
    r = run_head(d)
    np.testing.assert_array_equal(r["mu"].view(np.uint32), act["mu"].view(np.uint32))
    assert (r["adv"] == 0).all()
    np.testing.assert_array_equal(r["q"].view(np.uint32), d["z_v"].view(np.uint32))
    assert (r["d_l"] == 0).all() and (r["d_zmu"] == 0).all()
    # l = 0: L = I; z_mu = 0: mu = 0, d = u dyadic -> adv = -|u|^2 / 2 exactly, and so Q = V + adv for dyadic V
    rng = np.random.RandomState(A * 31 + B)
    d.update(l=np.zeros_like(d["l"]), z_mu=np.zeros_like(d["z_mu"]),
             u=(rng.randint(-16, 17, (B, A)) / 8.0).astype(np.float32),
             z_v=(rng.randint(-64, 65, B) / 4.0).astype(np.float32))
    r = run_head(d)
    want_adv = (-0.5 * (d["u"].astype(np.float64) ** 2).sum(1)).astype(np.float32)
    np.testing.assert_array_equal(r["adv"], want_adv)
    np.testing.assert_array_equal(r["q"], (d["z_v"] + want_adv).astype(np.float32))
    assert (r["mu"] == 0).all()


@pytest.mark.parametrize("A", [1, 6, 32])
def test_naf_head_acting_mode_leaves_gradients_alone(A):
    d = random_data(A, 64, seed=3)
    r = run_head(d, train=False, grad_canaries=True)
    for k in ("loss", "d_zv", "d_zmu", "d_l", "adv"):
        assert (r[k].view(np.int32) == np.int32(CANARY)).all(), k
    np.testing.assert_allclose(r["mu"], np.tanh(d["z_mu"].astype(np.float64)) * d["scale"], rtol=4e-7, atol=1e-7)


def test_naf_head_argument_errors():
    L, lib = _lib()
    x = torch.zeros(1 << 16, device="cuda")
    p = x.data_ptr()

    def desc(**kw):
        d = L.NafHeadDesc()
        for f in ("z_v", "z_mu", "l", "scale", "actions", "targets", "mu", "q", "loss", "d_zv", "d_zmu", "d_l"):
            setattr(d, f, p)
        d.batch, d.n_actions, d.ld_mu, d.ld_l, d.ld_actions = 8, 3, 3, 6, 3
        for k, v in kw.items():
            setattr(d, k, v)
        return d

    assert lib.cb200_naf_head(ctypes.byref(desc()), L.current_stream()) == 0
    bad = [dict(n_actions=0), dict(n_actions=33, ld_mu=33, ld_l=561, ld_actions=33), dict(batch=0), dict(z_mu=None),
           dict(scale=None), dict(mu=None), dict(l=None), dict(q=None), dict(loss=None), dict(d_zv=None),
           dict(d_zmu=None), dict(d_l=None), dict(z_v=None), dict(actions=None), dict(targets=None), dict(ld_l=5),
           dict(ld_mu=2)]
    for kw in bad:
        with pytest.raises(ValueError):
            L.check(lib.cb200_naf_head(ctypes.byref(desc(**kw)), L.current_stream()))
    with pytest.raises(ValueError):
        L.check(lib.cb200_naf_head(None, L.current_stream()))
    torch.cuda.synchronize()


def test_clip_by_value_against_numpy():
    L, lib = _lib()
    c = 0.75
    vals = np.array([0.0, -0.0, c, -c, np.nextafter(np.float32(c), np.float32(2)), 1e30, -1e30, np.inf, -np.inf,
                     np.nan, 0.5, -0.5, 1e-40], dtype=np.float32)
    rng = np.random.RandomState(0)
    g = np.concatenate([vals, (rng.randn(100003) * 2).astype(np.float32)])
    t = torch.from_numpy(g.copy()).cuda()
    L.check(lib.cb200_clip_by_value(t.data_ptr(), t.numel(), c, L.current_stream()))
    got = t.cpu().numpy()
    want = np.where(np.isnan(g), g, np.minimum(np.maximum(g, np.float32(-c)), np.float32(c)))
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    for n, clip in ((0, 1.0), (4, 0.0), (4, -1.0)):
        with pytest.raises(ValueError):
            L.check(lib.cb200_clip_by_value(t.data_ptr(), n, clip, L.current_stream()))


def test_every_naf_head_instantiation_ran():
    if {True, False} - RAN:
        d = random_data(3, 8)
        run_head(d, train=True)
        run_head(d, train=False)
    assert RAN == {True, False}


# ---- the agent -----------------------------------------------------------------------------------------------------
SHAPES = {"hopper": (11, 3), "halfcheetah": (17, 6), "humanoid": (376, 17)}


def _make(D, A, B, widths=None, clip=None, huber=False, seed=0, memory=None):
    from coach_b200.agents.naf_agent import NAFAgent, NAFAgentParameters
    from coach_b200.memories.memory import MemoryGranularity
    ap = NAFAgentParameters()
    net = ap.network_wrappers["main"]
    ap.memory.max_size = (MemoryGranularity.Transitions, 4096)
    if memory is not None:
        ap.memory = memory
    net.batch_size = B
    net.replace_mse_with_huber_loss = huber
    if widths is not None:
        net.embedder_units, net.middleware_parameters.scheme = (widths[0],), [widths[1]]
    if clip is not None:
        net.gradients_clipping_method, net.clip_gradients = clip
    return NAFAgent(ap, observation_dim=D, action_dim=A, action_low=-0.4, action_high=np.linspace(0.5, 2.0, A),
                    seed=seed)


def _columns(rng, n, D, A):
    done = (rng.rand(n) < 0.1).astype(np.uint8)
    done[-1] = 1
    return {"state:observation": rng.randn(n, D).astype(np.float32),
            "next_state:observation": rng.randn(n, D).astype(np.float32),
            "action": rng.uniform(-1, 1, (n, A)).astype(np.float32), "reward": rng.randn(n) * 3, "game_over": done}


LEARN_CASES = [("hopper", None, 32, None, False), ("hopper", (200, 200), 256, ("ClipByValue", 1e-3), False),
               ("halfcheetah", None, 256, ("ClipByValue", 1000.0), True),
               ("halfcheetah", (200, 200), 32, ("ClipByValue", 1e-3), True),
               ("humanoid", None, 256, ("ClipByValue", 1e-3), False), ("humanoid", (200, 200), 32, None, False),
               ("halfcheetah", None, 32, ("ClipByGlobalNorm", 1e-3), False)]


@pytest.mark.parametrize("shape,widths,B,clip,huber", LEARN_CASES,
                         ids=["-".join(str(x) for x in c) for c in LEARN_CASES])
def test_learn_steps_match_the_oracle(shape, widths, B, clip, huber):
    from coach_b200.core_types import DeviceBatch
    D, A = SHAPES[shape]
    ag = _make(D, A, B, widths, clip, huber)
    n_trunk = len(ag.trunk.layers)
    p = ag.ap.network_wrappers["main"]
    ag.main.target.copy_(ag.main.store.theta * 0.9 + 0.003)          # desynchronised target
    rng = np.random.RandomState(5)
    opt = None
    gtol = {}
    for step in range(3):
        cols = _columns(rng, B, D, A)
        batch = DeviceBatch({k: torch.from_numpy(v).cuda() for k, v in cols.items()}, B)
        named, named_t = ag.main.store.export_named(), ag.main.store.export_named(ag.main.target)
        if opt is None:
            opt = make_adam(named, p.learning_rate, p.adam_optimizer_beta1, p.adam_optimizer_beta2,
                            p.optimizer_epsilon)
        loss, losses, norm = ag.learn_from_batch(batch)
        torch.cuda.synchronize()
        assert losses == [loss]
        # TD targets bit for bit given the device's V(s')
        v_dev = ag.v_target.out.cpu().numpy()
        y = ac_td_targets(cols["reward"], cols["game_over"], v_dev, 0.99).astype(np.float32)
        np.testing.assert_array_equal(ag.td_targets.cpu().numpy().view(np.uint32), y.view(np.uint32))
        ref = onaf.naf_step(named, named_t, opt, dict(states=cols["state:observation"],
                                                      next_states=cols["next_state:observation"],
                                                      actions=cols["action"], rewards=cols["reward"],
                                                      game_overs=cols["game_over"].astype(bool)),
                            ag.scale_host, n_trunk, huber_loss=huber, clip=clip)
        close(ag.td_targets.cpu().numpy(), ref["td_targets"], name="td targets")
        close(loss, ref["loss"], name="loss")
        close(norm, ref["grad_norm"], name="unclipped norm")
        g = ag.main.store.export_named(ag.main.store.grad)
        for nm in ref["grads"]:
            # the clip keeps the error the unclipped gradient had: its tolerance is that of the unclipped tensor
            gtol[nm] = gtol.get(nm, 0.0) + 2e-5 * float(ref["raw_grads"][nm].abs().max())
            close(g[nm], ref["grads"][nm].numpy(), name="grad " + nm, atol=1e-5 * float(ref["raw_grads"][nm].abs()
                                                                                         .max()))
        new = ag.main.store.export_named()
        for nm in ref["new_params"]:
            # Adam's step moves by up to (1 - beta1) alpha / epsilon = 1x a gradient difference here (epsilon 1e-4),
            # and m carries it into the next steps: the gradient tolerances of the steps so far add up
            close(new[nm], ref["new_params"][nm].numpy(), name="param " + nm,
                  atol=1e-2 * p.learning_rate + gtol[nm])
        # polyak of the target, as the train() driver runs it
        ag.main.sync(0.001)
        torch.cuda.synchronize()
        want_t = polyak(named_t, new, 0.001)
        got_t = ag.main.store.export_named(ag.main.target)
        for nm in want_t:
            np.testing.assert_array_equal(got_t[nm], want_t[nm], err_msg="target " + nm)
    if clip is not None and clip[1] < 1:
        assert norm > clip[1]                   # the clip was active


def test_graph_replay_matches_eager(monkeypatch):
    res = []
    for graph in (0, 1):
        monkeypatch.setenv("CB200_AC_GRAPH", str(graph))
        ag = _make(17, 6, 32, clip=("ClipByValue", 1e-2), seed=3)
        ag.memory.store_columns(_columns(np.random.RandomState(1), 2000, 17, 6))
        np.random.seed(5)
        losses = []
        for _ in range(7):
            ag.total_steps_counter += 1
            losses.append(ag.train(fetch=True))
        torch.cuda.synchronize()
        res.append((losses, ag.main.store.theta.clone(), ag.main.target.clone()))
        if graph:
            assert ag._graph_step.graph is not None and ag._graph_step.launches > 15
    assert res[0][0] == res[1][0]
    assert torch.equal(res[0][1], res[1][1]) and torch.equal(res[0][2], res[1][2])


def test_train_driver_on_an_episodic_replay():
    ag = _make(11, 3, 32)
    ag.memory.store_columns(_columns(np.random.RandomState(2), 600, 11, 3))
    calls = []
    sync = ag.main.sync
    ag.main.sync = lambda rate=1.0: (calls.append(rate), sync(rate))
    np.random.seed(0)
    for call in range(3):
        ag.total_steps_counter += 1                     # one environment step between train() calls
        t0 = ag.main.target.clone()
        loss = ag.train()
        assert np.isfinite(loss)
        assert ag.training_iteration == 5 * (call + 1)
        assert calls == [0.001] * (call + 1)            # exactly one polyak update per call
        assert not torch.equal(t0, ag.main.target)
    ag.train()                                          # no environment step: no update
    assert len(calls) == 3


def test_choose_actions():
    from coach_b200.exploration_policies.ou_process import BatchedOUProcess
    E, D, A = 4, 11, 3
    ag = _make(D, A, 32, seed=4)
    rng = np.random.RandomState(9)
    pol, twin = BatchedOUProcess(A, E), BatchedOUProcess(A, E)
    np.random.seed(11)
    got = []
    for _ in range(6):
        states = rng.randn(E, D).astype(np.float32)
        actions, mu = ag.choose_actions(states, pol)
        close(mu, onaf.naf_mu(ag.main.store.export_named(), states, ag.scale_host, len(ag.trunk.layers)), name="mu")
        got.append((actions, mu))
    # the same draws as E reference OUProcess objects (BatchedOUProcess is pinned to them on the host)
    np.random.seed(11)
    for actions, mu in got:
        np.testing.assert_array_equal(actions, twin.get_actions(mu))


def test_refuses_a_prioritized_replay():
    from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplayParameters
    with pytest.raises(ValueError):
        _make(11, 3, 32, memory=PrioritizedExperienceReplayParameters())


def test_checkpoint_restore_continues_bit_identically(tmp_path):
    from coach_b200 import checkpoint
    cols = _columns(np.random.RandomState(3), 800, 17, 6)

    def fresh():
        ag = _make(17, 6, 32, clip=("ClipByValue", 1000.0), seed=8)
        ag.memory.store_columns(cols)
        return ag

    a = fresh()
    np.random.seed(1)
    for _ in range(3):
        a.total_steps_counter += 1
        a.train()
    checkpoint.save_checkpoint(a, str(tmp_path))
    state = np.random.get_state()
    cont = []
    for _ in range(3):
        a.total_steps_counter += 1
        cont.append(a.train())
    b = fresh()
    checkpoint.restore_checkpoint(b, str(tmp_path))
    np.random.set_state(state)
    again = []
    for _ in range(3):
        b.total_steps_counter += 1
        again.append(b.train())
    assert cont == again
    for x, y in ((a.main.store.theta, b.main.store.theta), (a.main.target, b.main.target),
                 (a.main.store.m, b.main.store.m), (a.main.adam_state, b.main.adam_state)):
        assert torch.equal(x, y)


# ---- two ranks (gloo, both on cuda:0: the pattern of tests/test_dqn_world2_gpu.py) ----------------------------------
def _run_ranked(data_seed):
    ag =_make(17, 6, 32, clip=("ClipByValue", 1e-3), seed=5)
    ag.memory.store_columns(_columns(np.random.RandomState(data_seed), 600, 17, 6))
    losses = []
    for step in range(4):
        random.seed(20 + step)
        np.random.seed(20 + step)
        losses.append(ag.learn_from_batch(ag.sample_batch())[0])
    torch.cuda.synchronize()
    return losses, ag.main.store.theta.cpu().numpy()


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, port, shard_by_rank, out_q):
    os.environ.update(RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                      CB200_GRAPH_COLLECTIVES="0")          # gloo collectives cannot be captured into a CUDA graph
    try:
        from coach_b200 import parallel
        assert parallel.init_from_env(backend="gloo") == (rank, 2)
        out_q.put((rank, _run_ranked(3 + rank if shard_by_rank else 3)))
        torch.distributed.destroy_process_group()
    except BaseException as exc:
        out_q.put((rank, "rank %d failed: %r" % (rank, exc)))
        raise


@functools.lru_cache(maxsize=None)
def _one_rank():
    return _run_ranked(3)


@pytest.mark.parametrize("shard_by_rank", [False, True])
def test_two_ranks(shard_by_rank):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, shard_by_rank, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = dict(q.get(timeout=600) for _ in procs)
        for r in range(2):
            assert not isinstance(res[r], str), res[r]
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.pid is not None:
                if p.is_alive():
                    p.terminate()
                p.join(timeout=30)
    (l0, t0), (l1, t1) = res[0], res[1]
    assert np.array_equal(t0, t1), "the ranks' parameters diverged"
    if shard_by_rank:
        assert not np.array_equal(t0, _one_rank()[1]), "rank 0 trained as if alone: no gradient exchange"
    else:
        # clip(g) + clip(g) and the 1/2 rescale are exact: identical shards reproduce one rank bit for bit
        assert l0 == l1 == _one_rank()[0] and np.array_equal(t0, _one_rank()[1])
