"""Discrete ClippedPPO on the GPU against oracle/clipped_ppo_discrete.py:

  cb200_ppo_categorical_head at the C ABI: A in {1, 2, 3, 18, 32} x B in {1, 64, 1000, 4096} x beta in {0, 0.01} within
  fp64 bounds, every clipping regime, an exact probe (old = new), out-of-range actions, argument errors, one launch per
  call, bit-identical repeats and a captured graph that follows the device rescaler;
  the agent: one minibatch step, whole training phases (eager and graph), the graph captures across phases while the
  clipping schedule moves or stays put, acting and a checkpoint round trip for both action kinds.

Generated ratios keep a margin from the clip bounds 1 -+ e, where fp32 and fp64 could pick different branches."""
import os
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from abi_util import _lib, assert_bits            # noqa: E402
from oracle import actor_critic as oac           # noqa: E402
from oracle import clipped_ppo_discrete as oc    # noqa: E402
from oracle import rl_math as orm                # noqa: E402
from test_learn_gpu import close                 # noqa: E402

EPS, RESCALER = 0.2, 0.7
MARGIN = 1e-4                                    # relative distance of every generated ratio from the clip bounds


def _softmax(z):
    e = np.exp(z - z.max(1, keepdims=True))
    return e / e.sum(1, keepdims=True)


def _ratios64(z, q, a):
    """fp64 ratio of each row's action (actions inside [0, A))"""
    lp = np.log(_softmax(z.astype(np.float64)))
    lq = np.log(q.astype(np.float64))
    lq = lq - np.log(np.exp(lq).sum(1, keepdims=True))
    r = np.arange(len(a))
    return np.exp(lp[r, a] - lq[r, a])


def _case(seed, B, A, spread=0.6):
    """logits, int64 actions, old probabilities (a perturbed softmax) and advantages; rows whose ratio would lie within
    MARGIN of a bound get new old probabilities"""
    rng = np.random.RandomState(seed)
    z = (rng.randn(B, A) * 1.5).astype(np.float32)
    a = rng.randint(0, A, B).astype(np.int64)
    adv = rng.randn(B).astype(np.float32)
    q = _softmax(z + rng.randn(B, A) * spread).astype(np.float32)
    lo, hi = oc.clip_bounds(EPS, RESCALER)
    for _ in range(50):
        r = _ratios64(z, q, a)
        near = (np.abs(r - lo) < MARGIN * lo) | (np.abs(r - hi) < MARGIN * hi)
        if not near.any():
            break
        q[near] = _softmax(z[near] + rng.randn(int(near.sum()), A) * spread).astype(np.float32)
    assert not near.any()
    return dict(z=z, a=a, q=q, adv=adv)


def _run(c, rescaler, beta, outs=None, clip_eps=EPS):
    L, lib = _lib()
    B, A = c["z"].shape
    t = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() for k, v in c.items()}
    r = rescaler if torch.is_tensor(rescaler) else torch.tensor([rescaler], dtype=torch.float32, device="cuda")
    dz, sc = outs if outs is not None else (torch.zeros((B, A), device="cuda"), torch.zeros(5, device="cuda"))
    L.check(lib.cb200_ppo_categorical_head(t["z"].data_ptr(), t["a"].data_ptr(), t["q"].data_ptr(),
                                           t["adv"].data_ptr(), B, A, clip_eps, r.data_ptr(), beta, dz.data_ptr(),
                                           sc.data_ptr(), L.current_stream()))
    torch.cuda.synchronize()
    return (dz.cpu().numpy(), sc.cpu().numpy()), t


def _check_against_fp64(c, got_dz, got_sc, rescaler, beta, clip_eps=EPS):
    d64, s64 = oc.categorical_head(c["z"], c["a"], c["q"], c["adv"], clip_eps, rescaler, beta, torch.float64)
    d32, _ = oc.categorical_head(c["z"], c["a"], c["q"], c["adv"], clip_eps, rescaler, beta, torch.float32)
    e_ours = np.abs(got_dz.astype(np.float64) - d64).max()
    e_orc = np.abs(d32.astype(np.float64) - d64).max()
    assert e_ours <= 4 * e_orc + 1e-5 * (np.abs(d64).max() + 1e-30), (e_ours, e_orc)
    for k, name in enumerate(("loss", "kl", "entropy", "mean ratio", "mean clipped ratio")):
        assert abs(float(got_sc[k]) - s64[k]) <= 2e-5 * (1 + abs(s64[k])), (name, got_sc[k], s64[k])


CASES = [(A, B, beta) for A in (1, 2, 3, 18, 32) for B in (1, 64, 1000, 4096) for beta in (0.0, 0.01)]


@pytest.mark.parametrize("A, B, beta", CASES)
def test_head_matches_fp64(A, B, beta):
    c = _case(1000 * A + B, B, A)
    (dz, sc), _ = _run(c, RESCALER, beta)
    _check_against_fp64(c, dz, sc, RESCALER, beta)


def test_cases_cover_every_regime():
    """inside the bounds, clipped above with A > 0 and below with A < 0 (zero surrogate gradient), and above / below
    with the other sign (the unclipped term is the minimum); the boundary case is test_exact_probe_and_boundary"""
    lo, hi = oc.clip_bounds(EPS, RESCALER)
    seen = set()
    for A, B, beta in CASES:
        c = _case(1000 * A + B, B, A)
        r = _ratios64(c["z"], c["q"], c["a"])
        pos = c["adv"] > 0
        seen |= {"inside"} if ((r > lo) & (r < hi)).any() else set()
        seen |= {"above, A > 0"} if ((r > hi) & pos).any() else set()
        seen |= {"below, A < 0"} if ((r < lo) & ~pos).any() else set()
        seen |= {"above, A < 0"} if ((r > hi) & ~pos).any() else set()
        seen |= {"below, A > 0"} if ((r < lo) & pos).any() else set()
    assert seen == {"inside", "above, A > 0", "below, A < 0", "above, A < 0", "below, A > 0"}, seen


@pytest.mark.parametrize("rescaler", [RESCALER, 0.0])
@pytest.mark.parametrize("A", [1, 2, 5, 18, 32])
def test_exact_probe_and_boundary(A, rescaler):
    """rows of equal logits and equal old probabilities: old = new exactly, so every ratio is 1 and KL is 0 bit for bit.
    With rescaler 0 both bounds are 1: the ratio sits on the boundary, where the surrogate gradient still passes."""
    rng = np.random.RandomState(A)
    B = 200
    c = dict(z=np.repeat(rng.randn(B, 1).astype(np.float32), A, 1), a=rng.randint(0, A, B).astype(np.int64),
             q=np.repeat(rng.rand(B, 1).astype(np.float32) + 0.1, A, 1), adv=rng.randn(B).astype(np.float32))
    (dz, sc), _ = _run(c, rescaler, 0.01)
    assert sc[1] == 0.0 and sc[3] == 1.0 and sc[4] == 1.0, sc
    _check_against_fp64(c, dz, sc, rescaler, 0.01)
    # the gradient of row i on its action: -(A_i / B) (1 - 1/A) (the entropy term of a uniform row is 0 up to
    # rounding), which the boundary case passes on as well
    if A > 1:
        r = np.arange(B)
        np.testing.assert_allclose(dz[r, c["a"]], -(c["adv"] / B) * (1 - np.float32(1.0 / A)), rtol=1e-5, atol=1e-9)


@pytest.mark.parametrize("A", [2, 18])
def test_out_of_range_actions_have_no_surrogate_term(A):
    c = _case(77 + A, 1000, A)
    c["a"][::7] = -1
    c["a"][3::11] = A
    c["a"][5::13] = A + 1000
    c["a"][1] = np.iinfo(np.int64).min
    (dz, sc), _ = _run(c, RESCALER, 0.01)
    _check_against_fp64(c, dz, sc, RESCALER, 0.01)
    (dz0, _), _ = _run(c, RESCALER, 0.0)
    bad = (c["a"] < 0) | (c["a"] >= A)
    assert (dz0[bad] == 0).all()                   # beta 0: no gradient at all from those rows


def test_argument_errors_write_nothing_and_one_launch_per_call():
    L, lib = _lib()
    c = _case(5, 64, 3)
    _, t = _run(c, RESCALER, 0.0)
    r = torch.tensor([RESCALER], device="cuda")
    dz = torch.full((64, 3), 7.0, device="cuda")
    sc = torch.full((5,), 7.0, device="cuda")
    p = dict(z=t["z"].data_ptr(), a=t["a"].data_ptr(), q=t["q"].data_ptr(), adv=t["adv"].data_ptr(), B=64, A=3,
             r=r.data_ptr(), dz=dz.data_ptr(), sc=sc.data_ptr())
    bad = [dict(B=0), dict(B=-1), dict(A=0), dict(A=33), dict(z=None), dict(a=None), dict(q=None), dict(adv=None),
           dict(r=None), dict(dz=None)]
    c0 = lib.cb200_launch_count()
    for b in bad:
        a = dict(p)
        a.update(b)
        rc = lib.cb200_ppo_categorical_head(a["z"], a["a"], a["q"], a["adv"], a["B"], a["A"], EPS, a["r"], 0.0,
                                            a["dz"], a["sc"], L.current_stream())
        assert rc == -1, b
    torch.cuda.synchronize()
    assert lib.cb200_launch_count() == c0, "a refused call launched"
    assert (dz == 7.0).all() and (sc == 7.0).all()
    with pytest.raises(ValueError):
        L.check(lib.cb200_ppo_categorical_head(None, p["a"], p["q"], p["adv"], 64, 3, EPS, p["r"], 0.0, p["dz"], None,
                                               L.current_stream()))
    for scalars in (None, p["sc"]):                # scalars are optional
        c0 = lib.cb200_launch_count()
        L.check(lib.cb200_ppo_categorical_head(p["z"], p["a"], p["q"], p["adv"], 64, 3, EPS, p["r"], 0.0, p["dz"],
                                               scalars, L.current_stream()))
        assert lib.cb200_launch_count() - c0 == 1
    torch.cuda.synchronize()
    assert float((dz * 0 + 1).sum()) == 192.0      # the library and torch stay usable


def test_repeat_calls_and_graph_replay_follow_the_device_rescaler():
    L, lib = _lib()
    c = _case(11, 4096, 18)
    B, A = c["z"].shape
    r = torch.tensor([RESCALER], device="cuda")
    outs = (torch.zeros((B, A), device="cuda"), torch.zeros(5, device="cuda"))
    first, t = _run(c, r, 0.01, outs)
    first = tuple(x.copy() for x in first)
    again, _ = _run(c, r, 0.01, outs)
    for x, y, n in zip(first, again, ("d_logits", "scalars")):
        assert_bits(y, x, n)
    g = torch.cuda.CUDAGraph()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side), torch.cuda.graph(g):
        L.check(lib.cb200_ppo_categorical_head(t["z"].data_ptr(), t["a"].data_ptr(), t["q"].data_ptr(),
                                               t["adv"].data_ptr(), B, A, EPS, r.data_ptr(), 0.01, outs[0].data_ptr(),
                                               outs[1].data_ptr(), L.current_stream()))
    torch.cuda.current_stream().wait_stream(side)
    g.replay()
    torch.cuda.synchronize()
    for x, y, n in zip(first, outs, ("d_logits", "scalars")):
        assert_bits(y.cpu().numpy(), x, n)
    r.fill_(0.3)                                    # the schedule moves between replays
    g.replay()
    torch.cuda.synchronize()
    eager, _ = _run(c, 0.3, 0.01)
    for x, y, n in zip(eager, outs, ("d_logits", "scalars")):
        assert_bits(y.cpu().numpy(), x, n)
    assert not np.array_equal(eager[1], first[1])  # and the new bounds clip other rows


# ---- agent ---------------------------------------------------------------------------------------------------------------
def _params(schedule=None, beta=0.01, epochs=2, playing=256, B=64):
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgentParameters
    from coach_b200.memories.memory import MemoryGranularity
    from coach_b200.schedules import LinearSchedule
    ap = ClippedPPOAgentParameters()
    net = ap.network_wrappers["main"]              # presets/CartPole_ClippedPPO.py
    net.learning_rate, net.optimizer_epsilon, net.adam_optimizer_beta2 = 0.0003, 1e-5, 0.999
    net.batch_size = B
    ap.memory.max_size = (MemoryGranularity.Transitions, 8192)
    ap.algorithm.beta_entropy = beta
    ap.algorithm.optimization_epochs = epochs
    ap.algorithm.num_consecutive_playing_steps.num_steps = playing
    ap.algorithm.clipping_decay_schedule = schedule if schedule is not None else LinearSchedule(1.0, 0.0, 1000)
    return ap


def _agent(A=3, D=8, graph=True, seed=0, continuous=False, **kw):
    """discrete actions, or continuous ones bounded to [-2, 2]"""
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgent
    space = dict(action_dim=A, action_low=-2.0, action_high=2.0) if continuous else dict(num_actions=A)
    ag = ClippedPPOAgent(_params(**kw), observation_dim=D, seed=seed, **space)
    ag.use_cuda_graph = graph
    return ag


def _draws(rng, E, A, continuous=False):
    """choose_actions' training draws for E environments"""
    return dict(normals=rng.standard_normal((E, A))) if continuous else dict(uniforms=rng.random_sample(E))


def _rollout(rng, n, D, A, ep_len, continuous=False):
    s = (rng.randn(n, D) * 2 + 0.3).astype(np.float32)
    a = rng.randn(n, A).astype(np.float32) if continuous else rng.randint(0, A, n).astype(np.int64)
    r = rng.randn(n)
    done = np.zeros(n, np.uint8)
    done[ep_len - 1::ep_len] = 1
    done[-1] = 1
    return s, a, r, done


def _store(ag, roll):
    s, a, r, done = roll
    ag.memory.store_columns({"state:observation": s, "next_state:observation": s, "action": a, "reward": r,
                             "game_over": done})
    ag.total_steps_counter += len(r)


def test_network_layout_and_init():
    ag = _agent(A=18, D=4)
    names = list(ag.net.store.entries)
    assert len(names) == 14 and not any("log_std" in n for n in names)
    named = ag.net.store.export_named()
    kernel, bias = named[names[11]], named[names[12]]               # policy_fc, then the head's rescaler
    assert kernel.shape == (64, 18) and (kernel != 0).all()
    assert bias.shape == (18,) and (bias == 0).all()
    limit = np.sqrt(6.0 / (64 + 18))               # TF's default glorot_uniform
    assert np.abs(kernel).max() <= limit and np.abs(kernel).max() > 0.9 * limit


@pytest.mark.parametrize("beta", [0.0, 0.01])
def test_minibatch_step_matches_oracle(beta):
    """one minibatch: loss terms, the head's scalars, every gradient tensor, the Adam update"""
    ag = _agent(beta=beta, graph=False)
    rng = np.random.RandomState(1)
    B, D, A = ag.B, ag.D, ag.A
    store = ag.net.store
    ag.sync()
    store.theta.add_(torch.from_numpy(rng.randn(store.size).astype(np.float32) * 0.2).cuda())
    named = store.export_named()
    old_named = store.export_named(ag.main.target)
    states = rng.randn(B, D).astype(np.float32)
    q = oc.old_probs(old_named, states)
    logits = oac.mlp([torch.from_numpy(v).double() for v in list(named.values())[7:13]], torch.from_numpy(states)
                     .double(), ["tanh", "tanh", None]).numpy()
    acts = rng.randint(0, A, B).astype(np.int64)
    lo, hi = oc.clip_bounds(EPS, 0.8)
    for _ in range(50):                            # keep the ratios a margin away from the bounds
        r = _ratios64(logits, q, acts)
        near = (np.abs(r - lo) < MARGIN) | (np.abs(r - hi) < MARGIN)
        if not near.any():
            break
        acts[near] = (acts[near] + 1) % A
    assert not near.any()
    mb = dict(states=states, actions=acts, advantages=rng.randn(B).astype(np.float32),
              value_targets=rng.randn(B).astype(np.float32), old_probs=q)
    ref = oc.minibatch_step(named, oac.make_adam(named, 3e-4, 0.9, 0.999, 1e-5), mb, EPS, 0.8, beta)
    ref64 = oc.minibatch_step(named, oac.make_adam(named, 3e-4, 0.9, 0.999, 1e-5, torch.float64), mb, EPS, 0.8, beta,
                              dtype=torch.float64)
    dev = store.theta.device
    data = dict(states=torch.from_numpy(states).to(dev), actions=torch.from_numpy(acts).to(dev),
                advantages=torch.from_numpy(mb["advantages"]).to(dev),
                value_targets=torch.from_numpy(mb["value_targets"]).reshape(-1, 1).to(dev),
                old_policy=torch.from_numpy(q).to(dev))
    cols, perm, _ = ag._training_rows(B)
    for k, t in data.items():
        cols[k].copy_(t)
    perm.copy_(torch.arange(B, dtype=torch.int64, device=dev))
    ag.cursor.zero_()
    ag.clip_eps = np.float32(EPS)
    ag.clip_rescaler.fill_(0.8)
    ag._minibatch_kernels()
    torch.cuda.synchronize()
    close(ag.v_loss.item(), ref["value_loss"], name="value loss")
    sc = ag.scalars.cpu().numpy()
    for k, name in enumerate(("policy loss", "kl", "entropy", "mean ratio", "mean clipped ratio")):
        close(sc[k], ref["scalars"][k], atol=1e-6, name=name)
    close(np.sqrt(ag.main.sumsq.item()), ref["grad_norm"], name="grad norm")
    assert ag.v_acc.item() == ag.v_loss.item() and ag.p_acc.item() == sc[0]       # the epoch sums
    got = store.export_named(store.grad)
    for name in ref["grads"]:
        close(got[name], ref["grads"][name].numpy(), rtol=1e-4, name="grad " + name)
        e_ours = np.abs(got[name] - ref64["grads"][name].numpy()).max()
        e_orc = np.abs(ref["grads"][name].numpy() - ref64["grads"][name].numpy()).max()
        assert e_ours <= 4 * e_orc + 2e-6 * (np.abs(ref["grads"][name].numpy()).max() + 1e-30), (name, e_ours, e_orc)
    newp = store.export_named()
    for name in ref["new_params"]:
        close(newp[name], ref["new_params"][name].numpy(), name="param " + name)
    assert int(ag.cursor.item()) == B


def _oracle_phase(named0, roll, order_seed, rescaler, epochs=2, B=64, beta=0.01):
    """observation normalisation -> V(s) -> GAE -> standardise -> old probabilities -> shuffled epochs"""
    s, a, r, done = roll
    n, D = s.shape
    rs = orm.RunningStats([D])
    rs.push(s)
    sn = rs.normalize(s).astype(np.float32)
    vals = oac.mlp([torch.from_numpy(v) for v in list(named0.values())[0:6]], torch.from_numpy(sn),
                   ["tanh", "tanh", None]).numpy()[:, 0]
    adv, tgt, nv = orm.ppo_fill_advantages(r, vals, done.astype(bool), 0.99, 0.95)
    assert nv == n
    q = oc.old_probs(named0, sn)                   # the target network = the weights at sync time
    opt = oac.make_adam(named0, 3e-4, 0.9, 0.999, 1e-5)
    cur = dict(named0)
    random.seed(order_seed)
    order = list(range(n))
    for _ in range(epochs):
        random.shuffle(order)
        for i in range(n // B):
            rows = order[i * B:(i + 1) * B]
            mb = dict(states=sn[rows], actions=a[rows], advantages=adv[rows].astype(np.float32),
                      value_targets=tgt[rows].astype(np.float32), old_probs=q[rows])
            out = oc.minibatch_step(cur, opt, mb, EPS, rescaler, beta)
            cur = {k: v.numpy() for k, v in out["new_params"].items()}
    return cur


def test_training_phase_eager_and_graph_agree_and_match_the_oracle():
    rng = np.random.RandomState(2)
    agents = [_agent(graph=g) for g in (False, True)]
    roll = _rollout(rng, 256, agents[0].D, agents[0].A, 50)
    named0 = agents[0].net.store.export_named()
    for ag in agents:
        ag.ap.algorithm.clipping_decay_schedule.current_value = 0.9
        _store(ag, roll)
        random.seed(5)
        ag.train()
    torch.cuda.synchronize()
    got = [ag.net.store.export_named() for ag in agents]
    for name in got[0]:
        assert_bits(got[1][name], got[0][name], "graph vs eager " + name)
    assert agents[1].graph_captures == 1 and agents[0].graph_captures == 0
    assert float(agents[1].clip_rescaler.item()) == np.float32(0.9)
    want = _oracle_phase(named0, roll, 5, 0.9)
    for name in want:
        close(got[0][name], want[name], rtol=5e-5, name="param " + name)      # 8 chained Adam steps
    assert agents[0].memory.num_transitions() == 0        # post_training_commands: memory.clean()


def _phases_across_the_schedule(continuous, moving):
    """three phases with acting between them, eager and graph: every phase stays bit-identical to eager execution.
    The discrete graph is captured once, so the replayed graph reads each phase's rescaler; the continuous step takes
    fp32(epsilon * value) as a launch argument and is captured once per distinct value."""
    from coach_b200.schedules import ConstantSchedule, LinearSchedule
    # ten epochs, as the presets train: each epoch's permutation must reach the device intact while the host shuffles
    # the next one
    agents = [_agent(graph=g, continuous=continuous, epochs=10,
                     schedule=LinearSchedule(1.0, 0.0, 600) if moving else ConstantSchedule(0.7)) for g in (False, True)]
    rng = np.random.RandomState(3)
    values = []
    for phase in range(3):
        roll = _rollout(rng, 256, 8, 3, 40, continuous)
        states = rng.randn(64, 8).astype(np.float32)
        draws = _draws(rng, 64, 3, continuous)
        for ag in agents:
            ag.choose_actions(states, **draws)
            _store(ag, roll)
            random.seed(10 + phase)
            ag.train()
        values.append(agents[1].ap.algorithm.clipping_decay_schedule.current_value)
        torch.cuda.synchronize()
        if not continuous:
            assert float(agents[1].clip_rescaler.item()) == np.float32(values[-1])
        a, b = agents[0].net.store.export_named(), agents[1].net.store.export_named()
        for name in a:
            assert_bits(b[name], a[name], "phase %d %s" % (phase, name))
        for x, y, name in zip(agents[0].last_losses, agents[1].last_losses, ("value loss", "policy loss")):
            assert_bits(y.cpu().numpy(), x.cpu().numpy(), "phase %d %s" % (phase, name))
    assert len(set(values)) == (3 if moving else 1)
    eps = {np.float32(agents[1].ap.algorithm.clip_likelihood_ratio_using_epsilon * v) for v in values}
    assert agents[1].graph_captures == (len(eps) if continuous else 1) and agents[0].graph_captures == 0


def test_one_graph_across_phases_while_the_schedule_moves():
    """the clipping schedule moves with acting between phases; the discrete graph is captured once"""
    _phases_across_the_schedule(continuous=False, moving=True)


@pytest.mark.parametrize("moving", [False, True], ids=["constant", "moving"])
def test_continuous_graph_captures_follow_the_clip_epsilon(moving):
    """a schedule that stays put between phases captures the continuous step once; a moving one once per distinct
    fp32 epsilon"""
    _phases_across_the_schedule(continuous=True, moving=moving)


def _oracle_probs(ag, states):
    """the policy's softmax on the states as the pre-network filter normalises them (no statistics update)"""
    flt = list(ag.pre_network_filter._observation_filters["observation"].values())[0]
    rs = flt.running_observation_stats
    x = rs.normalize(torch.from_numpy(states).cuda()).cpu().numpy()
    return oc.old_probs(ag.net.store.export_named(), x)


def test_discrete_acting_draws_numpy_choice_and_steps_the_schedule():
    from coach_b200.schedules import LinearSchedule
    ag = _agent(A=5, schedule=LinearSchedule(1.0, 0.0, 1000))
    _store(ag, _rollout(np.random.RandomState(4), 256, 8, 5, 64))
    ag.train()                                     # the filter holds statistics, the weights have moved
    flt = list(ag.pre_network_filter._observation_filters["observation"].values())[0]
    n0 = float(flt.running_observation_stats.n)
    rng = np.random.RandomState(5)
    E = 300
    states = (rng.randn(E, 8) * 3).astype(np.float32)
    u = rng.random_sample(E)
    actions, probs = ag.choose_actions(states, uniforms=u)
    np.testing.assert_array_equal(actions, oc.act(probs, u))
    np.testing.assert_allclose(probs, _oracle_probs(ag, states), rtol=2e-5, atol=1e-7)
    ev, probs_ev = ag.choose_actions(states, evaluation=True)
    np.testing.assert_array_equal(ev, oc.act(probs_ev))
    assert_bits(probs_ev, probs, "probabilities")
    assert len(set(actions.tolist())) == 5
    assert float(flt.running_observation_stats.n) == n0              # inference does not update the statistics
    want = oc.schedule_values(LinearSchedule(1.0, 0.0, 1000), 2 * E)[-1]
    assert ag.ap.algorithm.clipping_decay_schedule.current_value == want
    np.random.seed(9)                              # default draws: what E successive np.random.choice calls draw
    a2, p2 = ag.choose_actions(states[:7])
    np.random.seed(9)
    np.testing.assert_array_equal(a2, [np.random.choice(5, p=p) for p in p2])


def test_continuous_acting_draws_numpy_normal_and_steps_both_schedules():
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgent
    from coach_b200.schedules import LinearSchedule
    ap = _params(schedule=LinearSchedule(1.0, 0.0, 100))
    ap.exploration["BoxActionSpace"].noise_schedule = LinearSchedule(0.5, 0.1, 50)
    ag = ClippedPPOAgent(ap, observation_dim=8, action_dim=3, action_low=-2.0, action_high=2.0, seed=1)
    s = ag.net.store
    s.view(s.theta, ag.net.logstd_name).copy_(torch.tensor([-0.5, 0.0, 0.3]))
    rng = np.random.RandomState(6)
    E = 40
    states = rng.randn(E, 8).astype(np.float32)
    n = rng.standard_normal((E, 3))
    acts, means, stds = ag.choose_actions(states, normals=n)
    assert acts.dtype == np.float64
    np.testing.assert_allclose(stds, np.tile(np.exp(np.array([-0.5, 0.0, 0.3], np.float32)), (E, 1)), rtol=1e-6)
    assert (stds == stds[0]).all()
    assert_bits(acts, means.astype(np.float64) + stds.astype(np.float64) * n, "actions")
    ev, means_ev, _ = ag.choose_actions(states, evaluation=True)
    assert_bits(ev, means_ev, "evaluation")
    assert_bits(means_ev, means, "means")
    assert ap.algorithm.clipping_decay_schedule.current_value == \
        oc.schedule_values(LinearSchedule(1.0, 0.0, 100), 2 * E)[-1]
    assert ag.noise_schedule.current_value == oc.schedule_values(LinearSchedule(0.5, 0.1, 50), E)[-1]


def _checkpoint_round_trip(tmp_path, continuous):
    """save after a phase and acting, restore into an agent built from another seed, train one more phase in both"""
    from coach_b200 import checkpoint
    from coach_b200.schedules import LinearSchedule
    rng = np.random.RandomState(7)
    rolls = [_rollout(rng, 256, 8, 3, 64, continuous) for _ in range(2)]
    a = _agent(schedule=LinearSchedule(1.0, 0.0, 500), seed=0, continuous=continuous)
    _store(a, rolls[0])
    a.train()
    a.choose_actions(rng.randn(32, 8).astype(np.float32), **_draws(rng, 32, 3, continuous))
    name = checkpoint.save_checkpoint(a, str(tmp_path))
    # the network's files: weights, Adam slots, Adam state and the target buffer
    assert sorted(f[len(name) + 1:] for f in os.listdir(str(tmp_path)) if f.startswith(name + ".net_")) == \
        sorted("net_main.%s.npy" % k for k in ("theta", "m", "v", "adam_state", "target"))
    b = _agent(schedule=LinearSchedule(1.0, 0.0, 500), seed=3, continuous=continuous)
    checkpoint.restore_checkpoint(b, str(tmp_path), name)
    assert b.ap.algorithm.clipping_decay_schedule.current_value == a.ap.algorithm.clipping_decay_schedule.current_value
    for ag in (a, b):
        _store(ag, rolls[1])
        random.seed(8)
        ag.train()
    torch.cuda.synchronize()
    x, y = a.net.store.export_named(), b.net.store.export_named()
    for k in x:
        assert_bits(y[k], x[k], k)
    assert_bits(b.net.store.m.cpu().numpy(), a.net.store.m.cpu().numpy(), "adam m")
    assert_bits(b.main.target.cpu().numpy(), a.main.target.cpu().numpy(), "target")
    assert_bits(b.main.adam_state.cpu().numpy(), a.main.adam_state.cpu().numpy(), "adam state")


def test_checkpoint_restore_then_next_phase_is_bit_identical(tmp_path):
    _checkpoint_round_trip(tmp_path, continuous=False)


def test_continuous_checkpoint_restore_then_next_phase_is_bit_identical(tmp_path):
    _checkpoint_round_trip(tmp_path, continuous=True)
