"""GPU parity of the ClippedPPO learn path against the torch-CPU oracle (oracle/actor_critic.py) and the numpy oracle
of fill_advantages (oracle/rl_math.py).  Tolerances as in tests/test_learn_gpu.py (1e-5 relative to tensor scale)."""
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import actor_critic as oac     # noqa: E402  (checker only)
from oracle import rl_math as orm          # noqa: E402
from test_learn_gpu import close           # noqa: E402


def _agent(D=17, A=6, B=64, beta_entropy=0.0, seed=0, graph=True, truncate=True):
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgent, ClippedPPOAgentParameters
    from coach_b200.memories.memory import MemoryGranularity
    ap = ClippedPPOAgentParameters()
    net = ap.network_wrappers["main"]          # presets/Mujoco_ClippedPPO.py:29-36
    net.learning_rate, net.optimizer_epsilon, net.adam_optimizer_beta2 = 0.0003, 1e-5, 0.999
    ap.memory.max_size = (MemoryGranularity.Transitions, 8192)
    ap.network_wrappers["main"].batch_size = B
    ap.algorithm.beta_entropy = beta_entropy
    ap.algorithm.optimization_epochs = 2
    ap.algorithm.num_consecutive_playing_steps.num_steps = 256
    ap.algorithm.truncate_dataset_to_playing_steps = truncate
    ag = ClippedPPOAgent(ap, observation_dim=D, action_dim=A, seed=seed)
    ag.use_cuda_graph = graph
    return ag


def _rollout(rng, n, D, A, ep_len):
    s = rng.randn(n, D).astype(np.float32) * 2 + 0.3
    a = rng.randn(n, A).astype(np.float32)
    r = rng.randn(n)
    done = np.zeros(n, np.uint8)
    done[ep_len - 1::ep_len] = 1
    done[-1] = 1
    return s, a, r, done


@pytest.mark.parametrize("beta", [0.0, 0.01])
def test_ppo_head_and_minibatch_step_match_oracle(beta):
    """one minibatch: loss terms, every gradient tensor, the Adam update"""
    ag = _agent(beta_entropy=beta, graph=False)
    rng = np.random.RandomState(1)
    B, D, A = ag.B, ag.D, ag.A
    store = ag.net.store
    # make the policy differ from the old policy and the log-std non-trivial
    ag.sync()
    store.theta.add_(torch.randn(store.size, device=store.theta.device, generator=None) * 0.02)
    store.view(store.theta, ag.net.logstd_name).copy_(torch.tensor(rng.randn(A).astype(np.float32) * 0.3))
    named = store.export_named()
    old_named = store.export_named(ag.main.target)
    mb = dict(states=rng.randn(B, D).astype(np.float32), actions=rng.randn(B, A).astype(np.float32),
              advantages=rng.randn(B).astype(np.float32), value_targets=rng.randn(B).astype(np.float32))
    opt = oac.make_adam(named, 3e-4, 0.9, 0.999, 1e-5)
    ref = oac.ppo_minibatch_step(named, old_named, opt, mb, 0.2, beta)
    ref64 = oac.ppo_minibatch_step(named, old_named, oac.make_adam(named, 3e-4, 0.9, 0.999, 1e-5, torch.float64), mb,
                                   0.2, beta, dtype=torch.float64)
    dev = store.theta.device
    data = dict(states=torch.from_numpy(mb["states"]).to(dev), actions=torch.from_numpy(mb["actions"]).to(dev),
                advantages=torch.from_numpy(mb["advantages"]).to(dev),
                value_targets=torch.from_numpy(mb["value_targets"]).reshape(-1, 1).to(dev),
                old_policy=torch.from_numpy(ref["old_mu"]).to(dev))
    cols, perm, _ = ag._training_rows(B)
    for k, t in data.items():
        cols[k].copy_(t)
    perm.copy_(torch.arange(B, dtype=torch.int64, device=dev))
    ag.cursor.zero_()
    ag.clip_eps = np.float32(0.2)
    ag._minibatch_kernels()
    torch.cuda.synchronize()
    close(ag.v_loss.item(), ref["value_loss"], name="value loss")
    close(ag.scalars[0].item(), ref["policy_loss"], name="policy loss")
    close(ag.scalars[3].item(), ref["mean_ratio"], name="mean ratio")
    close(ag.scalars[2].item(), ref["entropy"], name="entropy")
    close(np.sqrt(ag.main.sumsq.item()), ref["grad_norm"], name="grad norm")
    assert ag.v_acc.item() == ag.v_loss.item() and ag.p_acc.item() == ag.scalars[0].item()   # the epoch sums
    got = store.export_named(store.grad)
    for name in ref["grads"]:
        close(got[name], ref["grads"][name].numpy(), name="grad " + name)
        e_ours = np.abs(got[name] - ref64["grads"][name].numpy()).max()
        e_orc = np.abs(ref["grads"][name].numpy() - ref64["grads"][name].numpy()).max()
        assert e_ours <= 4 * e_orc + 2e-6 * (np.abs(ref["grads"][name].numpy()).max() + 1e-30), (name, e_ours, e_orc)
    newp = store.export_named()
    for name in ref["new_params"]:
        close(newp[name], ref["new_params"][name].numpy(), name="param " + name)
    assert int(ag.cursor.item()) == B


@pytest.mark.parametrize("graph", [False, True])
def test_ppo_train_phase_matches_oracle(graph):
    """whole training phase: observation normalisation -> V(s) -> GAE -> standardise -> shuffled epochs (eager and
    CUDA-graph replay must give the same weights as the oracle loop)"""
    ag = _agent(graph=graph)
    rng = np.random.RandomState(2)
    n, D, A, B = 256, ag.D, ag.A, ag.B
    s, a, r, done = _rollout(rng, n, D, A, 50)
    ag.memory.store_columns({"state:observation": s, "next_state:observation": s, "action": a, "reward": r,
                             "game_over": done})
    store = ag.net.store
    named0 = store.export_named()
    ag.total_steps_counter = 256
    random.seed(5)
    ag.train()
    torch.cuda.synchronize()
    got = store.export_named()

    # ---- oracle ----
    random.seed(5)
    rs = orm.RunningStats([D])
    rs.push(s)
    sn = rs.normalize(s).astype(np.float32)
    named = {k: torch.from_numpy(v) for k, v in named0.items()}
    vals = oac.mlp(list(named.values())[0:6], torch.from_numpy(sn), ["tanh", "tanh", None]).numpy()[:, 0]
    adv, tgt, nv = orm.ppo_fill_advantages(r, vals, done.astype(bool), 0.99, 0.95)
    assert nv == n
    opt = oac.make_adam(named0, 3e-4, 0.9, 0.999, 1e-5)
    cur = dict(named0)
    old = dict(named0)                                   # target network = weights at sync time
    order = list(range(n))
    for epoch in range(2):
        random.shuffle(order)
        for i in range(n // B):
            rows = order[i * B:(i + 1) * B]
            mb = dict(states=sn[rows], actions=a[rows], advantages=adv[rows].astype(np.float32),
                      value_targets=tgt[rows].astype(np.float32))
            out = oac.ppo_minibatch_step(cur, old, opt, mb, 0.2, 0.0)
            cur = {k: v.numpy() for k, v in out["new_params"].items()}
    for name in cur:
        close(got[name], cur[name], rtol=5e-5, name="param " + name)     # 8 chained Adam steps
    assert ag.memory.num_transitions() == 0              # post_training_commands: memory.clean()


def test_episodic_replay_nstep_and_order():
    from coach_b200.memories.episodic_experience_replay import EpisodicExperienceReplay
    from coach_b200.memories.memory import MemoryGranularity
    from coach_b200.core_types import Transition
    mem = EpisodicExperienceReplay((MemoryGranularity.Transitions, 64), n_step=3, discount=0.9)
    rng = np.random.RandomState(0)
    rewards = []
    for ep_len in (5, 1, 7):
        ep = rng.randn(ep_len)
        rewards.append(ep)
        for t in range(ep_len):
            mem.store(Transition(state={'observation': np.array([float(len(rewards)), float(t)], dtype=np.float32)},
                                 action=np.zeros(2, np.float32), reward=float(ep[t]),
                                 next_state={'observation': np.zeros(2, np.float32)}, game_over=(t == ep_len - 1)))
    mem.store(Transition(state={'observation': np.zeros(2, np.float32)}, action=np.zeros(2, np.float32), reward=1.0,
                         next_state={'observation': np.zeros(2, np.float32)}, game_over=False))   # open episode
    assert mem.num_complete_episodes() == 3 and mem.num_transitions_in_complete_episodes() == 13
    assert mem.length() == 4
    b = mem.transitions_batch()
    assert b.size == 13
    obs = b.states(["observation"])["observation"].cpu().numpy()
    assert obs[:, 0].tolist() == [1.0] * 5 + [2.0] + [3.0] * 7
    want = np.concatenate([orm.n_step_returns(e, 0.9, 3) for e in rewards])
    np.testing.assert_array_equal(b.n_step_discounted_rewards().cpu().numpy(), want)
    np.random.seed(0)
    sb = mem.sample_batch(8)
    assert sb.size == 8
    mem.clean()
    assert mem.num_transitions_in_complete_episodes() == 0
