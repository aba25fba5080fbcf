"""Pins Bootstrapped DQN to the unmodified reference: tests/golden/bootstrapped.npz.

  BootstrappedDQNAgent.learn_from_batch   rl_coach/agents/bootstrapped_dqn_agent.py:57-86 (stand-in networks, as in
                                          oracle/make_golden_agents.py: the TD-target lists handed to the train op)
  BootstrappedDQNAgent.observe's masks    :88-92 (np.random.binomial(1, p, K) per transition)
  Bootstrapped / UCB exploration          exploration_policies/bootstrapped.py:41-88, ucb.py:45-90 (E seeded objects
                                          over T steps in TRAIN and TEST with a scripted set of episode starts)
  parameter defaults                      the agent, network, exploration and preset parameters

Protocol of the exploration records: at every step, first ``select_head()`` of each environment that starts an
episode (in environment order), then ``get_action`` of environment 0, 1, ..., each handed the K head outputs [1, A]
when ``requires_action_values()`` and None otherwise (value_optimization_agent.py:54-58).

Run in the build container only:   python -m oracle.make_golden_bootstrapped          TEST INFRASTRUCTURE ONLY.
"""
import os
import sys
from types import SimpleNamespace

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
OUT = os.path.join(os.path.dirname(HERE), "tests", "golden")

K, A = 10, 6


class _Sig(object):
    def add_sample(self, *_a, **_k):
        pass


def golden_prologue(out, rng, B=64):
    from rl_coach.agents.bootstrapped_dqn_agent import BootstrappedDQNAgent
    from rl_coach.core_types import Batch, Transition
    ts = []
    for i in range(B):
        t = Transition(state={'observation': rng.randn(4).astype(np.float32)}, action=int(rng.randint(0, A)),
                       reward=float(rng.choice([-1.0, 0.0, 1.0, 0.37])),
                       next_state={'observation': rng.randn(4).astype(np.float32)}, game_over=bool(rng.rand() < 0.2))
        t.info['mask'] = rng.binomial(1, 0.5, K)
        ts.append(t)
    ts[0].info['mask'][:] = 0                                             # a transition no head learns from
    batch = Batch(ts)
    q_next = [rng.randn(B, A).astype(np.float32) for _ in range(K)]
    q_online = [rng.randn(B, A).astype(np.float32) for _ in range(K)]
    q_select = [rng.randn(B, A).astype(np.float32) for _ in range(K)]
    for h in range(K):                                                    # ties: np.argmax takes the first
        i = 3 + h
        q_select[h][i, 1] = q_select[h][i, 4] = q_select[h][i].max() + 1.0
    rec = {}
    net = SimpleNamespace(
        target_network="T", online_network=SimpleNamespace(predict=lambda states: [q.copy() for q in q_select]),
        parallel_prediction=lambda pairs: [q.copy() for q in q_next] + [q.copy() for q in q_online],
        train_and_sync_networks=lambda states, targets: rec.update(targets=[np.array(t) for t in targets]) or
        (0.0, [0.0], 0.0))
    ap = SimpleNamespace(network_wrappers={'main': SimpleNamespace(input_embedders_parameters={'observation': None})},
                         algorithm=SimpleNamespace(discount=0.99),
                         exploration=SimpleNamespace(architecture_num_q_heads=K))
    fake = SimpleNamespace(ap=ap, networks={'main': net}, q_values=_Sig())
    BootstrappedDQNAgent.learn_from_batch(fake, batch)
    out["pro_q_next"], out["pro_q_online"], out["pro_q_select"] = np.stack(q_next), np.stack(q_online), np.stack(q_select)
    out["pro_actions"] = batch.actions().astype(np.int64)
    out["pro_rewards"] = batch.rewards().astype(np.float64)
    out["pro_game_overs"] = batch.game_overs().astype(np.uint8)
    out["pro_masks"] = np.stack([t.info['mask'] for t in ts]).astype(np.uint8)
    out["pro_discount"] = np.float64(0.99)
    assert all(t.dtype == np.float32 for t in rec["targets"])
    out["pro_targets"] = np.stack(rec["targets"])                         # [K, B, A], what the train op is fed


def golden_masks(out):
    """observe's draw: n sequential binomial(1, p, K) calls, and the stream position they leave"""
    for tag, p in (("p1", 1.0), ("p05", 0.5)):
        np.random.seed(77)
        m = np.stack([np.random.binomial(1, p, K) for _ in range(12)]).astype(np.uint8)
        out["masks_%s" % tag] = m
        out["masks_%s_next_rand" % tag] = np.float64(np.random.rand())


def _q_values(rng, T, E):
    """[T, E, K, A] float32: generic values on even steps, coarse ones (ties in the argmaxes and the votes) on odd"""
    q = rng.randn(T, E, K, A).astype(np.float32)
    coarse = (rng.randint(-2, 3, (T, E, K, A)) * 0.5).astype(np.float32)
    q[1::2] = coarse[1::2]
    return q


def golden_policies(out, rng, E=4, T_train=48, T_test=24):
    from rl_coach.core_types import RunPhase
    from rl_coach.exploration_policies.bootstrapped import Bootstrapped
    from rl_coach.exploration_policies.ucb import UCB
    from rl_coach.schedules import LinearSchedule
    from rl_coach.spaces import DiscreteActionSpace
    out["pol_E"], out["pol_eps"], out["pol_eval_eps"] = np.int64(E), np.array([0.9, 0.1, 40.0]), np.float64(0.3)
    out["pol_lamb"] = np.float64(0.1)
    resets = np.zeros((T_train + T_test, E), dtype=np.uint8)
    resets[0] = 1
    resets[rng.rand(T_train + T_test, E) < 0.15] = 1
    out["pol_resets"] = resets
    for tag in ("boot", "ucb"):
        q = _q_values(rng, T_train + T_test, E)
        out["pol_%s_q" % tag] = q
        np.random.seed(123)
        pols = []
        for _ in range(E):
            sched = LinearSchedule(0.9, 0.1, 40)
            if tag == "boot":
                pols.append(Bootstrapped(DiscreteActionSpace(A), sched, 0.3, K))
            else:
                pols.append(UCB(DiscreteActionSpace(A), sched, 0.3, K, 0.1))
            pols[-1].change_phase(RunPhase.TRAIN)                 # (a policy starts in the heatup phase)
        acts = np.zeros((T_train + T_test, E), dtype=np.int64)
        lav = np.full((T_train + T_test, E, A), np.nan)
        heads = np.zeros((T_train + T_test, E), dtype=np.int64)
        for t in range(T_train + T_test):
            if t == T_train:
                for p in pols:
                    p.change_phase(RunPhase.TEST)
            for e in range(E):
                if resets[t, e]:
                    pols[e].select_head()
            for e in range(E):
                p = pols[e]
                values = [q[t, e, k][None] for k in range(K)] if p.requires_action_values() else None
                a, _ = p.get_action(values)
                acts[t, e] = a
                heads[t, e] = getattr(p, "selected_head", 0)
                v = p.last_action_values
                if v is not None and not np.isscalar(v):
                    lav[t, e] = np.asarray(v, dtype=np.float64).reshape(-1)
        out["pol_%s_actions" % tag] = acts
        out["pol_%s_last_values" % tag] = lav
        out["pol_%s_heads" % tag] = heads
        out["pol_%s_final_eps" % tag] = np.array([p.epsilon_schedule.current_value for p in pols], dtype=np.float64)
        out["pol_%s_next_rand" % tag] = np.float64(np.random.rand())


def golden_parameters(out):
    from rl_coach.agents.bootstrapped_dqn_agent import BootstrappedDQNAgentParameters
    from rl_coach.exploration_policies.ucb import UCBParameters
    ap = BootstrappedDQNAgentParameters()
    head = ap.network_wrappers['main'].heads_parameters[0]
    out["par_head_copies"] = np.int64(head.num_output_head_copies)
    out["par_rescale"] = np.float64(head.rescale_gradient_from_head_by_factor)
    ex = ap.exploration
    out["par_num_q_heads"] = np.int64(ex.architecture_num_q_heads)
    out["par_share_prob"] = np.float64(ex.bootstrapped_data_sharing_probability)
    s = ex.epsilon_schedule
    out["par_boot_eps"] = np.array([s.initial_value, s.final_value, s.decay_steps], dtype=np.float64)
    out["par_eval_eps"] = np.float64(ex.evaluation_epsilon)
    u = UCBParameters()
    out["par_ucb_lamb"] = np.float64(u.lamb)
    out["par_ucb_eps"] = np.array([[sc.initial_value, sc.final_value, sc.decay_steps, st.num_steps]
                                   for sc, st in u.epsilon_schedule.schedules], dtype=np.float64)
    out["par_ucb_eval_eps"] = np.float64(u.evaluation_epsilon)
    out["par_batch_size"] = np.int64(ap.network_wrappers['main'].batch_size)
    out["par_memory_size"] = np.int64(ap.memory.max_size[1])
    out["par_double_dqn_select"] = np.int64(1)


def main():
    from oracle import ref_loader
    ref_loader.load()
    rng = np.random.RandomState(31337)
    out = {}
    golden_prologue(out, rng)
    golden_masks(out)
    golden_policies(out, rng)
    golden_parameters(out)
    np.savez_compressed(os.path.join(OUT, "bootstrapped.npz"), **out)
    print("bootstrapped", len(out), "arrays")


if __name__ == "__main__":
    main()
