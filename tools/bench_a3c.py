"""Actor-Critic (A3C) throughput: E lock-step streams, observe_batch + train (and choose_actions), and the fused head.

    python tools/bench_a3c.py [--steps 300] [--warmup 50]

Shapes: CartPole_A3C (obs 4, 2 actions, t_max 5, E in {16, 256}) and Atari_A3C (84x84x4 uint8, 6 actions, t_max 20,
E in {16, 64}), seeded synthetic episodes whose ends come with probability 0.02 per step.  Per shape, timed with CUDA
events over ``steps`` lock-steps after ``warmup``: env steps/s (E per lock-step) of observe_batch + train alone and with
choose_actions, learn steps/s, the mean rows per learn step and the padding fraction of the 32-row buckets, and
cb200_actor_critic_head against cb200_nstep_q_head (same rows, features and actions) over 100 launches.  Prints one
JSON line with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_bootstrapped import card      # noqa: E402
from tools.bench_nstep_q import stream, time_call, timed      # noqa: E402

SHAPES = [("cartpole", (4,), 2, 16), ("cartpole", (4,), 2, 256), ("atari", (84, 84, 4), 6, 16),
          ("atari", (84, 84, 4), 6, 64)]


def make(kind, obs, A, E):
    from coach_b200.agents.actor_critic_agent import ActorCriticAgent
    if kind == "atari":
        from coach_b200.presets.Atari_A3C import agent_params as ap
    else:
        from coach_b200.presets.CartPole_A3C import agent_params as ap
    return ActorCriticAgent(ap, observation_shape=obs, num_actions=A, num_envs=E, seed=0)


class _Acting(object):
    """bench_nstep_q.run's agent interface: choose_actions(states, policy) -> A3C's choose_actions(states)"""

    def __init__(self, agent):
        self.agent = agent

    def __getattr__(self, name):
        return getattr(self.agent, name)

    def choose_actions(self, states, _policy):
        return self.agent.choose_actions(states)


def heads(agent):
    """the agent's head on its largest bucket, and cb200_nstep_q_head on the same segment table, rows and features"""
    from coach_b200 import _lib
    st = _lib.current_stream()
    B = max(agent._buckets)
    d = agent._buckets[B].desc
    K, A, E = d.features, d.n_actions, agent.num_envs
    ac = time_call(lambda: agent.lib.cb200_actor_critic_head(ctypes.byref(d), st))
    z = lambda *s: torch.rand(*s, device="cuda")                                        # noqa: E731
    keep = dict(w=z(2, K, A), b=z(2, A), out=z(3, B, A), dh=z(B, K), dw=z(K, A), db=z(A), loss=z(1),
                boot=z(E), ws=z(((E + 3) // 4) * 4 * (K * A + A + 1)))
    q = _lib.NstepQHeadDesc()
    q.h_online, q.h_boot = d.h, d.h_boot
    q.w_target, q.w_online = keep["w"][0].data_ptr(), keep["w"][1].data_ptr()
    q.b_target, q.b_online = keep["b"][0].data_ptr(), keep["b"][1].data_ptr()
    q.actions, q.rewards, q.game_overs = d.actions, d.rewards, d.game_overs
    q.seg_offsets, q.seg_lengths, q.segments, q.rows = d.seg_offsets, d.seg_lengths, d.segments, d.rows
    q.discount, q.horizon, q.features, q.n_actions = 0.99, _lib.NSTEP_NSTEP, K, A
    q.q_online, q.dq, q.targets = (keep["out"][i].data_ptr() for i in range(3))
    q.loss, q.bootstrap, q.dh = keep["loss"].data_ptr(), keep["boot"].data_ptr(), keep["dh"].data_ptr()
    q.dw, q.db, q.workspace = keep["dw"].data_ptr(), keep["db"].data_ptr(), keep["ws"].data_ptr()
    ns = time_call(lambda: agent.lib.cb200_nstep_q_head(ctypes.byref(q), st))
    return B, ac, ns


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    name, power = card()
    out = {"gpu": name, "power_limit": power, "steps": args.steps, "shapes": {}}
    for kind, obs, A, E in SHAPES:
        agent = _Acting(make(kind, obs, A, E))
        n = args.warmup + 2 * args.steps
        data = stream(obs, A, E, n)
        timed(agent, data, 0, args.warmup, True)
        sec, learns, rows, bucket_rows = timed(agent, data, args.warmup, args.warmup + args.steps, False)
        sec_act = timed(agent, data, args.warmup + args.steps, n, True)[0]
        B, ac_us, ns_us = heads(agent.agent)
        out["shapes"]["%s_E%d" % (kind, E)] = {
            "t_max": agent.t_max, "env_steps_per_s": round(E * args.steps / sec, 1),
            "env_steps_per_s_with_acting": round(E * args.steps / sec_act, 1),
            "learn_steps_per_s": round(learns / sec, 1), "mean_rows_per_learn_step": round(rows / max(learns, 1), 2),
            "padding_fraction": round(1 - rows / bucket_rows, 3) if learns else None,
            "head_rows": B, "actor_critic_head_us": round(ac_us, 2), "nstep_q_head_us": round(ns_us, 2)}
        del agent
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
