"""Actor-Critic (A3C) throughput: E lock-step streams, observe_batch + train (and choose_actions), and the fused head.

    python tools/bench_a3c.py [--steps 300] [--warmup 50]

Shapes: CartPole_A3C (obs 4, 2 actions, t_max 5, E in {16, 256}) and Atari_A3C (84x84x4 uint8, 6 actions, t_max 20,
E in {16, 64}), seeded synthetic episodes whose ends come with probability 0.02 per step.  Per shape, timed with CUDA
events over ``steps`` lock-steps after ``warmup``: env steps/s (E per lock-step) of observe_batch + train alone and with
choose_actions, learn steps/s, the mean rows per learn step and the padding fraction of the 32-row buckets, and
cb200_actor_critic_head against cb200_nstep_q_head (same rows, features and actions) over 100 launches.

Mujoco_A3C shapes (continuous actions, whole episodes: t_max 10^7, max_episode_steps 1000): Hopper (obs 11, 3 action
dimensions) and Humanoid (obs 376, 17), E in {16, 64}, seeded synthetic episodes that end with probability 0.005 per
step and at the latest after 1000 steps, warmed up over at least 1000 lock-steps (the row buckets and their CUDA
graphs are built the first time a size occurs).  Per shape the same rates with ContinuousEntropy acting, the mean rows per
learn step and the padding of the geometric row buckets, cb200_actor_critic_gaussian_head's time per launch on the
largest bucket over 100 launches, and the device memory the buckets took (network instances, workspaces, graphs).
Prints one JSON line with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_bootstrapped import card      # noqa: E402
from tools.bench_nstep_q import stream, time_call, timed      # noqa: E402

SHAPES = [("cartpole", (4,), 2, 16), ("cartpole", (4,), 2, 256), ("atari", (84, 84, 4), 6, 16),
          ("atari", (84, 84, 4), 6, 64)]
MUJOCO = [("hopper", (11,), 3, 16), ("hopper", (11,), 3, 64), ("humanoid", (376,), 17, 16),
          ("humanoid", (376,), 17, 64)]


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


def mujoco_stream(obs, D, E, n, seed=0, p_end=0.005, cap=1000):
    """a pool of states, actions, rewards and game_overs [n, E]: episodes end with probability p_end, at most cap long"""
    rng = np.random.RandomState(seed)
    dones = rng.rand(n, E) < p_end
    length = np.zeros(E, np.int64)
    for t in range(n):
        length += 1
        dones[t] |= length >= cap
        length[dones[t]] = 0
    return (rng.uniform(-1, 1, (8, E) + obs).astype(np.float32), rng.randn(n, E, D) * 0.3,
            rng.choice([-1.0, 0.0, 1.0], (n, E)) / 20., dones)


def mujoco_run(agent, data, lo, hi, act):
    from coach_b200.memories.lockstep_segments import bucket_rows
    pool, actions, rewards, dones = data
    learns = rows = padded = 0
    for t in range(lo, hi):
        s, s2 = pool[t % 8], pool[(t + 1) % 8]
        if act:
            agent.choose_actions(s)
        agent.observe_batch(s, actions[t], rewards[t], s2, dones[t])
        if isinstance(agent.train(fetch=False), torch.Tensor):
            n = sum(end - start for _, start, end in agent.learned_segments)
            learns, rows, padded = learns + 1, rows + n, padded + bucket_rows(n)
    return learns, rows, padded


def mujoco_timed(agent, data, lo, hi, act):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    res = mujoco_run(agent, data, lo, hi, act)
    e1.record()
    torch.cuda.synchronize()
    return (e0.elapsed_time(e1) / 1e3,) + res


def mujoco(kind, obs, D, E, steps, warmup):
    from coach_b200.agents.actor_critic_agent import ActorCriticAgent
    from coach_b200.presets import Mujoco_A3C as m
    high = np.ones(D, np.float32)
    torch.cuda.synchronize()
    m0 = torch.cuda.memory_allocated()
    agent = ActorCriticAgent(m.agent_params, observation_shape=obs, action_dim=D, action_low=-high, action_high=high,
                             num_envs=E, seed=0, max_episode_steps=m.max_episode_steps)
    torch.cuda.synchronize()
    m1 = torch.cuda.memory_allocated()
    n = warmup + 2 * steps
    data = mujoco_stream(obs, D, E, n)
    mujoco_timed(agent, data, 0, warmup, True)
    sec, learns, rows, padded = mujoco_timed(agent, data, warmup, warmup + steps, False)
    sec_act = mujoco_timed(agent, data, warmup + steps, n, True)[0]
    from coach_b200 import _lib
    B = max(agent._buckets)
    d, st = agent._buckets[B].desc, _lib.current_stream()
    head_us = time_call(lambda: agent.lib.cb200_actor_critic_gaussian_head(ctypes.byref(d), st))
    torch.cuda.synchronize()
    res = {"obs": obs[0], "action_dim": D, "env_steps_per_s": round(E * steps / sec, 1),
           "env_steps_per_s_with_acting": round(E * steps / sec_act, 1), "learn_steps_per_s": round(learns / sec, 1),
           "mean_rows_per_learn_step": round(rows / max(learns, 1), 1),
           "padding_fraction": round(1 - rows / padded, 3) if learns else None, "buckets": len(agent._buckets),
           "head_rows": B, "gaussian_head_us": round(head_us, 2),
           "agent_mb": round((m1 - m0) / 2 ** 20, 1),
           "bucket_mb": round((torch.cuda.memory_allocated() - m1) / 2 ** 20, 1)}
    del agent
    torch.cuda.empty_cache()
    return "mujoco_%s_E%d" % (kind, E), res


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
    for kind, obs, D, E in MUJOCO:
        key, res = mujoco(kind, obs, D, E, args.steps, max(args.warmup, 1000))
        out["shapes"][key] = res
    print(json.dumps(out))


if __name__ == "__main__":
    main()
