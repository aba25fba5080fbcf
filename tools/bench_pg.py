"""Policy Gradients (REINFORCE) throughput: E lock-step streams, observe_batch + train, and the head and targets kernels.

    python tools/bench_pg.py [--steps 600] [--warmup 200]

Shapes: CartPole_PG (obs 4, 2 actions) and InvertedPendulum_PG (obs 4, one action in [-3, 3]) at E in {16, 64, 256},
seeded synthetic episodes whose lengths are uniform in [10, 200] (CartPole) or [10, 1000] (InvertedPendulum), both
presets' apply_gradients_every_x_episodes = 5 and t_max 20000.  Per shape, timed with CUDA events over ``steps``
lock-steps after ``warmup``: env steps/s (E per lock-step) of observe_batch + train, learn steps/s (one per part of at
most 5 episodes), the mean rows per learn step, the learn-step buckets (network instances / CUDA graphs) the run
created and the peak device memory torch allocated (rollout ring, learn buffers, buckets), and over 100 launches each
cb200_policy_gradient_head and cb200_pg_targets on the agent's largest bucket.  Prints one JSON line with the card's
name and power limit.
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
from tools.bench_nstep_q import time_call      # noqa: E402

SHAPES = [(kind, E) for kind in ("cartpole", "pendulum") for E in (16, 64, 256)]


def make(kind, E):
    from coach_b200.agents.policy_gradients_agent import PolicyGradientsAgent
    if kind == "pendulum":
        from coach_b200.presets import InvertedPendulum_PG as P
        kw = dict(action_dim=P.action_dim, action_low=P.action_low, action_high=P.action_high)
    else:
        from coach_b200.presets import CartPole_PG as P
        kw = dict(num_actions=P.num_actions)
    return PolicyGradientsAgent(P.agent_params, observation_shape=P.observation_shape, num_envs=E, seed=0, **kw)


def stream(kind, E, n, seed=0):
    rng = np.random.RandomState(seed)
    cap = 1000 if kind == "pendulum" else 200
    pool = rng.uniform(-1, 1, (8, E, 4)).astype(np.float32)
    actions = rng.uniform(-3, 3, (n, E, 1)).astype(np.float32) if kind == "pendulum" else rng.randint(0, 2, (n, E))
    dones = np.zeros((n, E), dtype=bool)
    for e in range(E):
        t = -1
        while t < n:
            t += rng.randint(10, cap + 1)
            if t < n:
                dones[t, e] = True
    return pool, actions, rng.choice([0.0, 1.0], (n, E)), dones


def run(agent, data, lo, hi):
    pool, actions, rewards, dones = data
    learns = rows = 0
    for t in range(lo, hi):
        agent.observe_batch(pool[t % 8], actions[t], rewards[t], pool[(t + 1) % 8], dones[t])
        agent.train(fetch=False)
        learns += len(agent.last_parts)
        rows += sum(end - start for _, start, end in agent.learned_segments)
    return learns, rows


def timed(agent, data, lo, hi):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    learns, rows = run(agent, data, lo, hi)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3, learns, rows


def kernels(agent):
    """cb200_policy_gradient_head and cb200_pg_targets on the agent's largest bucket (its last table)"""
    from coach_b200 import _lib
    st = _lib.current_stream()
    B = max(agent._buckets)
    d = agent._buckets[B].desc
    head = time_call(lambda: agent.lib.cb200_policy_gradient_head(ctypes.byref(d), st))
    off, ln = agent.segments.seg_table()
    tg = time_call(lambda: agent.lib.cb200_pg_targets(agent.returns.data_ptr(), off, ln, agent.num_envs, B,
                                                      agent.rescaler, agent.table[0].data_ptr(),
                                                      agent.table[1].data_ptr(), agent.t_max,
                                                      agent.targets.data_ptr(), None, None, st))
    return B, head, tg


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=600)
    ap.add_argument("--warmup", type=int, default=200)
    args = ap.parse_args()
    name, power = card()
    out = {"gpu": name, "power_limit": power, "steps": args.steps, "shapes": {}}
    for kind, E in SHAPES:
        torch.cuda.reset_peak_memory_stats()
        agent = make(kind, E)
        data = stream(kind, E, args.warmup + args.steps)
        timed(agent, data, 0, args.warmup)
        sec, learns, rows = timed(agent, data, args.warmup, args.warmup + args.steps)
        peak = torch.cuda.max_memory_allocated()
        B, head_us, tg_us = kernels(agent)
        out["shapes"]["%s_E%d" % (kind, E)] = {
            "env_steps_per_s": round(E * args.steps / sec, 1), "learn_steps_per_s": round(learns / sec, 1),
            "mean_rows_per_learn_step": round(rows / max(learns, 1), 1), "buckets": len(agent._buckets),
            "peak_device_mb": round(peak / 2 ** 20), "head_rows": B,
            "policy_gradient_head_us": round(head_us, 2), "pg_targets_us": round(tg_us, 2)}
        del agent
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
