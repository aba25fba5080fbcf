"""NAF learn-step throughput through train() and the fused head launch.

    python tools/bench_naf.py [--calls 100] [--warmup 4]

Mujoco_NAF agents (embedder and middleware Dense(200), ClipByValue(1000), batch 32) at the Hopper (11 / 3),
HalfCheetah (17 / 6) and Humanoid (376 / 17) shapes, each on a 1M-transition episodic replay filled with
``store_columns`` (episodes of 1000 steps).  ``train()`` runs the reference's 5 learn steps per call and the polyak
update after the first; ``calls`` calls are timed with CUDA events after ``warmup`` calls (eager steps and the CUDA
graph capture).  At batch 32 these steps are launch- and latency-bound: a few dozen microsecond kernels per step,
replayed as one CUDA graph.  The head launch is timed over 200 back-to-back launches.  One JSON line per shape, with
the card's name and power limit read in the same run.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_bootstrapped import card  # noqa: E402  (tools/ is on sys.path when run as a script)

SHAPES = {"hopper": (11, 3), "halfcheetah": (17, 6), "humanoid": (376, 17)}
N = 1 << 20


def make(D, A):
    import copy
    from coach_b200.agents.naf_agent import NAFAgent
    from coach_b200.memories.memory import MemoryGranularity
    from coach_b200.presets import Mujoco_NAF
    ap = copy.deepcopy(Mujoco_NAF.agent_params)
    ap.memory.max_size = (MemoryGranularity.Transitions, N)
    agent = NAFAgent(ap, observation_dim=D, action_dim=A, seed=0)
    rng = np.random.RandomState(0)
    chunk = 1 << 16
    for i in range(0, N, chunk):
        done = np.zeros(chunk, np.uint8)
        done[999::1000] = 1
        done[-1] = 1
        agent.memory.store_columns({"state:observation": rng.randn(chunk, D).astype(np.float32),
                                    "next_state:observation": rng.randn(chunk, D).astype(np.float32),
                                    "action": rng.uniform(-1, 1, (chunk, A)).astype(np.float32),
                                    "reward": rng.randn(chunk), "game_over": done})
    return agent


def time_train(agent, calls, warmup):
    for _ in range(warmup):
        agent.total_steps_counter += 1
        agent.train(fetch=False)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        agent.total_steps_counter += 1
        agent.train(fetch=False)
    e1.record()
    torch.cuda.synchronize()
    steps = calls * agent.ap.algorithm.num_consecutive_training_steps
    return steps / (e0.elapsed_time(e1) / 1e3)


def time_head(agent, n=200):
    from coach_b200 import _lib
    d = ctypes.byref(agent.head_desc)
    st = _lib.current_stream()
    for _ in range(10):
        _lib.check(agent.lib.cb200_naf_head(d, st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        _lib.check(agent.lib.cb200_naf_head(d, st))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=4)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_naf.py measures the GPU: no CUDA device")
    name, power = card()
    for shape, (D, A) in SHAPES.items():
        agent = make(D, A)
        rates = [round(time_train(agent, args.calls, args.warmup), 1) for _ in range(args.repeats)]
        best = max(rates)
        print(json.dumps({"gpu": name, "power_limit": power, "shape": shape, "obs": D, "actions": A,
                          "batch": agent.B, "learn_steps_per_s": rates, "us_per_step": round(1e6 / best, 1),
                          "kernels_per_learn_step": agent._graph_step.launches, "head_us": round(time_head(agent), 2)}))
        del agent
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
