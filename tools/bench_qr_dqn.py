"""Quantile Regression DQN vs C51 vs DQN learn-step throughput, and the QR head launch vs the C51 head launch.

    python tools/bench_qr_dqn.py [--steps 200] [--repeats 3]

Atari shapes (84x84x4, 6 actions), a 2^16-slot uniform replay, batch 32 (the preset) and 512.  Agents: QR-DQN with
200 quantiles, C51 with 51 atoms and DQN.  The agents alternate; each run warms up (eager steps and the CUDA graph
capture) and then times ``steps`` learn steps with CUDA events.  The head kernels (cb200_qr_head, cb200_c51_head) are
timed over 100 back-to-back launches on the agents' own last batch.  Prints one JSON line with the card's name and
power limit.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_bootstrapped import card, time_steps      # noqa: E402


def make(kind, B):
    from coach_b200.memories.memory import MemoryGranularity
    if kind == "dqn":
        from coach_b200.agents.dqn_agent import DQNAgent as cls, DQNAgentParameters as P
    elif kind == "c51":
        from coach_b200.agents.categorical_dqn_agent import CategoricalDQNAgent as cls, \
            CategoricalDQNAgentParameters as P
    else:
        from coach_b200.agents.qr_dqn_agent import QuantileRegressionDQNAgent as cls, \
            QuantileRegressionDQNAgentParameters as P
    ap = P()
    ap.memory.max_size = (MemoryGranularity.Transitions, 1 << 16)
    ap.network_wrappers["main"].batch_size = B
    agent = cls(ap, observation_shape=(84, 84, 4), num_actions=6, seed=0)
    rng = np.random.RandomState(0)
    n = 1 << 16
    chunk = 4096
    frames = torch.randint(0, 256, (chunk, 84, 84, 4), dtype=torch.uint8, device="cuda",
                           generator=torch.Generator("cuda").manual_seed(0))
    for i in range(0, n, chunk):
        agent.memory.store_columns({"state:observation": frames, "next_state:observation": torch.roll(frames, 1, 0),
                                    "action": rng.randint(0, 6, chunk).astype(np.int64),
                                    "reward": rng.randint(-1, 2, chunk).astype(np.float64),
                                    "game_over": (rng.rand(chunk) < 0.01).astype(np.uint8)})
    return agent


def time_head(agent, n=100):
    """the agent's head launch on its last batch (the inputs the learn step left in place)"""
    from coach_b200 import _lib
    st = _lib.current_stream()
    net = agent.networks["main"]
    cols = agent.batch_buffers
    if hasattr(agent, "qr_desc"):
        d = ctypes.byref(agent.qr_desc)
        call = lambda: agent.lib.cb200_qr_head(d, st)                                   # noqa: E731
    else:
        call = lambda: agent._head_targets(cols, net.target_s2.q, None, net.online_s.q, st) or 0   # noqa: E731
    for _ in range(10):
        _lib.check(call())
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        _lib.check(call())
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    res = {"gpu": name, "power_limit": power, "steps": args.steps, "steps_per_s": {}, "head_us": {}}
    for B in (32, 512):
        agents = {"qr_dqn_N200": make("qr", B), "c51": make("c51", B), "dqn": make("dqn", B)}
        runs = {k: [] for k in agents}
        for _ in range(args.repeats):
            for k, a in agents.items():                     # alternated
                runs[k].append(round(time_steps(a, args.steps, args.warmup), 1))
        for k in agents:
            res["steps_per_s"]["%s_B%d" % (k, B)] = runs[k]
        res["head_us"]["qr_head_N200_B%d" % B] = round(time_head(agents["qr_dqn_N200"]), 2)
        res["head_us"]["c51_head_N51_B%d" % B] = round(time_head(agents["c51"]), 2)
        del agents
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
