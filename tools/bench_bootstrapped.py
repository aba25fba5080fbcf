"""Bootstrapped DQN vs DDQN learn-step throughput, and the ensemble head launch vs the DQN head launch.

    python tools/bench_bootstrapped.py [--steps 200] [--repeats 3]

Atari shapes (84x84x4, 6 actions), a 2^16-slot uniform replay, batch 32 (the preset) and 512.  Agents: DDQN and
Bootstrapped DQN with 10 heads at p = 1.0 and 0.5.  The agents alternate; each run warms up (eager steps and the CUDA
graph capture) and then times ``steps`` learn steps with CUDA events.  The head kernels are timed over 100
back-to-back launches.  Prints one JSON line with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def make(kind, B, p=1.0):
    from coach_b200.memories.memory import MemoryGranularity
    if kind == "ddqn":
        from coach_b200.agents.dqn_agent import DDQNAgent as cls, DDQNAgentParameters as P
    else:
        from coach_b200.agents.bootstrapped_dqn_agent import BootstrappedDQNAgent as cls, \
            BootstrappedDQNAgentParameters as P
    ap = P()
    ap.memory.max_size = (MemoryGranularity.Transitions, 1 << 16)
    ap.network_wrappers["main"].batch_size = B
    if kind != "ddqn":
        ap.exploration.bootstrapped_data_sharing_probability = p
    agent = cls(ap, observation_shape=(84, 84, 4), num_actions=6, seed=0)
    rng = np.random.RandomState(0)
    n = 1 << 16
    chunk = 4096
    frames = torch.randint(0, 256, (chunk, 84, 84, 4), dtype=torch.uint8, device="cuda",
                           generator=torch.Generator("cuda").manual_seed(0))
    for i in range(0, n, chunk):
        cols = {"state:observation": frames, "next_state:observation": torch.roll(frames, 1, 0),
                "action": rng.randint(0, 6, chunk).astype(np.int64),
                "reward": rng.randint(-1, 2, chunk).astype(np.float64),
                "game_over": (rng.rand(chunk) < 0.01).astype(np.uint8)}
        if kind != "ddqn":
            cols["info:mask"] = agent.draw_bootstrap_masks(chunk)
        agent.memory.store_columns(cols)
    return agent


def time_steps(agent, steps, warmup):
    for _ in range(warmup):
        agent.learn_from_batch(agent.sample_batch(), fetch=False)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        agent.learn_from_batch(agent.sample_batch(), fetch=False)
    e1.record()
    torch.cuda.synchronize()
    return steps / (e0.elapsed_time(e1) / 1e3)


def time_head(agent, n=100):
    from coach_b200 import _lib
    fn = agent.lib.cb200_ensemble_head_fused if hasattr(agent, "num_heads") else agent.lib.cb200_dqn_head_fused
    d = ctypes.byref(agent.head_desc)
    st = _lib.current_stream()
    for _ in range(10):
        _lib.check(fn(d, st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        _lib.check(fn(d, st))
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / n


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [s.strip() for s in out.split(",")]
        return name, power
    except Exception as exc:                                  # noqa: BLE001
        return torch.cuda.get_device_name(), "unknown (%s)" % exc


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    res = {"gpu": name, "power_limit": power, "steps": args.steps, "steps_per_s": {}, "head_us": {}}
    for B in (32, 512):
        agents = {"ddqn": make("ddqn", B), "boot_p1": make("boot", B, 1.0), "boot_p05": make("boot", B, 0.5)}
        runs = {k: [] for k in agents}
        for _ in range(args.repeats):
            for k, a in agents.items():                     # alternated
                runs[k].append(round(time_steps(a, args.steps, args.warmup), 1))
        for k in agents:
            res["steps_per_s"]["%s_B%d" % (k, B)] = runs[k]
        res["head_us"]["dqn_head_fused_B%d" % B] = round(time_head(agents["ddqn"]), 2)
        res["head_us"]["ensemble_head_fused_K10_B%d" % B] = round(time_head(agents["boot_p05"]), 2)
        del agents
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
