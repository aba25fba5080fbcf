"""PAL and Mixed Monte Carlo vs DDQN learn-step throughput, and the fused head launch per target rule.

    python tools/bench_pal_mmc.py [--steps 200] [--repeats 3]

Atari shapes (84x84x4, 6 actions), a 2^16-slot episodic replay filled with ``store_columns`` (episodes of ~100
steps), batch 32 (the preset) and 512.  Agents: DDQN, MMC, PAL.  The agents alternate; each run warms up (eager steps
and the CUDA graph capture) and then times ``steps`` learn steps with CUDA events.  The head launch of each rule is
timed over 100 back-to-back launches.  Prints one JSON line with the card's name and power limit.
"""
import argparse
import ctypes
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from bench_bootstrapped import card, time_steps  # noqa: E402  (tools/ is on sys.path when run as a script)


def make(kind, B):
    from coach_b200.memories.episodic_experience_replay import EpisodicExperienceReplayParameters
    from coach_b200.memories.memory import MemoryGranularity
    if kind == "ddqn":
        from coach_b200.agents.dqn_agent import DDQNAgent as cls, DDQNAgentParameters as P
    elif kind == "mmc":
        from coach_b200.agents.mmc_agent import MixedMonteCarloAgent as cls, MixedMonteCarloAgentParameters as P
    else:
        from coach_b200.agents.pal_agent import PALAgent as cls, PALAgentParameters as P
    ap = P()
    ap.memory = EpisodicExperienceReplayParameters()
    ap.memory.max_size = (MemoryGranularity.Transitions, 1 << 16)
    ap.network_wrappers["main"].batch_size = B
    agent = cls(ap, observation_shape=(84, 84, 4), num_actions=6, seed=0)
    rng = np.random.RandomState(0)
    n, chunk = 1 << 16, 4096
    frames = torch.randint(0, 256, (chunk, 84, 84, 4), dtype=torch.uint8, device="cuda",
                           generator=torch.Generator("cuda").manual_seed(0))
    for i in range(0, n, chunk):
        done = (rng.rand(chunk) < 0.01).astype(np.uint8)
        done[-1] = 1
        agent.memory.store_columns({"state:observation": frames, "next_state:observation": torch.roll(frames, 1, 0),
                                    "action": rng.randint(0, 6, chunk).astype(np.int64),
                                    "reward": rng.randint(-1, 2, chunk).astype(np.float64), "game_over": done})
    return agent


def time_head(agent, rule, n=100):
    from coach_b200 import _lib
    d = agent.head_desc
    saved = d.target_rule
    d.target_rule = rule
    st = _lib.current_stream()
    for _ in range(10):
        _lib.check(agent.lib.cb200_dqn_head_fused(ctypes.byref(d), st))
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        _lib.check(agent.lib.cb200_dqn_head_fused(ctypes.byref(d), st))
    e1.record()
    torch.cuda.synchronize()
    d.target_rule = saved
    return e0.elapsed_time(e1) * 1e3 / n


def main():
    from coach_b200 import _lib
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    name, power = card()
    res = {"gpu": name, "power_limit": power, "steps": args.steps, "steps_per_s": {}, "head_us": {}}
    for B in (32, 512):
        agents = {k: make(k, B) for k in ("ddqn", "mmc", "pal")}
        runs = {k: [] for k in agents}
        for _ in range(args.repeats):
            for k, a in agents.items():                     # alternated
                runs[k].append(round(time_steps(a, args.steps, args.warmup), 1))
        for k in agents:
            res["steps_per_s"]["%s_B%d" % (k, B)] = runs[k]
        # every rule on the PAL agent's descriptor (it carries every input a rule reads)
        for rname, rule in (("dqn", _lib.TARGET_DQN), ("mmc", _lib.TARGET_MMC), ("pal", _lib.TARGET_PAL),
                            ("pal_persistent", _lib.TARGET_PAL_PERSISTENT)):
            res["head_us"]["%s_B%d" % (rname, B)] = round(time_head(agents["pal"], rule), 2)
        del agents
        torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
