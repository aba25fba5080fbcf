"""PPO (KL penalty) training-phase throughput against ClippedPPO at the same shape, and the KL head's time.

    python tools/bench_ppo.py [--phases 5] [--warmup 1]

Hopper shape (17-dim observations, 6 action dimensions), Dense(64) / Dense(64) tanh networks, a seeded synthetic
5000-step rollout of 5 episodes of 1000 steps.  PPO trains on it at B = 128 (1 critic epoch, 10 actor epochs of 39
in-order minibatches); ClippedPPO at the same shape and B = 128 (10 shuffled epochs of 39 minibatches, its preset's
other values).  Per agent, the rollout is stored and one ``train()`` phase runs per timed repetition, timed with CUDA
events after ``warmup`` untimed phases (which build the CUDA graphs): training phases/s.  The heads alone:
cb200_ppo_kl_head and cb200_ppo_continuous_head at B = 128 and B = 4096, A = 6, over 1000 launches each (CUDA events).
Prints one JSON line with the card's name and power limit.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_bootstrapped import card      # noqa: E402
from tools.bench_nstep_q import time_call      # noqa: E402

D, A, N, EP = 17, 6, 5000, 1000


def rollout(seed=0):
    rng = np.random.RandomState(seed)
    s = rng.randn(N, D).astype(np.float32)
    a = rng.randn(N, A).astype(np.float32)
    r = rng.randn(N)
    done = np.zeros(N, np.uint8)
    done[EP - 1::EP] = 1
    return {"state:observation": s, "next_state:observation": s, "action": a, "reward": r, "game_over": done}


def make_ppo():
    from coach_b200.agents.ppo_agent import PPOAgent
    from coach_b200.memories.memory import MemoryGranularity
    from coach_b200.presets import Mujoco_PPO as preset
    ap = preset.agent_params
    ap.memory.max_size = (MemoryGranularity.Transitions, 2 * N)
    return PPOAgent(ap, observation_dim=D, action_dim=A, action_low=-1.0, action_high=1.0, seed=0)


def make_clipped():
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgent
    from coach_b200.memories.memory import MemoryGranularity
    from coach_b200.presets import Mujoco_ClippedPPO as preset
    ap = preset.agent_params
    ap.memory.max_size = (MemoryGranularity.Transitions, 2 * N)
    ap.network_wrappers['main'].batch_size = 128
    ap.algorithm.num_consecutive_playing_steps.num_steps = N
    return ClippedPPOAgent(ap, observation_dim=D, action_dim=A, seed=0)


def phases_per_second(agent, cols, phases, warmup):
    def phase():
        agent.memory.store_columns(cols)
        agent.total_steps_counter += N
        agent.train()
    for _ in range(warmup):
        phase()
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(phases):
        # the replay ingest is host work outside the training phase; only train() is timed
        agent.memory.store_columns(cols)
        agent.total_steps_counter += N
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        agent.train()
        e1.record()
        torch.cuda.synchronize()
        total += e0.elapsed_time(e1) / 1e3
    return phases / total


def head_times(B):
    from coach_b200 import _lib
    lib = _lib.load()
    rng = np.random.RandomState(B)
    t = lambda *s: torch.from_numpy(rng.randn(*s).astype(np.float32)).cuda()       # noqa: E731
    mu, ls, act, omu, ols, adv = t(B, A), t(A) * 0.3, t(B, A), t(B, A), t(A) * 0.3, t(B)
    d_mu, d_ls, sc, k = torch.zeros(B, A, device="cuda"), torch.zeros(A, device="cuda"), \
        torch.zeros(5, device="cuda"), torch.tensor([0.2], device="cuda")
    st = _lib.current_stream()
    kl = time_call(lambda: lib.cb200_ppo_kl_head(mu.data_ptr(), ls.data_ptr(), act.data_ptr(), omu.data_ptr(),
                                                 ols.data_ptr(), adv.data_ptr(), B, A, k.data_ptr(), 0.02, 1000.0, 1,
                                                 0.0, d_mu.data_ptr(), d_ls.data_ptr(), sc.data_ptr(), st), n=1000)
    clipped = time_call(lambda: lib.cb200_ppo_continuous_head(mu.data_ptr(), ls.data_ptr(), act.data_ptr(),
                                                              omu.data_ptr(), ols.data_ptr(), adv.data_ptr(), B, A,
                                                              0.2, 0.0, d_mu.data_ptr(), d_ls.data_ptr(),
                                                              sc.data_ptr(), st), n=1000)
    return {"kl_head_us": round(kl, 2), "clipped_head_us": round(clipped, 2)}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--phases", type=int, default=5)
    p.add_argument("--warmup", type=int, default=1)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_ppo.py measures on a GPU; none is visible")
    name, power = card()
    cols = rollout()
    out = {"gpu": name, "power_limit": power, "shape": {"obs": D, "actions": A, "rollout": N, "batch": 128},
           "ppo_phases_per_s": round(phases_per_second(make_ppo(), cols, args.phases, args.warmup), 3),
           "clipped_ppo_phases_per_s": round(phases_per_second(make_clipped(), cols, args.phases, args.warmup), 3),
           "heads": {"B128": head_times(128), "B4096": head_times(4096)}}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
