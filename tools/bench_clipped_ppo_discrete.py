"""Discrete ClippedPPO training-phase throughput and the categorical clipped-surrogate head's time.

    python tools/bench_clipped_ppo_discrete.py [--phases 5] [--warmup 1]

Two shapes, each on a seeded synthetic 2048-step rollout of 8 episodes of 256 steps, trained at B = 64 for 10 shuffled
epochs of 32 minibatches with the CartPole_ClippedPPO values: CartPole (4-dim observations, 2 actions) and a wide one
(128-dim observations, Atari's 18 actions).  Per shape, the rollout is stored and one ``train()`` phase runs per timed
repetition, timed with CUDA events after ``warmup`` untimed phases (the first captures the minibatch graph; later
phases replay it): training phases/s.  The head alone: cb200_ppo_categorical_head at A = 18 and B = 64 / 4096 over 1000
launches each (CUDA events).  Prints one JSON line with the card's name and power limit.
"""
import argparse
import copy
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.bench_bootstrapped import card      # noqa: E402
from tools.bench_nstep_q import time_call      # noqa: E402

N, EP = 2048, 256
SHAPES = {"cartpole": (4, 2), "wide": (128, 18)}


def rollout(D, A, seed=0):
    rng = np.random.RandomState(seed)
    s = rng.randn(N, D).astype(np.float32)
    done = np.zeros(N, np.uint8)
    done[EP - 1::EP] = 1
    return {"state:observation": s, "next_state:observation": s, "action": rng.randint(0, A, N).astype(np.int64),
            "reward": rng.randn(N), "game_over": done}


def make_agent(D, A):
    from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgent
    from coach_b200.memories.memory import MemoryGranularity
    from coach_b200.presets import CartPole_ClippedPPO as preset
    ap = copy.deepcopy(preset.agent_params)
    ap.memory.max_size = (MemoryGranularity.Transitions, 2 * N)
    return ClippedPPOAgent(ap, observation_dim=D, num_actions=A, seed=0)


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
    assert agent.graph_captures == 1
    return phases / total


def head_us(B, A=18):
    from coach_b200 import _lib
    lib = _lib.load()
    rng = np.random.RandomState(B)
    z = torch.from_numpy(rng.randn(B, A).astype(np.float32)).cuda()
    q = torch.softmax(z + torch.from_numpy(rng.randn(B, A).astype(np.float32)).cuda() * 0.5, 1)
    act = torch.from_numpy(rng.randint(0, A, B).astype(np.int64)).cuda()
    adv = torch.from_numpy(rng.randn(B).astype(np.float32)).cuda()
    dz, sc, r = torch.zeros(B, A, device="cuda"), torch.zeros(5, device="cuda"), torch.tensor([1.0], device="cuda")
    st = _lib.current_stream()
    return round(time_call(lambda: lib.cb200_ppo_categorical_head(z.data_ptr(), act.data_ptr(), q.data_ptr(),
                                                                  adv.data_ptr(), B, A, 0.2, r.data_ptr(), 0.01,
                                                                  dz.data_ptr(), sc.data_ptr(), st), n=1000), 2)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--phases", type=int, default=5)
    p.add_argument("--warmup", type=int, default=1)
    args = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/bench_clipped_ppo_discrete.py measures on a GPU; none is visible")
    name, power = card()
    out = {"gpu": name, "power_limit": power, "rollout": N, "batch": 64, "epochs": 10, "phases_per_s": {}}
    for key, (D, A) in SHAPES.items():
        out["phases_per_s"][key] = {"obs": D, "actions": A, "value": round(
            phases_per_second(make_agent(D, A), rollout(D, A), args.phases, args.warmup), 3)}
    out["head_us"] = {"A18_B64": head_us(64), "A18_B4096": head_us(4096)}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
