"""N-step Q-learning throughput: E lock-step streams, observe_batch + train (and choose_actions), and the fused head.

    python tools/bench_nstep_q.py [--steps 300] [--warmup 50]

Shapes: CartPole (obs 4, 2 actions, E in {16, 256}) and Atari (84x84x4 uint8, 6 actions, the Atari_NStepQ network,
E in {16, 64}), t_max 5, seeded synthetic episodes whose ends come with probability 0.02 per step.  Per shape, timed
with CUDA events over ``steps`` lock-steps after ``warmup``: env steps/s (E per lock-step) of observe_batch + train
alone and with choose_actions, learn steps/s, the mean rows per learn step and the padding fraction of the 32-row
buckets, and cb200_nstep_q_head against cb200_dqn_head_fused (same rows, features and actions) over 100 launches.
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

SHAPES = [("cartpole", (4,), 2, 16), ("cartpole", (4,), 2, 256), ("atari", (84, 84, 4), 6, 16),
          ("atari", (84, 84, 4), 6, 64)]


def make(kind, obs, A, E):
    from coach_b200.agents.n_step_q_agent import NStepQAgent
    if kind == "atari":
        from coach_b200.presets.Atari_NStepQ import agent_params as ap
    else:
        from coach_b200.presets.CartPole_NStepQ import agent_params as ap
    return NStepQAgent(ap, observation_shape=obs, num_actions=A, num_envs=E, seed=0)


def stream(obs, A, E, n, seed=0):
    rng = np.random.RandomState(seed)
    if len(obs) == 3:
        pool = rng.randint(0, 256, (8, E) + obs).astype(np.uint8)
    else:
        pool = rng.uniform(-1, 1, (8, E) + obs).astype(np.float32)
    return pool, rng.randint(0, A, (n, E)), rng.choice([-1.0, 0.0, 1.0], (n, E)), rng.rand(n, E) < 0.02


def run(agent, data, lo, hi, act):
    from coach_b200.exploration_policies.e_greedy import EGreedyParameters
    pool, actions, rewards, dones = data
    pol = EGreedyParameters().make(agent.num_actions, agent.num_envs)
    learns = rows = bucket_rows = 0
    for t in range(lo, hi):
        s, s2 = pool[t % 8], pool[(t + 1) % 8]
        if act:
            agent.choose_actions(s, pol)
        agent.observe_batch(s, actions[t], rewards[t], s2, dones[t])
        if isinstance(agent.train(fetch=False), torch.Tensor):
            n = sum(end - start for _, start, end in agent.learned_segments)
            learns, rows, bucket_rows = learns + 1, rows + n, bucket_rows + max(32, -(-n // 32) * 32)
    return learns, rows, bucket_rows


def timed(agent, data, lo, hi, act):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    learns, rows, bucket_rows = run(agent, data, lo, hi, act)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3, learns, rows, bucket_rows


def time_call(call, n=100):
    from coach_b200 import _lib
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


def heads(agent):
    """the agent's head on its largest bucket, and cb200_dqn_head_fused on the same rows / features / actions"""
    from coach_b200 import _lib
    st = _lib.current_stream()
    B = max(agent._buckets)
    d = agent._buckets[B].desc
    K, A = d.features, d.n_actions
    ns = time_call(lambda: agent.lib.cb200_nstep_q_head(ctypes.byref(d), st))
    z = lambda *s: torch.rand(*s, device="cuda")                                        # noqa: E731
    keep = dict(h=z(3, B, K), w=z(2, K, A), b=z(2, A), out=z(6, B, A), dh=z(B, K), dw=z(K, A), db=z(A), loss=z(1),
                ws=z(((B + 15) // 16) * 8 * (K * A + A + 1)), td=torch.zeros(B, dtype=torch.float64, device="cuda"),
                a=torch.zeros(B, dtype=torch.int64, device="cuda"), r=torch.zeros(B, dtype=torch.float64,
                                                                                     device="cuda"),
                g=torch.zeros(B, dtype=torch.uint8, device="cuda"))
    q = _lib.DqnHeadDesc()
    q.h_next, q.h_online, q.h_select = (keep["h"][i].data_ptr() for i in range(3))
    q.w_target, q.w_online = keep["w"][0].data_ptr(), keep["w"][1].data_ptr()
    q.b_target, q.b_online = keep["b"][0].data_ptr(), keep["b"][1].data_ptr()
    q.actions, q.rewards, q.game_overs = keep["a"].data_ptr(), keep["r"].data_ptr(), keep["g"].data_ptr()
    q.discount, q.batch, q.features, q.n_actions = 0.99, B, K, A
    q.q_online, q.q_next, q.targets, q.dq = (keep["out"][i].data_ptr() for i in range(4))
    q.td_err, q.loss, q.dh, q.dw, q.db = keep["td"].data_ptr(), keep["loss"].data_ptr(), keep["dh"].data_ptr(), \
        keep["dw"].data_ptr(), keep["db"].data_ptr()
    q.workspace = keep["ws"].data_ptr()
    dq = time_call(lambda: agent.lib.cb200_dqn_head_fused(ctypes.byref(q), st))
    return B, ns, dq


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=300)
    ap.add_argument("--warmup", type=int, default=50)
    args = ap.parse_args()
    name, power = card()
    out = {"gpu": name, "power_limit": power, "steps": args.steps, "shapes": {}}
    for kind, obs, A, E in SHAPES:
        agent = make(kind, obs, A, E)
        n = args.warmup + 2 * args.steps
        data = stream(obs, A, E, n)
        run(agent, data, 0, args.warmup, True)
        sec, learns, rows, bucket_rows = timed(agent, data, args.warmup, args.warmup + args.steps, False)
        sec_act = timed(agent, data, args.warmup + args.steps, n, True)[0]
        B, ns_us, dqn_us = heads(agent)
        mean_rows = rows / max(learns, 1)
        out["shapes"]["%s_E%d" % (kind, E)] = {
            "env_steps_per_s": round(E * args.steps / sec, 1),
            "env_steps_per_s_with_acting": round(E * args.steps / sec_act, 1),
            "learn_steps_per_s": round(learns / sec, 1), "mean_rows_per_learn_step": round(mean_rows, 2),
            "padding_fraction": round(1 - rows / bucket_rows, 3) if learns else None,
            "head_rows": B, "nstep_q_head_us": round(ns_us, 2), "dqn_head_fused_us": round(dqn_us, 2)}
        del agent
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
