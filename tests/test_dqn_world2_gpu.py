"""Two-rank DQN learn step (gloo process group, both ranks on cuda:0).  The gradient all-reduce sits between the backward
and the optimizer part of the step: with identical shards the sum g + g and the 1/2 rescale are exact, so both ranks
must reproduce a one-rank run bit for bit (a wrong scale, a missing join or Adam reading a half-reduced buffer shows);
with different shards the ranks must stay in lock-step and differ from rank 0 training alone (the exchange happened)."""
import functools
import os
import random
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu

CASES = {"plain_head": dict(dueling=False, double=False, clip=None, middleware=True),
         "dueling_clip10": dict(dueling=True, double=True, clip=10.0, middleware=False)}
DATA_SEED = 3


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _run(case, data_seed):
    """6 learn steps (2 eager, CUDA-graph capture, 3 replays) of a B = 128 image DQN + PER agent: losses, gradient
    norms, final parameters and sum tree"""
    from test_learn_gpu import _make_agent
    c = CASES[case]
    torch.manual_seed(0)
    agent = _make_agent((84, 84, 4), 6, 128, c["dueling"], c["double"], True, c["clip"], True, seed=5,
                        middleware=c["middleware"])
    rng = np.random.RandomState(data_seed)
    n = 512
    agent.memory.store_columns({
        "state:observation": rng.randint(0, 256, (n, 84, 84, 4)).astype(np.uint8),
        "next_state:observation": rng.randint(0, 256, (n, 84, 84, 4)).astype(np.uint8),
        "action": rng.randint(0, 6, n).astype(np.int64), "reward": rng.randint(-1, 2, n).astype(np.float64),
        "game_over": (rng.rand(n) < 0.1).astype(np.uint8)})
    agent.memory.update_priorities(np.arange(n), np.abs(rng.randn(n)))
    losses, norms = [], []
    for step in range(6):
        random.seed(20 + step)
        np.random.seed(20 + step)
        loss, _, gnorm = agent.learn_from_batch(agent.sample_batch())
        losses.append(loss)
        norms.append(gnorm)
    torch.cuda.synchronize()
    assert agent._graphs is not None
    return losses, norms, agent.net_def.store.theta.cpu().numpy(), agent.memory.sum_tree.cpu().numpy()


@functools.lru_cache(maxsize=None)
def _one_rank(case):
    return _run(case, DATA_SEED)


def _worker(rank, port, case, shard_by_rank, out_q):
    os.environ.update(RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK="0", MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    try:
        from coach_b200 import parallel
        assert parallel.init_from_env(backend="gloo") == (rank, 2)
        out_q.put((rank, _run(case, DATA_SEED + rank if shard_by_rank else DATA_SEED)))
        torch.distributed.destroy_process_group()
    except BaseException as exc:
        out_q.put((rank, "rank %d failed: %r" % (rank, exc)))
        raise


def _two_ranks(case, shard_by_rank):
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, port, case, shard_by_rank, q)) for r in range(2)]
    try:
        for p in procs:
            p.start()
        res = dict(q.get(timeout=600) for _ in procs)
        for r in range(2):
            assert not isinstance(res[r], str), res[r]
        for p in procs:
            p.join(timeout=120)
            assert p.exitcode == 0
    finally:
        for p in procs:
            if p.pid is not None:
                if p.is_alive():
                    p.terminate()
                p.join(timeout=30)
    return res[0], res[1]


def _equal(a, b):
    la, na, ta, sa = a
    lb, nb, tb, sb = b
    return la == lb and na == nb and np.array_equal(ta, tb) and np.array_equal(sa, sb)


@pytest.mark.parametrize("case", sorted(CASES))
def test_two_ranks_on_identical_shards_match_one_rank(case):
    r0, r1 = _two_ranks(case, shard_by_rank=False)
    assert _equal(r0, r1), "the ranks diverged"
    assert _equal(r0, _one_rank(case)), "two ranks on identical shards differ from one rank"


@pytest.mark.parametrize("case", sorted(CASES))
def test_two_ranks_on_different_shards_stay_in_lock_step(case):
    r0, r1 = _two_ranks(case, shard_by_rank=True)
    assert np.array_equal(r0[2], r1[2]), "the ranks' parameters diverged"
    assert not np.array_equal(r0[2], _one_rank(case)[2]), "rank 0 trained as if alone: no gradient exchange"
