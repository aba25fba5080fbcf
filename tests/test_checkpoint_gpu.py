"""Checkpoint / restore (coach_b200/checkpoint.py; reference conventions graph_manager.py:616-658, checkpoint.py:115-155,
shared_running_stats.py:170-189): a restored agent continues bit-identically."""
import os
import pickle
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _dqn(seed=0, B=128):
    from coach_b200.agents.dqn_agent import DDQNAgent, DDQNAgentParameters
    from coach_b200.memories.memory import MemoryGranularity
    from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplayParameters
    from coach_b200.schedules import LinearSchedule
    ap = DDQNAgentParameters()
    ap.memory = PrioritizedExperienceReplayParameters()
    ap.memory.beta = LinearSchedule(0.4, 1, 1000)
    ap.memory.max_size = (MemoryGranularity.Transitions, 1024)
    ap.network_wrappers["main"].batch_size = B
    return DDQNAgent(ap, observation_shape=(84, 84, 4), num_actions=6, seed=seed)


def _fill(agent, n, seed):
    rng = np.random.RandomState(seed)
    agent.memory.store_columns({"state:observation": rng.randint(0, 256, (n, 84, 84, 4)).astype(np.uint8),
                                "next_state:observation": rng.randint(0, 256, (n, 84, 84, 4)).astype(np.uint8),
                                "action": rng.randint(0, 6, n).astype(np.int64),
                                "reward": rng.randint(-1, 2, n).astype(np.float64),
                                "game_over": (rng.rand(n) < 0.1).astype(np.uint8)})
    agent.memory.update_priorities(np.arange(n), np.abs(rng.randn(n)))


def _steps(agent, k, seed):
    out = []
    for i in range(k):
        random.seed(seed + i)
        np.random.seed(seed + i)
        batch = agent.sample_batch()
        out.append((agent.learn_from_batch(batch)[0], batch.info("idx").clone()))
    torch.cuda.synchronize()
    return out


def _as_legacy_format(agent, path, name):
    """rewrites a DQN checkpoint the way it was written while eager agents kept their Adam powers on the host: the
    advanced powers in the metadata, the device copy (adam_state.npy) at its initial betas.  Returns the powers."""
    import json
    prefix = os.path.join(path, name)
    state = prefix + ".net_main.adam_state.npy"
    powers = np.load(state)
    p = agent.networks["main"].params
    np.save(state, np.array([p.adam_optimizer_beta1, p.adam_optimizer_beta2], dtype=np.float32))
    with open(prefix + ".agent.json") as f:
        meta = json.load(f)
    meta["networks"]["main"]["host"] = {"beta1_power": float(powers[0]), "beta2_power": float(powers[1])}
    with open(prefix + ".agent.json", "w") as f:
        json.dump(meta, f)
    return powers


def test_dqn_agent_continues_bit_identically_after_restore(tmp_path):
    _check_continuation(tmp_path, B=128, legacy=False)


@pytest.mark.parametrize("legacy", [False, True], ids=["current_format", "legacy_format"])
def test_eager_dqn_agent_continues_bit_identically_after_restore(tmp_path, legacy):
    """B = 32: every step eager (Adam's step state on the device as in the CUDA-graph steps)"""
    _check_continuation(tmp_path, B=32, legacy=legacy)


def _check_continuation(tmp_path, B, legacy):
    from coach_b200 import checkpoint
    a = _dqn(B=B)
    _fill(a, 700, 1)                                   # ring not full: only the live rows are written
    _steps(a, 4, 50)                                   # B = 128: eager steps + CUDA-graph capture + a replay
    assert (a._graphs is not None) == (B >= 128)
    a.total_steps_counter = 1234
    name = checkpoint.save_checkpoint(a, str(tmp_path), checkpoint_id=3)
    assert name == "3_Step-1234.ckpt" and checkpoint.read_state_file(str(tmp_path)) == name
    adam_state = a.networks["main"].adam_state.clone()
    if legacy:
        powers = _as_legacy_format(a, str(tmp_path), name)
        assert np.array_equal(powers, adam_state.cpu().numpy()) and powers[0] < np.float32(0.9)
    want = _steps(a, 3, 80)
    theta_want = a.net_def.store.theta.clone()
    tree_want = a.memory.sum_tree.clone()
    b = _dqn(seed=99, B=B)                             # different initial weights, empty replay
    checkpoint.restore_checkpoint(b, str(tmp_path))
    assert b.total_steps_counter == 1234 and b.memory.num_transitions() == a.memory.num_transitions()
    assert torch.equal(b.networks["main"].adam_state, adam_state)
    got = _steps(b, 3, 80)
    for (lw, iw), (lg, ig) in zip(want, got):
        assert lw == lg and torch.equal(iw, ig)
    assert torch.equal(b.net_def.store.theta, theta_want) and torch.equal(b.memory.sum_tree, tree_want)
    assert torch.equal(b.networks["main"].adam_state, a.networks["main"].adam_state)
    assert float(b.memory.beta.current_value) == float(a.memory.beta.current_value)
    with pytest.raises(FileNotFoundError):
        checkpoint.restore_checkpoint(b, str(tmp_path / "nothing_here"))


def test_running_stats_use_the_reference_pickle_format(tmp_path):
    from coach_b200.filters.filter import DeviceRunningStats
    st = DeviceRunningStats("cuda")
    st.set_params(shape=[17], clip_values=(-5.0, 5.0))
    x = torch.randn(300, 17, device="cuda") * 3 + 1
    st.push(x)
    st.save_state_to_checkpoint(str(tmp_path), "7_Step-10.ckpt.observation.normalize_observation")
    path = os.path.join(str(tmp_path), "7_Step-10.ckpt.observation.normalize_observation.srs")
    with open(path, "rb") as f:
        d = pickle.load(f)
    assert set(d) == {"_mean", "_std", "_count", "_sum", "_sum_squares"}           # shared_running_stats.py:171-175
    st2 = DeviceRunningStats("cuda")
    st2.set_params(shape=[17], clip_values=(-5.0, 5.0))
    st2.restore_state_from_checkpoint(str(tmp_path), "7_Step-10.ckpt.observation.normalize_observation")
    assert st2._count == st._count and torch.equal(st2._mean, st._mean) and torch.equal(st2._std, st._std)
    q = torch.randn(8, 17, device="cuda")
    assert torch.equal(st2.normalize(q), st.normalize(q))
