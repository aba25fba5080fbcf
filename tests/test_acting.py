"""The batched epsilon-greedy of the device acting path against the actions the reference's policy objects (one
EGreedy per environment, all drawing from numpy's global generator in agent order) selected on the same q-value stream
(tests/golden/acting.npz, written by oracle/make_golden_boundary.py).  CPU only."""
import os

import numpy as np
import pytest

from oracle.make_golden_boundary import A, E, T, acting_q


@pytest.mark.parametrize("test_phase", [False, True])
def test_batched_e_greedy_selects_the_reference_actions(test_phase, golden_dir):
    from coach_b200.exploration_policies.e_greedy import BatchedEGreedy, RunPhase
    from coach_b200.schedules import LinearSchedule
    fx = np.load(os.path.join(golden_dir, "acting.npz"))
    phase = "test" if test_phase else "train"
    want = fx["actions_" + phase]
    q = acting_q()
    np.random.seed(11)
    mine = BatchedEGreedy(A, E, LinearSchedule(1.0, 0.1, 25), 0.05)
    mine.change_phase(RunPhase.TEST if test_phase else RunPhase.TRAIN)
    got = np.zeros((T, E), dtype=np.int64)
    for t in range(T):
        got[t], probs = mine.get_actions(q[t])
        assert np.allclose(probs.sum(1), 1.0)
    np.testing.assert_array_equal(got, want)
    assert float(mine.epsilon_schedules[0].current_value) == float(fx["epsilon_" + phase])
