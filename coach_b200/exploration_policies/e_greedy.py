"""epsilon-greedy action selection for a batch of rollout shards: rl_coach/exploration_policies/e_greedy.py:80-140 for
DiscreteActionSpace, vectorised over E environments that are stepped in lock-step.

The reference runs one ``EGreedy`` object per agent; all of them draw from numpy's GLOBAL generator, in agent order.
``BatchedEGreedy.get_actions`` consumes that stream in exactly the same order for environments 0 .. E-1 -- per
environment: (exploit) ``np.random.random(A)`` for the random tie-break among the maximal action values, or (explore)
``np.random.choice(actions)``; then ``step_epsilon``'s fresh ``np.random.rand()`` -- so a seeded run selects the same
actions as E reference policies fed the same action values (tests/test_acting.py).  The Q-values come from the device
in one [E, A] read-back (a few hundred bytes); the arithmetic on them is the reference's numpy arithmetic.
"""
import numpy as np

from coach_b200.schedules import LinearSchedule, Schedule


class RunPhase(object):
    HEATUP, TRAIN, TEST = "Heatup", "Training", "Testing"


class EGreedyParameters(object):
    """exploration_policies/e_greedy.py:29-41, discrete action spaces (the continuous fall-back is not carried)"""

    def __init__(self):
        self.epsilon_schedule = LinearSchedule(0.5, 0.01, 50000)
        self.evaluation_epsilon = 0.05

    @property
    def path(self):
        return 'coach_b200.exploration_policies.e_greedy:BatchedEGreedy'

    def make(self, num_actions, num_envs):
        return BatchedEGreedy(num_actions, num_envs, self.epsilon_schedule, self.evaluation_epsilon)


class BatchedEGreedy(object):
    def __init__(self, num_actions: int, num_envs: int, epsilon_schedule: Schedule, evaluation_epsilon: float):
        self.num_actions, self.num_envs = int(num_actions), int(num_envs)
        self.epsilon_schedules = [epsilon_schedule] + [_clone(epsilon_schedule) for _ in range(num_envs - 1)]
        self.evaluation_epsilon = evaluation_epsilon
        self.phase = RunPhase.TRAIN
        # e_greedy.py:78: drawn at construction, one policy after the other
        self.current_random_value = np.array([np.random.rand() for _ in range(self.num_envs)])

    def change_phase(self, phase):
        self.phase = phase

    def epsilon(self, env=0):
        return self.evaluation_epsilon if self.phase == RunPhase.TEST else self.epsilon_schedules[env].current_value

    def requires_action_values(self):
        """e_greedy.py:80-82, per environment"""
        return np.array([self.current_random_value[e] >= self.epsilon(e) for e in range(self.num_envs)])

    def get_actions(self, action_values):
        """action_values [E, A] (numpy / anything np.asarray accepts).  Returns (actions int64 [E],
        probabilities [E, A]) -- e_greedy.py:84-103 applied to environment 0, 1, ... in turn."""
        q = np.asarray(action_values)
        E, A = self.num_envs, self.num_actions
        assert q.shape == (E, A)
        actions = np.zeros(E, dtype=np.int64)
        probs = np.zeros((E, A))
        for e in range(E):
            eps = self.epsilon(e)
            if self.current_random_value[e] < eps:
                actions[e] = np.random.choice(np.arange(A))                              # action_space.sample()
                probs[e] = 1.0 / A
            else:
                v = q[e]
                actions[e] = np.argmax(np.random.random(v.shape) * (np.isclose(v, v.max())))   # random tie-break
                probs[e, actions[e]] = 1
            # step_epsilon (:125-130)
            if self.phase == RunPhase.TRAIN:
                self.epsilon_schedules[e].step()
            self.current_random_value[e] = np.random.rand()
        return actions, probs


def _clone(s):
    import copy
    return copy.deepcopy(s)
