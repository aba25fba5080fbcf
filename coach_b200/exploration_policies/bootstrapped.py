"""Ensemble exploration for Bootstrapped DQN, batched over E environments stepped in lock-step:

  BatchedBootstrapped  <- rl_coach/exploration_policies/bootstrapped.py:41-88
      TRAIN: epsilon-greedy on the values of the head selected for the environment's episode;
      TEST:  epsilon-greedy on the one-hot of the heads' majority vote (np.bincount of their argmaxes, first maximum).
  BatchedUCB           <- rl_coach/exploration_policies/ucb.py:45-90
      TRAIN: epsilon-greedy on mean + lamb * std over the heads;  TEST: on the mean.

Both keep the reference's random-number consumption per environment: the epsilon-greedy draws of
e_greedy.BatchedEGreedy, and (Bootstrapped) ``np.random.randint(num_heads)`` from numpy's global stream whenever the
caller starts an episode of environment e (``select_head(e)``, bootstrapped_dqn_agent.py:53-55).  The values the
epsilon-greedy step reads are computed on the device (cb200_ensemble_action_values, in ``ensemble_mode()``) and read
back as [E, A]; ``ensemble_values`` is the same arithmetic in numpy on host arrays [E, heads, A].
"""
import numpy as np

from coach_b200 import _lib
from coach_b200.base_parameters import EnvironmentSteps
from coach_b200.exploration_policies.e_greedy import BatchedEGreedy, RunPhase
from coach_b200.schedules import LinearSchedule, PieceWiseSchedule


class BootstrappedParameters(object):
    """exploration_policies/bootstrapped.py:26-35 (EGreedyParameters' evaluation epsilon 0.05)"""

    def __init__(self):
        self.architecture_num_q_heads = 10
        self.bootstrapped_data_sharing_probability = 1.0
        self.epsilon_schedule = LinearSchedule(1, 0.01, 1000000)
        self.evaluation_epsilon = 0.05

    @property
    def path(self):
        return 'coach_b200.exploration_policies.bootstrapped:BatchedBootstrapped'

    def make(self, num_actions, num_envs):
        return BatchedBootstrapped(num_actions, num_envs, self.epsilon_schedule, self.evaluation_epsilon,
                                   self.architecture_num_q_heads)


class UCBParameters(BootstrappedParameters):
    """exploration_policies/ucb.py:27-39"""

    def __init__(self):
        super().__init__()
        self.epsilon_schedule = PieceWiseSchedule([
            (LinearSchedule(1, 0.1, 1000000), EnvironmentSteps(1000000)),
            (LinearSchedule(0.1, 0.01, 4000000), EnvironmentSteps(4000000))
        ])
        self.lamb = 0.1

    @property
    def path(self):
        return 'coach_b200.exploration_policies.bootstrapped:BatchedUCB'

    def make(self, num_actions, num_envs):
        return BatchedUCB(num_actions, num_envs, self.epsilon_schedule, self.evaluation_epsilon,
                          self.architecture_num_q_heads, self.lamb)


class BatchedBootstrapped(BatchedEGreedy):
    lamb = 0.0

    def __init__(self, num_actions, num_envs, epsilon_schedule, evaluation_epsilon, architecture_num_q_heads):
        super().__init__(num_actions, num_envs, epsilon_schedule, evaluation_epsilon)
        self.num_heads = int(architecture_num_q_heads)
        self.selected_head = np.zeros(self.num_envs, dtype=np.int32)
        self.last_action_values = [0] * self.num_envs

    def select_head(self, env=0):
        """bootstrapped.py:61-62, at the start of every episode of environment ``env``"""
        self.selected_head[env] = np.random.randint(self.num_heads)

    def ensemble_mode(self):
        return _lib.ENSEMBLE_SELECT if self.phase == RunPhase.TRAIN else _lib.ENSEMBLE_VOTE

    def ensemble_values(self, q):
        """q [E, heads, A] (host) -> the [E, A] values the epsilon-greedy step reads (bootstrapped.py:64-81)"""
        q = np.asarray(q)
        out = np.zeros((self.num_envs, self.num_actions), dtype=np.float32)
        for e in range(self.num_envs):
            if self.phase == RunPhase.TRAIN:
                out[e] = q[e][self.selected_head[e]]
            else:
                counts = np.bincount(np.argmax(q[e], axis=-1))
                out[e] = np.eye(self.num_actions)[np.argmax(counts)]
        return out

    def _observe_values(self, e, v, exploit):
        # the reference's get_all_q_values_for_states hands None to an exploring policy (value_optimization_agent.py:54-58)
        self.last_action_values[e] = v if exploit else None

    def get_actions(self, action_values):
        """action_values [E, A]: ``ensemble_values`` of the heads' outputs.  Returns (actions int64 [E], probabilities)"""
        v = np.asarray(action_values)
        exploit = self.requires_action_values()       # environment e's draw only changes during its own turn below
        for e in range(self.num_envs):
            self._observe_values(e, v[e], bool(exploit[e]))
        return super().get_actions(v)


class BatchedUCB(BatchedBootstrapped):
    def __init__(self, num_actions, num_envs, epsilon_schedule, evaluation_epsilon, architecture_num_q_heads, lamb):
        super().__init__(num_actions, num_envs, epsilon_schedule, evaluation_epsilon, architecture_num_q_heads)
        self.lamb = lamb

    def select_head(self, env=0):
        """ucb.py:58-59: no head to select, no random draw"""

    def ensemble_mode(self):
        return _lib.ENSEMBLE_UCB if self.phase == RunPhase.TRAIN else _lib.ENSEMBLE_MEAN

    def ensemble_values(self, q):
        """q [E, heads, A] (host, float32) -> mean + lamb * std (TRAIN) or mean (TEST) per environment (ucb.py:64-71)"""
        q = np.asarray(q)
        out = np.zeros((self.num_envs, self.num_actions), dtype=np.float32)
        for e in range(self.num_envs):
            mean = np.mean(q[e], axis=0)
            out[e] = mean + self.lamb * np.std(q[e], axis=0) if self.phase == RunPhase.TRAIN else mean
        return out

    def _observe_values(self, e, v, exploit):
        # ucb.py:64-71: only recomputed when the policy exploits; an exploring step keeps the previous values
        if exploit:
            self.last_action_values[e] = v
