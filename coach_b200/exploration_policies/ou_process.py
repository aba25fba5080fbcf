"""Ornstein-Uhlenbeck exploration for a batch of rollout shards: rl_coach/exploration_policies/ou_process.py:29-84,
vectorised over E environments that are stepped in lock-step.

The reference runs one ``OUProcess`` object per agent; all of them draw from numpy's GLOBAL generator, in agent order.
``BatchedOUProcess.get_actions`` consumes that stream in the same order for environments 0 .. E-1, one
``np.random.randn(A)`` per environment in the TRAIN phase and none otherwise, and evaluates the reference's numpy
expression on each environment's state, so a seeded run returns the same actions as E reference policies fed the same
means (tests/test_naf_host.py).
"""
import numpy as np

from coach_b200.exploration_policies.e_greedy import RunPhase


class OUProcessParameters(object):
    def __init__(self):
        self.mu = 0
        self.theta = 0.15
        self.sigma = 0.2
        self.dt = 0.01

    @property
    def path(self):
        return 'coach_b200.exploration_policies.ou_process:BatchedOUProcess'


class BatchedOUProcess(object):
    def __init__(self, action_dim: int, num_envs: int, mu: float = 0, theta: float = 0.15, sigma: float = 0.2,
                 dt: float = 0.01):
        self.action_dim, self.num_envs = int(action_dim), int(num_envs)
        shape = (self.action_dim,)
        self.mu = float(mu) * np.ones(shape)
        self.theta = float(theta)
        self.sigma = float(sigma) * np.ones(shape)
        self.dt = dt
        self.state = [np.zeros(shape) for _ in range(self.num_envs)]
        self.phase = RunPhase.TRAIN

    def change_phase(self, phase):
        self.phase = phase

    def reset(self, env=None):
        """zeroes the state of environment ``env`` (of every environment when None)"""
        for e in (range(self.num_envs) if env is None else [env]):
            self.state[e] = np.zeros((self.action_dim,))

    def _noise(self, e):
        x = self.state[e]
        dx = self.theta * (self.mu - x) * self.dt + self.sigma * np.random.randn(len(x)) * np.sqrt(self.dt)
        self.state[e] = x + dx
        return self.state[e]

    def get_actions(self, action_values):
        """action_values [E, A] (the policy means).  Returns the actions [E, A]: ou_process.py:69-77 applied to
        environment 0, 1, ... in turn."""
        q = np.asarray(action_values)
        E, A = self.num_envs, self.action_dim
        assert q.shape == (E, A), q.shape
        out = np.zeros((E, A))
        for e in range(E):
            noise = self._noise(e) if self.phase == RunPhase.TRAIN else np.zeros((A,))
            out[e] = q[e].squeeze() + noise
        return out
