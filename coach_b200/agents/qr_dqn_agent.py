"""Quantile Regression DQN learn step on the GPU.  Drop-in for

  rl_coach/agents/qr_dqn_agent.py:28-137                                            parameters, learn_from_batch
  rl_coach/architectures/tensorflow_components/heads/quantile_regression_q_head.py:24-71   quantile Huber loss, q_values

The network is the DQN network with a Dense(num_actions * atoms) head whose output is read as [B, A, N] quantiles.  One
learn step = replay sample + gather -> target(s') and online(s) forward -> ``cb200_qr_head`` (Q' = mean quantile, the
target action, the fp64 TD targets, the reference's permuted quantile midpoints, the pairwise quantile Huber loss and
d loss / d quantiles) -> backward -> Adam.  The head defines its loss itself: the total loss is the SUM over the batch
of the per-sample pair sums, divided by N, and no importance weights enter it (quantile_regression_q_head.py:59-62).
The reference never updates priorities nor reads importance weights in this agent: a prioritized replay is refused.
"""
import ctypes

import torch

from coach_b200 import _lib
from coach_b200.agents.dqn_agent import DQNAgent, DQNAgentParameters, DQNAlgorithmParameters, DQNNetworkParameters
from coach_b200.exploration_policies.e_greedy import EGreedyParameters
from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplayParameters
from coach_b200.schedules import LinearSchedule


class QuantileRegressionDQNNetworkParameters(DQNNetworkParameters):
    """qr_dqn_agent.py:28-33"""

    def __init__(self):
        super().__init__()
        self.heads_parameters = ["QuantileRegressionQHead"]
        self.learning_rate = 0.00005
        self.optimizer_epsilon = 0.01 / 32


class QuantileRegressionDQNAlgorithmParameters(DQNAlgorithmParameters):
    """qr_dqn_agent.py:36-50: atoms = N quantiles per action, huber_loss_interval = kappa"""

    def __init__(self):
        super().__init__()
        self.atoms = 200
        self.huber_loss_interval = 1


class QuantileRegressionDQNAgentParameters(DQNAgentParameters):
    """qr_dqn_agent.py:53-63"""

    def __init__(self):
        super().__init__()
        self.algorithm = QuantileRegressionDQNAlgorithmParameters()
        self.network_wrappers = {"main": QuantileRegressionDQNNetworkParameters()}
        self.exploration = EGreedyParameters()
        self.exploration.epsilon_schedule = LinearSchedule(1, 0.01, 1000000)
        self.exploration.evaluation_epsilon = 0.001

    @property
    def path(self):
        return 'coach_b200.agents.qr_dqn_agent:QuantileRegressionDQNAgent'


class QuantileRegressionDQNAgent(DQNAgent):
    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, device=None,
                 seed=None):
        ap = agent_parameters
        if isinstance(ap.memory, PrioritizedExperienceReplayParameters):
            raise NotImplementedError("QuantileRegressionDQNAgent with a prioritized replay: the reference agent never "
                                      "updates priorities (qr_dqn_agent.py:97-137) nor reads importance weights")
        if "DuelingQHead" in getattr(ap.network_wrappers["main"], "heads_parameters", []):
            raise NotImplementedError("QuantileRegressionDQNAgent: the quantile head is a plain Dense(actions x atoms) "
                                      "layer; a dueling head has no quantile form")
        self.atoms = int(ap.algorithm.atoms)
        if not 1 <= self.atoms <= 1024:
            raise ValueError("QuantileRegressionDQNAgent: 1 <= atoms <= 1024 (got %d)" % self.atoms)
        super().__init__(agent_parameters, parent, observation_shape, num_actions, device, seed)
        B, N, dev = self.batch_size, self.atoms, self.device
        self.qr_targets = torch.zeros((B, N), dtype=torch.float32, device=dev)
        self.taus = torch.zeros((B, N), dtype=torch.float32, device=dev)
        self.target_actions = torch.zeros(B, dtype=torch.int64, device=dev)
        self._qr_ws = torch.zeros(B, dtype=torch.float32, device=dev)
        d = _lib.QrHeadDesc()
        d.discount = float(self.ap.algorithm.discount)
        d.kappa = float(self.ap.algorithm.huber_loss_interval)
        d.batch, d.n_actions, d.n_atoms = B, self.num_actions, N
        d.dq, d.loss = self.networks["main"].online_s.dq.data_ptr(), self.loss_dev.data_ptr()
        d.targets, d.taus = self.qr_targets.data_ptr(), self.taus.data_ptr()
        d.target_actions, d.workspace = self.target_actions.data_ptr(), self._qr_ws.data_ptr()
        self.qr_desc = d

    def _head_outputs(self):
        return self.num_actions * self.atoms

    def _head_targets(self, cols, q_next, q_select, q_online, st):
        """one launch: the TD targets, the midpoints, the loss and d loss / d quantiles of the training network"""
        d = self.qr_desc
        d.next, d.online = q_next.data_ptr(), q_online.data_ptr()
        d.actions, d.rewards, d.game_overs = (cols["action"].data_ptr(), cols["reward"].data_ptr(),
                                              cols["game_over"].data_ptr())
        _lib.check(self.lib.cb200_qr_head(ctypes.byref(d), st))

    def _head_loss_grad(self, weights, st):
        pass          # cb200_qr_head already wrote the loss and d loss / d quantiles of the training network

    def get_all_q_values_for_states(self, states):
        """qr_dqn_agent.py:72-80: the mean quantile per action, [E, num_actions] float64 on the device"""
        quantiles = super().get_all_q_values_for_states(states)
        E = int(quantiles.shape[0])
        q = torch.empty((E, self.num_actions), dtype=torch.float64, device=self.device)
        _lib.check(self.lib.cb200_qr_q_values(quantiles.data_ptr(), E * self.num_actions, self.atoms, q.data_ptr(),
                                              _lib.current_stream()))
        return q
