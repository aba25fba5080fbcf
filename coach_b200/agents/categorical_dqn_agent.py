"""Categorical DQN (C51) learn step on the GPU -- SURVEY.md 8(f2).  Drop-in for

  rl_coach/agents/categorical_dqn_agent.py:33-165   parameters, z_values, learn_from_batch
  rl_coach/architectures/tensorflow_components/heads/categorical_q_head.py:26-57

The network is the DQN network with a Dense(num_actions * atoms) head.  One learn step = replay sample + gather ->
target(s') and online(s) forward -> ``cb200_c51_head`` (softmax, target action, projection of r + (1 - done) * gamma * z
onto the support in fp64 in the reference's loop order, cross entropy, d loss / d logits) -> backward -> Adam -> tree
update with the taken action's cross entropy.  The head defines its loss itself: the total loss is the SUM of the
[batch, actions] cross-entropy tensor and the importance weights do not enter it (head.py:152-158,
general_network.py:352-360) -- kept.
"""
import numpy as np
import torch

from coach_b200 import _lib
from coach_b200.agents.dqn_agent import DQNAgent, DQNAgentParameters, DQNAlgorithmParameters, DQNNetworkParameters


class CategoricalDQNNetworkParameters(DQNNetworkParameters):
    def __init__(self):
        super().__init__()
        self.heads_parameters = ["CategoricalQHead"]


class CategoricalDQNAlgorithmParameters(DQNAlgorithmParameters):
    """categorical_dqn_agent.py:41-57: v_min / v_max bound the support, atoms is its resolution"""

    def __init__(self):
        super().__init__()
        self.v_min = -10.0
        self.v_max = 10.0
        self.atoms = 51


class CategoricalDQNAgentParameters(DQNAgentParameters):
    def __init__(self):
        super().__init__()
        self.algorithm = CategoricalDQNAlgorithmParameters()
        self.network_wrappers = {"main": CategoricalDQNNetworkParameters()}

    @property
    def path(self):
        return 'coach_b200.agents.categorical_dqn_agent:CategoricalDQNAgent'


class CategoricalDQNAgent(DQNAgent):
    double_q_selection = False       # RainbowDQNAgent's rule: the online network picks the target action

    def __init__(self, agent_parameters, parent=None, **kwargs):
        alg = agent_parameters.algorithm
        z = np.linspace(alg.v_min, alg.v_max, alg.atoms)                                     # categorical_dqn_agent.py:77
        top = (z[-1] - z[0]) / (z[1] - z[0])
        if top > alg.atoms - 1:
            raise ValueError(
                "CategoricalDQNAgent: the support linspace(%r, %r, %d) puts v_max at bin position %r > %d; the reference "
                "agent raises IndexError on the first sample whose projected target reaches v_max" %
                (alg.v_min, alg.v_max, alg.atoms, float(top), alg.atoms - 1))
        super().__init__(agent_parameters, parent, **kwargs)
        alg = self.ap.algorithm
        B, A, N, dev = self.batch_size, self.num_actions, int(alg.atoms), self.device
        self.z_values = z
        self._z = torch.from_numpy(self.z_values).to(dev)
        # the head's own support: float32 constant cast to float64 (categorical_q_head.py:36-37)
        self._z_head = torch.from_numpy(self.z_values.astype(np.float32).astype(np.float64)).to(dev)
        self.loss_rows = torch.zeros((B, A), dtype=torch.float32, device=dev)
        self.q_online = torch.zeros((B, A), dtype=torch.float64, device=dev)
        self.target_actions = torch.zeros(B, dtype=torch.int64, device=dev)

    def _head_outputs(self):
        return self.num_actions * int(self.ap.algorithm.atoms)

    def distribution_prediction_to_q_values(self, prediction):
        """categorical_dqn_agent.py:83-84 (host arrays)"""
        return np.dot(prediction, self.z_values)

    def _bootstrap(self, cols):
        """(discount factor, per-sample bootstrap column or None for 1 - game_over, reward column)"""
        return float(self.ap.algorithm.discount), None, cols["reward"]

    def _head_targets(self, cols, q_next, q_select, q_online, st):
        net = self.networks["main"]
        gamma_n, boot, rewards = self._bootstrap(cols)
        sel = q_select if (self.double_q_selection and q_select is not q_next) else None
        _lib.check(self.lib.cb200_c51_head(
            q_next.data_ptr(), q_online.data_ptr(), sel.data_ptr() if sel is not None else None,
            cols["action"].data_ptr(), rewards.data_ptr(), cols["game_over"].data_ptr(),
            boot.data_ptr() if boot is not None else None, self._z.data_ptr(), gamma_n, self.batch_size,
            self.num_actions, int(self.ap.algorithm.atoms), 0, self.targets.data_ptr(), net.online_s.dq.data_ptr(),
            self.loss_rows.data_ptr(), self.loss_dev.data_ptr(), self.td_err.data_ptr(), self.q_online.data_ptr(),
            self.target_actions.data_ptr(), st))

    def _head_loss_grad(self, weights, st):
        pass          # cb200_c51_head already wrote the loss and d loss / d logits of the training network

    def get_all_q_values_for_states(self, states):
        """categorical_dqn_agent.py:87-94: the head's q_values output, [E, num_actions] float64 on the device"""
        logits = super().get_all_q_values_for_states(states)
        E = int(logits.shape[0])
        q = torch.empty((E, self.num_actions), dtype=torch.float64, device=self.device)
        _lib.check(self.lib.cb200_c51_q_values(logits.data_ptr(), self._z_head.data_ptr(), E * self.num_actions,
                                               int(self.ap.algorithm.atoms), q.data_ptr(), _lib.current_stream()))
        return q
