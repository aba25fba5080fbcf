"""Persistent Advantage Learning learn step on the GPU.  Drop-in for

  rl_coach/agents/pal_agent.py:26-112     parameters, learn_from_batch

The step is the Mixed Monte Carlo step of mmc_agent.py plus one feature forward: the target network on s
(QNetworkWrapper.target_s, beside target(s') on the side stream, over the same input as online(s)).  The fused head then
computes the advantage-learning target of the taken action (cb200_dqn_head_fused, CB200_TARGET_PAL /
CB200_TARGET_PAL_PERSISTENT):

  t = y - alpha * adv               adv = max_a Q_target(s) - Q_target(s, a)
  t = y - alpha * min(adv, nadv)    (persistent)  nadv = max_a Q_target(s') - Q_target(s', a*)
  target = (1 - rho) t + rho R      R = the sample's Monte Carlo return

in the reference's numpy rounding order.  Refused, as for MMC: a prioritized or non-episodic memory, a dueling head, a
network the fused head cannot take.
"""
import torch

from coach_b200 import _lib
from coach_b200.agents.dqn_agent import DQNAgentParameters, DQNAlgorithmParameters
from coach_b200.agents.mmc_agent import MonteCarloTargetAgent
from coach_b200.memories.episodic_experience_replay import EpisodicExperienceReplayParameters


class PALAlgorithmParameters(DQNAlgorithmParameters):
    """pal_agent.py:26-45"""

    def __init__(self):
        super().__init__()
        self.pal_alpha = 0.9
        self.persistent_advantage_learning = False
        self.monte_carlo_mixing_rate = 0.1


class PALAgentParameters(DQNAgentParameters):
    """pal_agent.py:48-56: the DQN parameters with the episodic replay"""

    def __init__(self):
        super().__init__()
        self.algorithm = PALAlgorithmParameters()
        self.memory = EpisodicExperienceReplayParameters()

    @property
    def path(self):
        return 'coach_b200.agents.pal_agent:PALAgent'


class PALAgent(MonteCarloTargetAgent):
    """pal_agent.py:59-112"""
    target_on_s = True

    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, device=None,
                 seed=None):
        alg = agent_parameters.algorithm
        self.alpha = float(alg.pal_alpha)
        self.persistent = bool(alg.persistent_advantage_learning)
        self.target_rule = _lib.TARGET_PAL_PERSISTENT if self.persistent else _lib.TARGET_PAL
        super().__init__(agent_parameters, parent, observation_shape, num_actions, device, seed)

    def _build_head_desc(self):
        super()._build_head_desc()
        d, net = self.head_desc, self.networks["main"]
        d.h_target_s = net.target_s.trunk.acts[-2].data_ptr()
        d.pal_alpha = self.alpha
        self.q_target_s = torch.zeros((self.batch_size, self.num_actions), dtype=torch.float32, device=self.device)
        d.q_target_s = self.q_target_s.data_ptr()
