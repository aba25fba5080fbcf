"""Mixed Monte Carlo learn step on the GPU.  Drop-in for

  rl_coach/agents/mmc_agent.py:26-84      parameters, learn_from_batch

The step is the DDQN schedule of dqn_agent.DQNAgent -- replay sample + gather, the feature layers of target(s'),
online(s) and online(s'), one fused head launch, the backward pass below the head, Adam, the same CUDA graphs.  Only the
target of the taken action differs: the double-DQN target mixed with the sample's Monte Carlo return,
(1 - rho) y + rho R (cb200_dqn_head_fused, CB200_TARGET_MMC).  R is the episodic replay's ``n_step_discounted_rewards``
column, computed on the GPU when an episode closes.

``MonteCarloTargetAgent`` is the part MMC and PAL (pal_agent.py) share: the checks, the returns column and the head
descriptor.  The reference never updates PER priorities in these agents and never reads importance weights: a
prioritized memory is refused, as is any memory without Monte Carlo returns.  There is no unfused path: a dueling head
or a network the fused head cannot take is refused too.
"""
import torch

from coach_b200 import _lib
from coach_b200.agents.dqn_agent import DDQNAgent, DQNAgentParameters, DQNAlgorithmParameters
from coach_b200.memories.episodic_experience_replay import EpisodicExperienceReplayParameters
from coach_b200.memories.prioritized_experience_replay import PrioritizedExperienceReplayParameters


class MixedMonteCarloAlgorithmParameters(DQNAlgorithmParameters):
    """mmc_agent.py:26-35"""

    def __init__(self):
        super().__init__()
        self.monte_carlo_mixing_rate = 0.1


class MixedMonteCarloAgentParameters(DQNAgentParameters):
    """mmc_agent.py:38-47: the DQN parameters with the episodic replay"""

    def __init__(self):
        super().__init__()
        self.algorithm = MixedMonteCarloAlgorithmParameters()
        self.memory = EpisodicExperienceReplayParameters()

    @property
    def path(self):
        return 'coach_b200.agents.mmc_agent:MixedMonteCarloAgent'


class MonteCarloTargetAgent(DDQNAgent):
    """a DDQN step whose target of the taken action mixes in the Monte Carlo return (target rule ``target_rule``)"""
    target_rule = _lib.TARGET_MMC

    def __init__(self, agent_parameters, parent=None, observation_shape=None, num_actions=None, device=None,
                 seed=None):
        ap = agent_parameters
        name = type(self).__name__
        if isinstance(ap.memory, PrioritizedExperienceReplayParameters):
            raise NotImplementedError("%s with a prioritized replay: the reference agent never updates priorities nor "
                                      "reads importance weights" % name)
        if not isinstance(ap.memory, EpisodicExperienceReplayParameters):
            raise NotImplementedError("%s needs the episodic replay: its targets read the episodes' Monte Carlo "
                                      "returns (n_step_discounted_rewards)" % name)
        if "DuelingQHead" in getattr(ap.network_wrappers["main"], "heads_parameters", ["QHead"]):
            raise NotImplementedError("%s runs on the fused Q head; a dueling head has no fused path" % name)
        self.mixing_rate = float(ap.algorithm.monte_carlo_mixing_rate)
        super().__init__(agent_parameters, parent, observation_shape, num_actions, device, seed)
        if self.head_desc is None:
            raise NotImplementedError("the fused Q head cannot take this network (feature layer of %s, %d actions)"
                                      % (self.net_def.middleware_units or "the embedder", self.num_actions))

    # ---- the hooks of DQNAgent -----------------------------------------------------------------------------------------
    def _memory_columns(self):
        return {"n_step_discounted_rewards": torch.zeros(self.batch_size, dtype=torch.float64, device=self.device)}

    def _build_head_desc(self):
        super()._build_head_desc()
        d = self.head_desc
        d.target_rule = self.target_rule
        d.mc_mixing_rate = self.mixing_rate
        self.q_select = torch.zeros((self.batch_size, self.num_actions), dtype=torch.float32, device=self.device)
        d.q_select = self.q_select.data_ptr()
        self._head_columns["mc_returns"] = "n_step_discounted_rewards"

    # ---- the learn step ----------------------------------------------------------------------------------------------
    def learn_from_batch(self, batch, fetch=True):
        """-> (total_loss, losses, unclipped_grads), as DQNAgent.learn_from_batch"""
        if "n_step_discounted_rewards" not in batch.columns:
            raise ValueError("the batch carries no Monte Carlo returns (column 'n_step_discounted_rewards'): sample it "
                             "from the episodic replay")
        return super().learn_from_batch(batch, fetch)


class MixedMonteCarloAgent(MonteCarloTargetAgent):
    """mmc_agent.py:50-84: target = (1 - rho) (r + (1 - done) discount Q_target(s', argmax Q_online(s'))) + rho R"""
    target_rule = _lib.TARGET_MMC
