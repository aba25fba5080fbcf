"""rl_coach/presets/Mujoco_PPO.py:24-37 (agent parameters).  The observation filter normalises observations before they
reach the agent; the caller applies it, as for Mujoco_A3C.  The default shapes are InvertedPendulum-v2's (the preset's
reward-test level): 4-dimensional observations and one action in [-3, 3] (gym's float32 Box bounds)."""
import numpy as np

from coach_b200.agents.ppo_agent import PPOAgentParameters
from coach_b200.base_parameters import Dense
from coach_b200.filters.filter import InputFilter, ObservationNormalizationFilter

agent_params = PPOAgentParameters()
agent_params.network_wrappers['actor'].learning_rate = 5e-5
agent_params.network_wrappers['critic'].learning_rate = 5e-5
for _net in ('actor', 'critic'):
    agent_params.network_wrappers[_net].input_embedders_parameters['observation'].scheme = [Dense(64)]
    agent_params.network_wrappers[_net].middleware_parameters.scheme = [Dense(64)]
agent_params.input_filter = InputFilter()
agent_params.input_filter.add_observation_filter('observation', 'normalize', ObservationNormalizationFilter())
agent_params.algorithm.initial_kl_coefficient = 0.2
agent_params.algorithm.gae_lambda = 1.0

observation_dim, action_dim = 4, 1
action_low, action_high = np.full(1, -3, np.float32), np.full(1, 3, np.float32)
