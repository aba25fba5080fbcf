"""rl_coach/presets/InvertedPendulum_PG.py:21-31 (agent parameters); InvertedPendulum-v2 has 4-dimensional observations
and one action in [-3, 3] (gym's float32 Box bounds)"""
import numpy as np

from coach_b200.agents.policy_gradients_agent import PolicyGradientsAgentParameters
from coach_b200.filters.filter import InputFilter, ObservationNormalizationFilter, RewardRescaleFilter

agent_params = PolicyGradientsAgentParameters()
agent_params.algorithm.apply_gradients_every_x_episodes = 5
agent_params.algorithm.num_steps_between_gradient_updates = 20000
agent_params.network_wrappers['main'].learning_rate = 0.0005
agent_params.input_filter = InputFilter()
agent_params.input_filter.add_reward_filter('rescale', RewardRescaleFilter(1 / 20.))
agent_params.input_filter.add_observation_filter('observation', 'normalize', ObservationNormalizationFilter())

observation_shape, action_dim = (4,), 1
action_low, action_high = np.full(1, -3, np.float32), np.full(1, 3, np.float32)
