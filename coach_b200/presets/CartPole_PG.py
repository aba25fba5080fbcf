"""rl_coach/presets/CartPole_PG.py:22-34 (agent parameters)"""
from coach_b200.agents.policy_gradients_agent import PolicyGradientsAgentParameters
from coach_b200.filters.filter import InputFilter, RewardRescaleFilter

agent_params = PolicyGradientsAgentParameters()
agent_params.algorithm.discount = 0.99
agent_params.algorithm.apply_gradients_every_x_episodes = 5
agent_params.algorithm.num_steps_between_gradient_updates = 20000
agent_params.network_wrappers['main'].optimizer_type = 'Adam'
agent_params.network_wrappers['main'].learning_rate = 0.0005
agent_params.input_filter = InputFilter()
agent_params.input_filter.add_reward_filter('rescale', RewardRescaleFilter(1 / 200.))

observation_shape, num_actions = (4,), 2
