"""rl_coach/presets/CartPole_NStepQ.py:17-27 (agent parameters; the reference validates it with 8 workers)"""
from coach_b200.agents.n_step_q_agent import NStepQAgentParameters
from coach_b200.base_parameters import EnvironmentSteps
from coach_b200.filters.filter import InputFilter, RewardRescaleFilter

agent_params = NStepQAgentParameters()
agent_params.algorithm.discount = 0.99
agent_params.network_wrappers['main'].learning_rate = 0.0001
agent_params.algorithm.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(100)
agent_params.input_filter = InputFilter()
agent_params.input_filter.add_reward_filter('rescale', RewardRescaleFilter(1 / 200.))

observation_shape, num_actions, num_envs = (4,), 2, 8
