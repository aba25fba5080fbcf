"""rl_coach/presets/CartPole_QR_DQN.py:24-42"""
from coach_b200.agents.qr_dqn_agent import QuantileRegressionDQNAgentParameters
from coach_b200.base_parameters import EnvironmentSteps
from coach_b200.memories.memory import MemoryGranularity
from coach_b200.schedules import LinearSchedule

agent_params = QuantileRegressionDQNAgentParameters()
agent_params.algorithm.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(100)
agent_params.algorithm.discount = 0.99
agent_params.algorithm.num_consecutive_playing_steps = EnvironmentSteps(1)
agent_params.algorithm.atoms = 50
agent_params.network_wrappers['main'].learning_rate = 0.0005
agent_params.memory.max_size = (MemoryGranularity.Transitions, 40000)
agent_params.exploration.epsilon_schedule = LinearSchedule(1.0, 0.01, 10000)

observation_shape, num_actions = (4,), 2
