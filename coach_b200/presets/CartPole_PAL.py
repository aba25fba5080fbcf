"""rl_coach/presets/CartPole_PAL.py:22-37 (PAL on CartPole: episodic replay of 40k transitions, MSE loss)"""
from coach_b200.agents.pal_agent import PALAgentParameters
from coach_b200.base_parameters import EnvironmentSteps
from coach_b200.memories.memory import MemoryGranularity

agent_params = PALAgentParameters()
agent_params.algorithm.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(100)
agent_params.algorithm.discount = 0.99
agent_params.algorithm.num_consecutive_playing_steps = EnvironmentSteps(1)
agent_params.network_wrappers['main'].learning_rate = 0.00025
agent_params.network_wrappers['main'].replace_mse_with_huber_loss = False
agent_params.memory.max_size = (MemoryGranularity.Transitions, 40000)

observation_shape, num_actions = (4,), 2
