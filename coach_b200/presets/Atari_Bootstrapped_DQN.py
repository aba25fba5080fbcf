"""rl_coach/presets/Atari_Bootstrapped_DQN.py:16-17 (Bootstrapped DQN on Atari, uniform replay, Bootstrapped
exploration)"""
from coach_b200.agents.bootstrapped_dqn_agent import BootstrappedDQNAgentParameters

agent_params = BootstrappedDQNAgentParameters()
agent_params.network_wrappers['main'].learning_rate = 0.00025

observation_shape, num_actions = (84, 84, 4), 6
