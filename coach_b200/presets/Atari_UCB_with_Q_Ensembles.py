"""rl_coach/presets/Atari_UCB_with_Q_Ensembles.py:8-10 (Bootstrapped DQN on Atari with UCB exploration over the Q
ensemble)"""
from coach_b200.agents.bootstrapped_dqn_agent import BootstrappedDQNAgentParameters
from coach_b200.exploration_policies.bootstrapped import UCBParameters

agent_params = BootstrappedDQNAgentParameters()
agent_params.network_wrappers['main'].learning_rate = 0.00025
agent_params.exploration = UCBParameters()

observation_shape, num_actions = (84, 84, 4), 6
