"""rl_coach/presets/Atari_QR_DQN.py:10-12 (Quantile Regression DQN on Atari, uniform replay)"""
from coach_b200.agents.qr_dqn_agent import QuantileRegressionDQNAgentParameters

agent_params = QuantileRegressionDQNAgentParameters()
agent_params.network_wrappers['main'].learning_rate = 0.00005       # called alpha in the paper
agent_params.algorithm.huber_loss_interval = 1                     # k = 0: strict quantile loss, k = 1: Huber

observation_shape, num_actions = (84, 84, 4), 6
