"""rl_coach/presets/CartPole_ClippedPPO.py:27-53 (agent parameters): discrete ClippedPPO on CartPole's 4-dim
observations and 2 actions"""
from coach_b200.agents.clipped_ppo_agent import ClippedPPOAgentParameters
from coach_b200.base_parameters import EnvironmentSteps
from coach_b200.schedules import LinearSchedule

agent_params = ClippedPPOAgentParameters()
agent_params.network_wrappers['main'].learning_rate = 0.0003
agent_params.network_wrappers['main'].hidden_units = 64          # embedder [Dense(64)] + middleware [Dense(64)], tanh
agent_params.network_wrappers['main'].batch_size = 64
agent_params.network_wrappers['main'].optimizer_epsilon = 1e-5
agent_params.network_wrappers['main'].adam_optimizer_beta2 = 0.999
agent_params.algorithm.clip_likelihood_ratio_using_epsilon = 0.2
agent_params.algorithm.clipping_decay_schedule = LinearSchedule(1.0, 0, 1000000)
agent_params.algorithm.beta_entropy = 0
agent_params.algorithm.gae_lambda = 0.95
agent_params.algorithm.discount = 0.99
agent_params.algorithm.optimization_epochs = 10
agent_params.algorithm.estimate_state_value_using_gae = True
agent_params.algorithm.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(2048)

observation_dim, num_actions = 4, 2
