"""rl_coach/presets/Atari_A3C.py:22-29 (agent parameters)"""
from coach_b200.agents.actor_critic_agent import ActorCriticAgentParameters
from coach_b200.base_parameters import MiddlewareParameters

agent_params = ActorCriticAgentParameters()
agent_params.algorithm.apply_gradients_every_x_episodes = 1
agent_params.algorithm.num_steps_between_gradient_updates = 20
agent_params.algorithm.beta_entropy = 0.05
agent_params.network_wrappers['main'].middleware_parameters = MiddlewareParameters()
agent_params.network_wrappers['main'].learning_rate = 0.0001

observation_shape, num_actions = (84, 84, 4), 6
