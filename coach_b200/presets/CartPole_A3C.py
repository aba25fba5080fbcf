"""rl_coach/presets/CartPole_A3C.py:22-37 (agent parameters; the reference validates it with 8 workers)"""
from coach_b200.agents.actor_critic_agent import ActorCriticAgentParameters, PolicyGradientRescaler
from coach_b200.filters.filter import InputFilter, RewardRescaleFilter

agent_params = ActorCriticAgentParameters()
agent_params.algorithm.policy_gradient_rescaler = PolicyGradientRescaler.GAE
agent_params.algorithm.discount = 0.99
agent_params.algorithm.apply_gradients_every_x_episodes = 1
agent_params.algorithm.num_steps_between_gradient_updates = 5
agent_params.algorithm.gae_lambda = 1
agent_params.algorithm.beta_entropy = 0.01
agent_params.network_wrappers['main'].optimizer_type = 'Adam'
agent_params.network_wrappers['main'].learning_rate = 0.0001
agent_params.input_filter = InputFilter()
agent_params.input_filter.add_reward_filter('rescale', RewardRescaleFilter(1 / 200.))

observation_shape, num_actions, num_envs = (4,), 2, 8
