"""rl_coach/presets/Mujoco_A3C.py:24-34 (agent parameters; the reference validates it with 8 workers on its reward-test
level inverted_pendulum).  Segments are whole episodes: t_max is 10^7 and the mujoco_v2 levels end every episode within
their 1000-step time limit, so the rollout ring holds max_episode_steps rows per stream.  The default shapes are
InvertedPendulum-v2's: 4-dimensional observations and one action in [-3, 3] (gym's float32 Box bounds)."""
import numpy as np

from coach_b200.agents.actor_critic_agent import ActorCriticAgentParameters
from coach_b200.filters.filter import InputFilter, ObservationNormalizationFilter, RewardRescaleFilter

agent_params = ActorCriticAgentParameters()
agent_params.algorithm.apply_gradients_every_x_episodes = 1
agent_params.algorithm.num_steps_between_gradient_updates = 10000000
agent_params.algorithm.beta_entropy = 0.0001
agent_params.network_wrappers['main'].learning_rate = 0.00001
agent_params.input_filter = InputFilter()
agent_params.input_filter.add_reward_filter('rescale', RewardRescaleFilter(1 / 20.))
agent_params.input_filter.add_observation_filter('observation', 'normalize', ObservationNormalizationFilter())

observation_shape, action_dim = (4,), 1
action_low, action_high = np.full(1, -3, np.float32), np.full(1, 3, np.float32)
num_envs, max_episode_steps = 8, 1000
