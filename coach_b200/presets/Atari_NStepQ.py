"""rl_coach/presets/Atari_NStepQ.py:19-23 (agent parameters)"""
from coach_b200.agents.n_step_q_agent import NStepQAgentParameters
from coach_b200.base_parameters import Conv2d, Dense

agent_params = NStepQAgentParameters()
agent_params.network_wrappers['main'].learning_rate = 0.0001
agent_params.network_wrappers['main'].input_embedders_parameters['observation'].scheme = [Conv2d(16, 8, 4),
                                                                                          Conv2d(32, 4, 2)]
agent_params.network_wrappers['main'].middleware_parameters.scheme = [Dense(256)]

observation_shape, num_actions = (84, 84, 4), 6
