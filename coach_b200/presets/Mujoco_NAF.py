"""rl_coach/presets/Mujoco_NAF.py:22-26: NAF with a [Dense(200)] embedder, a [Dense(200)] middleware and gradients
clipped by value at 1000."""
from coach_b200.agents.naf_agent import NAFAgentParameters

agent_params = NAFAgentParameters()
agent_params.network_wrappers['main'].embedder_units = (200,)
agent_params.network_wrappers['main'].middleware_parameters.scheme = [200]
agent_params.network_wrappers['main'].clip_gradients = 1000
agent_params.network_wrappers['main'].gradients_clipping_method = "ClipByValue"

observation_dim, action_dim = 11, 3          # Hopper
