"""rl_coach/presets/Doom_Health_MMC.py:22-31 (Mixed Monte Carlo on ViZDoom's health gathering: an episodic replay of
200 episodes, MSE loss).

Geometry: the observation is the 60x76 luma frame stacked 3 times (environments/doom_environment.py:93-99), uint8
(60, 76, 3).  The 4 actions are no-op plus the three buttons of ViZDoom's stock ``health_gathering.cfg`` (turn left,
turn right, move forward) under MultiSelectActionSpace(max_simultaneous_selected_actions=1,
allow_no_action_to_be_selected=True).  That cfg ships with ViZDoom, not with the reference tree, so the button count
comes from ViZDoom's distribution.

The ring of an episode-sized replay is sized in transitions (``transition_capacity``): 2^17 transitions hold 200
episodes of 655 steps on average.
"""
from coach_b200.agents.mmc_agent import MixedMonteCarloAgentParameters
from coach_b200.base_parameters import EnvironmentSteps
from coach_b200.memories.memory import MemoryGranularity

agent_params = MixedMonteCarloAgentParameters()
agent_params.network_wrappers['main'].learning_rate = 0.00025
agent_params.memory.max_size = (MemoryGranularity.Episodes, 200)
agent_params.memory.transition_capacity = 1 << 17
agent_params.algorithm.num_steps_between_copying_online_weights_to_target = EnvironmentSteps(1000)
agent_params.algorithm.num_consecutive_playing_steps = EnvironmentSteps(1)
agent_params.network_wrappers['main'].replace_mse_with_huber_loss = False

observation_shape, num_actions = (60, 76, 3), 4
