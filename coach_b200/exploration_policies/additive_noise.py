"""The Gaussian exploration parameters of the continuous policy agents:

  rl_coach/exploration_policies/additive_noise.py:29-39   AdditiveNoiseParameters (Policy Gradients: a fixed std)
  rl_coach/exploration_policies/continuous_entropy.py     ContinuousEntropyParameters (A3C: the std is a network output
                                                          and the entropy term lives in the head's loss)

Acting itself runs on the device (cb200_policy_act, cb200_gaussian_policy_act).
"""
from coach_b200.schedules import LinearSchedule


class AdditiveNoiseParameters(object):
    """exploration_policies/additive_noise.py:29-39"""

    def __init__(self):
        self.noise_schedule = LinearSchedule(0.1, 0.1, 50000)
        self.evaluation_noise = 0.05
        self.noise_as_percentage_from_action_space = True

    @property
    def path(self):
        return 'rl_coach.exploration_policies.additive_noise:AdditiveNoise'


class ContinuousEntropyParameters(AdditiveNoiseParameters):
    """exploration_policies/continuous_entropy.py: AdditiveNoise whose std is the second output of the policy head"""

    @property
    def path(self):
        return 'rl_coach.exploration_policies.continuous_entropy:ContinuousEntropy'
