"""Schedules used on the hot path (PER beta, exploration epsilon), mirroring ``rl_coach/schedules.py:23-91``.

``LinearSchedule.step`` keeps the reference's *recurrence* (repeated subtraction + ``np.clip``) rather than a closed
form: the accumulated floating-point error is observable in the importance weights, so it is part of the contract
(SURVEY.md quirk Q5).
"""
import numpy as np


class Schedule(object):
    def __init__(self, initial_value: float):
        self.initial_value = initial_value
        self.current_value = initial_value

    def step(self):
        raise NotImplementedError("")


class ConstantSchedule(Schedule):
    def step(self):
        pass


class LinearSchedule(Schedule):
    def __init__(self, initial_value: float, final_value: float, decay_steps: int):
        super().__init__(initial_value)
        self.final_value = final_value
        self.decay_steps = decay_steps
        self.decay_delta = (initial_value - final_value) / float(decay_steps)

    def step(self):
        self.current_value -= self.decay_delta
        if self.final_value < self.initial_value:
            self.current_value = np.clip(self.current_value, self.final_value, self.initial_value)
        if self.final_value > self.initial_value:
            self.current_value = np.clip(self.current_value, self.initial_value, self.final_value)


class PieceWiseSchedule(Schedule):
    """rl_coach/schedules.py:66-91: sub-schedules applied one after the other, each for its number of steps (the UCB
    exploration's epsilon).  schedules: [(Schedule, EnvironmentSteps), ...]"""

    def __init__(self, schedules):
        super().__init__(schedules[0][0].initial_value)
        self.schedules = schedules
        self.current_schedule = schedules[0]
        self.current_schedule_idx = 0
        self.current_schedule_step_count = 0

    def step(self):
        self.current_schedule[0].step()
        if self.current_schedule_idx < len(self.schedules) - 1 \
                and self.current_schedule_step_count >= self.current_schedule[1].num_steps:
            self.current_schedule_idx += 1
            self.current_schedule = self.schedules[self.current_schedule_idx]
            self.current_schedule_step_count = 0
        self.current_value = self.current_schedule[0].current_value
        self.current_schedule_step_count += 1
