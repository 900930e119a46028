"""The reference's Adam hyper-parameters and their per-step schedule (core/NtsScheduler.hpp:639-736), shared by the
dense `toolkits.Parameter` and the row-sparse `feature_table.ShardedEmbedding`: both update with the current alpha,
beta1 and beta2 and then call next()."""
from __future__ import annotations

import numpy as np


class AdamSchedule:
    """Attributes alpha, beta1, beta2 (the current values the update uses), epsilon, weight_decay, the initial values
    alpha_t, beta1_t, beta2_t, curr_epoch (steps taken) and decay_rate, decay_epoch."""

    def _init_schedule(self, alpha, beta1, beta2, epsilon, weight_decay):
        # the reference keeps every hyper-parameter in `ValueType` = float and does the schedule arithmetic in float
        # (1 - 0.999f != 0.001: a 1.3e-5 relative difference in V that the golden vectors of tests/test_adam.py see)
        f32 = np.float32
        self.alpha = f32(alpha)
        self.beta1, self.beta2, self.epsilon = f32(beta1), f32(beta2), f32(epsilon)
        self.alpha_t, self.beta1_t, self.beta2_t = f32(alpha), f32(beta1), f32(beta2)
        self.weight_decay = f32(weight_decay)
        self.curr_epoch = 0
        self.decay_rate, self.decay_epoch = 1, -1

    def set_decay(self, decay_rate, decay_epoch):
        # the reference stores both in `int` members (NtsScheduler.hpp:663-664): 0.97 truncates to 0
        self.decay_rate, self.decay_epoch = int(decay_rate), int(decay_epoch)

    def next(self):
        """NtsScheduler.hpp:727-736: the bias correction folded into alpha, and the learning-rate decay."""
        if self.decay_epoch != -1 and self.curr_epoch != 0 and self.curr_epoch % self.decay_epoch == 0:
            self.alpha_t *= self.decay_rate
        one = np.float32(1)
        self.alpha_t = np.float32(self.alpha_t)
        self.alpha = np.float32(self.alpha_t * np.sqrt(one - self.beta2) / (one - self.beta1))
        self.beta1 = np.float32(self.beta1 * self.beta1_t)
        self.beta2 = np.float32(self.beta2 * self.beta2_t)
        self.curr_epoch += 1
