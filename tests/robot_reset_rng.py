"""The robot reset's random action in numpy (test infrastructure; robogym_b200/csrc/rg_arm.inl documents the counter):
component d of environment `env` is numpy's 53-bit double from Philox4x32-10 keyed by (seed, env) at counter (d, 0, 5, epoch),
mapped as gym 0.15.3's Box.sample maps a bounded float32 box: low + (high - low) * u in float64, cast to float32."""
import numpy as np

from placement_rng import philox, u53

ARM = 5          # purpose counter after the layout goals' 4


def initial_action(seed, env, epoch, dim, low=-1.0, high=1.0):
    r = philox(np.array([(d, 0, ARM, epoch) for d in range(dim)], dtype=np.uint64), seed, env)
    u = np.array([u53(a, b) for a, b in r[:, :2]])
    return (np.float64(low) + (np.float64(high) - np.float64(low)) * u).astype(np.float32)


class ReplayActionSpace:
    """stands in for the reference environment's action_space: sample() returns the replay draw of one environment"""

    def __init__(self, space, seed, env, epoch):
        self.space, self.seed, self.env, self.epoch = space, int(seed), int(env), int(epoch)

    def sample(self):
        assert np.all(self.space.low == -1.0) and np.all(self.space.high == 1.0) and self.space.dtype == np.float32
        return initial_action(self.seed, self.env, self.epoch, self.space.shape[0])

    def __getattr__(self, name):
        return getattr(self.space, name)
