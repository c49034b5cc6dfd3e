"""A replay RandomState that draws the same numbers as the goal-orientation kernel (test infrastructure;
robogym_b200/csrc/rg_goal.inl documents the counters).  It reuses the Philox4x32-10, 53-bit uniform and bounded-integer
constructions of tests/placement_rng.py, on the goal orientations' own purpose counter."""
import numpy as np

from placement_rng import bounded, philox, u53

GOAL_ROT = 2


class GoalRotReplayRandomState:
    """The draws of one goal-orientation sample (rg_goal_orientations): `uniform(low, high, size=n)` gives object i
    low + (high - low) * u from words (x, y) of counter (i, 0, 2, epoch), `randint(low, high, size=n)` gives low + a bounded
    integer in [0, high - low - 1] from word z of the same counter."""

    def __init__(self, seed, env, epoch):
        self.seed, self.env, self.epoch = int(seed), int(env), int(epoch)

    def _words(self, n):
        return philox(np.array([(i, 0, GOAL_ROT, self.epoch) for i in range(n)], dtype=np.uint64).reshape(-1, 4), self.seed, self.env)

    def uniform(self, low=0.0, high=1.0, size=None):
        w = self._words(int(size))
        u = np.array([u53(r[0], r[1]) for r in w])
        return low + (high - low) * u

    def randint(self, low, high=None, size=None):
        if high is None:
            low, high = 0, low
        w = self._words(int(size))
        return np.array([low + bounded(r[2], high - low - 1) for r in w], dtype=np.int64)
