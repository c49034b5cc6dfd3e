"""A replay RandomState for the layout goals (rg_layout_goals; test infrastructure): the draws the reference's domino and
attached-block goal generators make, on the layout goals' own purpose counter (robogym_b200/csrc/rg_place.inl documents the
counters).

`LayoutReplayRandomState(seed, env, epoch)`'s d-th draw reads counter (d, 0, 4, epoch), d counting `random()`, each value of
`uniform(low, high)` and every step of `permutation` in call order; `random()` and `uniform` use words (x, y), permutation
steps word x.  So the k-th random() of DominoStateGoal is draw k, and AttachedBlockStateGoal's permutation takes draws 0-6
and its origin draws 7 and 8."""
import numpy as np

from goal_variants_rng import GoalVariantsReplayRandomState

LAYOUT = 4


class LayoutReplayRandomState(GoalVariantsReplayRandomState):
    def _modifier_word(self):
        d = self.modifier_draws
        self.modifier_draws += 1
        return self._draw((d, 0, LAYOUT, self.epoch))

    def uniform(self, low, high):
        """uniform(low, high) of scalars or arrays: low + (high - low) * u, one draw per value"""
        low, high = np.asarray(low, dtype=np.float64), np.asarray(high, dtype=np.float64)
        u = np.array([self.random() for _ in range(np.broadcast(low, high).size)]).reshape(np.broadcast(low, high).shape)
        out = low + (high - low) * u
        return float(out) if out.ndim == 0 else out

    def permutation(self, x):
        """numpy's permutation of an array's rows: a shuffle (Fisher-Yates from the end) of their indices, one draw per step"""
        arr = np.array(x)
        idx = np.arange(len(arr))
        self.modifier_shuffle(idx)
        return arr[idx]
