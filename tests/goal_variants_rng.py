"""A replay RandomState for the goal modifiers (rg_goal_modify; test infrastructure): the placement replay of
tests/placement_rng.py plus the draws the reference's stacking, pick-and-place and training goals make after their placement,
on the modifiers' own purpose counter (robogym_b200/csrc/rg_place.inl documents the counters).

`GoalVariantsReplayRandomState(seed, env, epoch)` places as `ReplayRandomState` does.  Its d-th modifier draw reads counter
(d, 0, 3, epoch), d counting `random()`, scalar `uniform(low, high)`, `randint`, every step of `modifier_shuffle` and every
step of `choice` in call order; `random()` and `uniform` use words (x, y), the integers word x."""
import numpy as np

from placement_rng import ReplayRandomState, bounded, u53

MODIFY = 3


class GoalVariantsReplayRandomState(ReplayRandomState):
    def __init__(self, seed, env, epoch):
        super().__init__(seed, env, epoch)
        self.modifier_draws = 0

    def _modifier_word(self):
        d = self.modifier_draws
        self.modifier_draws += 1
        return self._draw((d, 0, MODIFY, self.epoch))

    def random(self):
        """numpy's random(): the next modifier draw's 53-bit double"""
        r = self._modifier_word()
        return u53(r[0], r[1])

    def uniform(self, low, high):
        """a modifier's scalar uniform(low, high) (a height); two values are a placement proposal, as ReplayRandomState's"""
        if np.ndim(low) == 0 and np.ndim(high) == 0:
            return float(low) + (float(high) - float(low)) * self.random()
        return super().uniform(low, high)

    def randint(self, low, high=None):
        """randint(high) / randint(low, high): low + a bounded integer in [0, high - low - 1] from the next modifier draw"""
        if high is None:
            low, high = 0, low
        assert high > low
        return int(low) + bounded(self._modifier_word()[0], int(high) - int(low) - 1)

    def modifier_shuffle(self, x):
        """numpy's shuffle (Fisher-Yates from the end) of a list or array, each step one modifier draw"""
        n = len(x)
        for s in range(n - 1):
            i = n - 1 - s
            j = bounded(self._modifier_word()[0], i)
            x[i], x[j] = x[j], x[i]

    def choice(self, a, size, replace=False):
        """`size` distinct elements of `a` in draw order, by a partial Fisher-Yates draw (step s swaps element s with one of
        s..n-1), each step one modifier draw"""
        assert not replace
        a = list(a)
        n = len(a)
        for s in range(size):
            j = s + bounded(self._modifier_word()[0], n - 1 - s)
            a[s], a[j] = a[j], a[s]
        return np.array(a[:size])
