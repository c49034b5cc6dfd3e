"""A replay RandomState for the object groups (rg_object_groups; test infrastructure): the draws the reference's
`_randomize_object_groups` and `_sample_default_quaternions` make, on the groups' own purpose counter
(robogym_b200/csrc/rg_groups.inl documents the counters and the draw order).

`GroupsReplayRandomState(seed, env, epoch)`'s d-th draw reads counter (d, 0, 6, epoch), d counting every value of `uniform`
and `random`, every value `randint` draws and every step of `permutation` / `shuffle`, in call order; after `yaws()` the
j-th value reads counter (j, 1, 6, epoch) instead.  Doubles use words (x, y), integers word x.  `choice` is the legacy
RandomState's own composition of those calls: with `p`, cumsum / divide / `random_sample` / searchsorted(side="right");
without, `randint` (with replacement) or `permutation(pop)[:size]` (without).  `randint` over a one-value range returns it
without a draw, as numpy's bounded-integer fill does."""
import numpy as np

from placement_rng import bounded, philox, u53

GROUPS = 6


class GroupsReplayRandomState:
    def __init__(self, seed, env, epoch):
        self.seed, self.env, self.epoch = int(seed), int(env), int(epoch)
        self.row = 0
        self.draws = [0, 0]

    def yaws(self):
        """the following draws are the initial yaws': counter (j, 1, 6, epoch)"""
        self.row = 1

    def _word(self):
        d = self.draws[self.row]
        self.draws[self.row] += 1
        return philox(np.array((d, self.row, GROUPS, self.epoch), dtype=np.uint64), self.seed, self.env)

    def _doubles(self, size):
        n = 1 if size is None else int(np.prod(size))
        u = np.array([u53(*self._word()[:2]) for _ in range(n)])
        return float(u[0]) if size is None else u.reshape(size)

    def random(self, size=None):
        return self._doubles(size)

    random_sample = random

    def uniform(self, low=0.0, high=1.0, size=None):
        """low + (high - low) * u, numpy's arithmetic for scalar bounds"""
        low, high = float(low), float(high)
        return low + (high - low) * self._doubles(size)

    def randint(self, low, high=None, size=None):
        if high is None:
            low, high = 0, low
        span = int(high) - int(low) - 1
        assert span >= 0
        n = 1 if size is None else int(np.prod(size))
        v = np.array([int(low) + (bounded(self._word()[0], span) if span > 0 else 0) for _ in range(n)], dtype=np.int64)
        return int(v[0]) if size is None else v.reshape(size)

    def shuffle(self, x):
        """numpy's shuffle of a sequence's first axis: Fisher-Yates from the end, one draw per step"""
        n = len(x)
        for s in range(n - 1):
            i = n - 1 - s
            j = bounded(self._word()[0], i)
            if isinstance(x, np.ndarray):
                x[[i, j]] = x[[j, i]]
            else:
                x[i], x[j] = x[j], x[i]

    def permutation(self, x):
        arr = np.arange(x) if isinstance(x, (int, np.integer)) else np.array(x)
        idx = np.arange(len(arr))
        self.shuffle(idx)
        return arr[idx]

    def choice(self, a, size=None, replace=True, p=None):
        arr = np.asarray(a) if not isinstance(a, (int, np.integer)) else None
        pop = int(a) if arr is None else len(arr)
        if replace:
            if p is not None:
                cdf = np.asarray(p, dtype=np.float64).cumsum()
                cdf /= cdf[-1]
                idx = cdf.searchsorted(self.random_sample(size), side="right")
            else:
                idx = self.randint(0, pop, size=size)
        else:
            assert p is None
            if (1 if size is None else int(np.prod(size))) > pop:
                raise ValueError("Cannot take a larger sample than population when 'replace=False'")
            idx = self.permutation(pop)[:(1 if size is None else size)]
            if size is None:
                idx = idx[0]
        return idx if arr is None else arr[idx]
