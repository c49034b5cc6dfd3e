"""Philox4x32-10 in numpy and a replay RandomState that draws the same numbers as the placement kernel (test infrastructure;
robogym_b200/csrc/rg_place.inl documents the counters).

`ReplayRandomState(seed, env, epoch)` has the two methods the reference's placement functions call: `shuffle` (Fisher-Yates
from the end, as numpy's; step s of the t-th shuffle draws j in [0, i] from counter (s, t, 0, epoch)) and `uniform(low, high)`
for two values (the p-th call reads counter (p, 0, 1, epoch): low + (high - low) * u, u numpy's 53-bit double)."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
SHUFFLE, PROPOSAL = 0, 1
_MASK = np.uint64(0xFFFFFFFF)


def philox(ctr, k0, k1):
    """Philox4x32-10 of counters ctr [..., 4] (uint32) under the key (k0, k1) -> [..., 4] uint32"""
    c = np.asarray(ctr, dtype=np.uint64) & _MASK
    c0, c1, c2, c3 = c[..., 0], c[..., 1], c[..., 2], c[..., 3]
    k0, k1 = np.uint64(k0 & 0xFFFFFFFF), np.uint64(k1 & 0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = np.uint64(M0) * c0, np.uint64(M1) * c2
        c0, c1, c2, c3 = (p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & _MASK, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & _MASK
        k0, k1 = (k0 + np.uint64(W0)) & _MASK, (k1 + np.uint64(W1)) & _MASK
    return np.stack([c0, c1, c2, c3], axis=-1).astype(np.uint32)


def u53(a, b):
    """numpy's random_sample from two 32-bit words"""
    return (float(int(a) >> 5) * 67108864.0 + float(int(b) >> 6)) / 9007199254740992.0


def bounded(u, i):
    """an integer in [0, i] from one 32-bit word"""
    return (int(u) * (i + 1)) >> 32


class ReplayRandomState:
    def __init__(self, seed, env, epoch):
        self.seed, self.env, self.epoch = int(seed), int(env), int(epoch)
        self.shuffles = 0
        self.proposals = 0

    def _draw(self, c):
        return philox(np.array(c, dtype=np.uint64), self.seed, self.env)

    def shuffle(self, x):
        t = self.shuffles
        self.shuffles += 1
        n = len(x)
        if n < 2:
            return
        steps = np.array([(s, t, SHUFFLE, self.epoch) for s in range(n - 1)], dtype=np.uint64)
        words = self._draw(steps)[:, 0]
        for s in range(n - 1):
            i = n - 1 - s
            j = bounded(words[s], i)
            x[[i, j]] = x[[j, i]]

    def uniform(self, low, high):
        p = self.proposals
        self.proposals += 1
        r = self._draw((p, 0, PROPOSAL, self.epoch))
        u = np.array([u53(r[0], r[1]), u53(r[2], r[3])])
        low, high = np.asarray(low, dtype=np.float64), np.asarray(high, dtype=np.float64)
        assert low.shape == (2,) and high.shape == (2,)
        return low + (high - low) * u
