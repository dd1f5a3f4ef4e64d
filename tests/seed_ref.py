"""Brute-force reference of the seed stage of the candidate filter (DESIGN.md section 5; eb_common.h: SeedIndexParams,
SeedPlanParams, seed_threshold; eb_core.h: seed_windows), in numpy and plain Python.

Index: every target position i has the key of its Lidx codes, codes past the end counting as 0; bucketStart holds the
counts per key, then their exclusive prefix sums.  Plan of a read with threshold t: seed j is read[a, a+Ls) with
a = j * (m // (t+1)); its occurrences are found by comparing it with the target at every position (not through a
radix table), and each gives the candidate end column E = p + (m - a) - 1.  A seed whose index range (positions whose
padded key starts like the seed) is longer than maxBucket saturates the read, as do more than CAP candidates; else
the sorted candidates are grouped into windows."""
import numpy as np

SEED_NONE, SEED_WINDOWS, SEED_SATURATED = 0, 1, 2
K1_RANGE_GAP = 256


def padded_keys(tcodes, Lidx, sigma, numPos=None):
    """Key of the Lidx codes at each position 0..numPos-1 (codes past the end count as 0)."""
    n = len(tcodes)
    numPos = n if numPos is None else numPos
    padded = np.concatenate([np.asarray(tcodes, dtype=np.int64), np.zeros(Lidx, dtype=np.int64)])
    k = np.zeros(numPos, dtype=np.int64)
    for x in range(Lidx):
        k = k * sigma + padded[x:x + numPos]
    return k


def index(tcodes, Lidx, sigma, numPos=None):
    """(bucketStart [sigma^Lidx + 1], keys of the indexed positions)."""
    keys = padded_keys(tcodes, Lidx, sigma, numPos)
    counts = np.bincount(keys, minlength=sigma ** Lidx)
    bs = np.zeros(sigma ** Lidx + 1, dtype=np.int64)
    np.cumsum(counts, out=bs[1:])
    return bs, keys


def same_positions(bucketStart, positions, keys):
    """Does `positions` (laid out by bucketStart) hold, per bucket, exactly the positions whose key it is?"""
    bucket = np.repeat(np.arange(len(bucketStart) - 1), np.diff(np.asarray(bucketStart, dtype=np.int64)))
    got = np.asarray(positions, dtype=np.int64)[np.lexsort((positions, bucket))]
    return np.array_equal(got, np.argsort(keys, kind="stable"))


def seed_threshold(m, kBound, Ls, seedK):
    bound = m if (kBound < 0 or kBound > m) else kBound
    t = min(m // Ls - 1, seedK, bound)
    return t if (m >= 2 * Ls and t > -1) else -1


class Target:
    """Exact occurrences of words in one encoded target, by comparing the word with the target at every position."""

    def __init__(self, tcodes):
        self.codes = bytes(np.asarray(tcodes, dtype=np.uint8))
        self.n = len(self.codes)
        self._occ, self._prefix = {}, {}

    def occurrences(self, word):
        """Positions p with target[p, p + len(word)) == word (p + len(word) <= n)."""
        L = len(word)
        if L not in self._occ:
            d = {}
            for p in range(self.n - L + 1):
                d.setdefault(self.codes[p:p + L], []).append(p)
            self._occ[L] = d
        return self._occ[L].get(bytes(word), [])

    def range_length(self, word):
        """Positions i in [0, n) whose codes i, i+1, ... (zero past the end) start with `word`."""
        L = len(word)
        if L not in self._prefix:
            padded = self.codes + bytes(L)
            d = {}
            for i in range(self.n):
                w = padded[i:i + L]
                d[w] = d.get(w, 0) + 1
            self._prefix[L] = d
        return self._prefix[L].get(bytes(word), 0)


def windows(E, m, t, n, spread):
    """(ws, lo, hi) of the windows over sorted candidates E.  Candidates share a window while the banded sweep can
    cover them (last - first <= 63 - 4t); when no banded window fits t, while the gap to the previous one is at most
    K1_RANGE_GAP and the group spans at most `spread`.  Tracked columns [lo, hi] = [first - t, last + t] are kept
    disjoint from the previous window's and clipped to [0, n-1]; the sweep starts m + t columns early, at a
    multiple of 16."""
    band = 63 - 4 * t
    out, prev_hi, i = [], -1, 0
    while i < len(E):
        first = last = E[i]
        i += 1
        while i < len(E) and ((E[i] - first <= band) if band >= 0 else
                              (E[i] - last <= K1_RANGE_GAP and E[i] - first <= spread)):
            last = E[i]
            i += 1
        lo = max(first - t, prev_hi + 1, 0)
        hi = min(last + t, n - 1)
        if lo > hi:
            continue
        prev_hi = hi
        out.append((max(0, lo - (m + t)) & ~15, lo, hi))
    return out


def candidates(target, q, t, Ls, Lidx, sigma, maxBucket):
    """(saturated by a long range, candidate end columns) of read q (codes) with threshold t."""
    m = len(q)
    stride = m // (t + 1)
    Lk = min(Ls, Lidx)
    long_range, E = False, []
    for j in range(t + 1):
        a = j * stride
        seed = bytes(q[a:a + Ls])
        if max(seed) >= sigma:
            continue
        if target.range_length(seed[:Lk]) > maxBucket:
            long_range = True
            continue
        E.extend(p + (m - a) - 1 for p in target.occurrences(seed))
    return long_range, E


def plan_read(target, q, t, Ls, Lidx, sigma, maxBucket, spread, cap):
    """(state, thr, [(t + 1, ws, len, tf), ...]) of one read."""
    if t < 0:
        return SEED_SATURATED, -1, []
    long_range, E = candidates(target, q, t, Ls, Lidx, sigma, maxBucket)
    if long_range or len(E) > cap:
        return SEED_SATURATED, t, []
    wins = [(t + 1, ws, hi - ws + 1, lo - ws) for ws, lo, hi in windows(sorted(E), len(q), t, target.n, spread)]
    return (SEED_WINDOWS if wins else SEED_NONE), t, wins
