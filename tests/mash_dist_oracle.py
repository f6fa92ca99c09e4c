"""Plain restatement of the Mash distance between grouped sketches (pg_mash_dist), for checking its device path.  TEST
INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and tools/bench_mash_dist.py.

common and denom come from Mash's compareSketches loop, literally, in plain Python (merge_counts restates them with
NumPy set operations, for rows of millions of values); the distance from math.log with the same branches; the p-value
from scipy.stats.binom.sf, and exactly, to 50 digits, from p_value_exact.  Nothing here follows the device design: no
merge path, no warp, no incomplete beta function."""
from __future__ import annotations

import math

import mpmath
import numpy as np

U32 = 1 << 32
U64MAX = (1 << 64) - 1


def compare(A, B, s: int):
    """(common, denom) of two strictly ascending value lists, by Mash's loop."""
    a, b = len(A), len(B)
    i = j = common = denom = 0
    while denom < s and i < a and j < b:
        if A[i] < B[j]:
            i += 1
        elif B[j] < A[i]:
            j += 1
        else:
            i += 1
            j += 1
            common += 1
        denom += 1
    if denom < s:
        denom += min(a - i, s - denom)
        denom += min(b - j, s - denom)
    return common, denom


def distance(common: int, denom: int, k: int) -> float:
    if common == denom:
        return 0.0
    if common == 0:
        return 1.0
    j = common / denom
    return min(-math.log(2.0 * j / (1.0 + j)) / k, 1.0)


def pair_r(k: int, len_q: int, len_r: int) -> float:
    """Mash's r: the chance that a k-mer of one random genome is in the sketch space of the other, as the header states it."""
    four_k = math.ldexp(1.0, 2 * k) if 2 * k < 1024 else math.inf
    pq, pr = 1.0 / (1.0 + four_k / float(len_q)), 1.0 / (1.0 + four_k / float(len_r))
    den = pq + pr - pq * pr
    return pq * pr / den if den > 0.0 else 0.0


def p_value(common: int, denom: int, k: int, len_q: int, len_r: int) -> float:
    from scipy.stats import binom

    if common == 0:
        return 1.0
    r = pair_r(k, len_q, len_r)
    if r == 0.0:
        return 0.0
    return float(binom.sf(common - 1, denom, r))


def _dbinom_exact(x: int, n: int, R):
    """P[Binomial(n, R) = x] as an mpf, from log-gamma at the working precision."""
    return mpmath.exp(mpmath.loggamma(n + 1) - mpmath.loggamma(x + 1) - mpmath.loggamma(n - x + 1) + x * mpmath.log(R) + (n - x) * mpmath.log1p(-R))


def p_value_exact(common: int, denom: int, r) -> mpmath.mpf:
    """P[Binomial(denom, r) >= common] to 50 digits, r a double (or an mpf) in [0, 1].  The binomial terms are summed
    from the shorter side of the mode: upward from common for an upper tail, else 1 - the downward sum from
    common - 1; one term from log-gamma, the rest by the term ratio, until a term falls below 1e-45 of the sum."""
    n, c = int(denom), int(common)
    if c <= 0 or r >= 1:
        return mpmath.mpf(1)
    if c > n or r <= 0:
        return mpmath.mpf(0)
    with mpmath.workdps(60):  # log-gamma of n ~ 2^24 spends 9 of the digits
        R = mpmath.mpf(r)
        rq = R / (1 - R)
        cut = mpmath.mpf(10) ** -45
        if c >= (n + 1) * R:
            t = _dbinom_exact(c, n, R)
            s, i = t, c
            while i < n:
                t = t * (n - i) / (i + 1) * rq
                s += t
                i += 1
                if t < s * cut:
                    break
            return +s
        t = _dbinom_exact(c - 1, n, R)
        s, i = t, c - 1
        while i > 0:
            t = t * i / ((n - i + 1) * rq)
            s += t
            i -= 1
            if t < s * cut:
                break
        return 1 - s


def p_value_kappa(common: int, denom: int, r, p=None) -> float:
    """|d ln p / d ln r| of the exact tail, = common * dbinom(common; denom, r) / p: what a difference of one ulp in r
    can do to the p-value, relative.  p, when given, is p_value_exact(common, denom, r)."""
    if common <= 0 or common > denom or not 0 < r < 1:
        return 0.0
    with mpmath.workdps(60):
        p = p_value_exact(common, denom, r) if p is None else p
        return float(common * _dbinom_exact(int(common), int(denom), mpmath.mpf(r)) / p)


def master_list(rng, n: int) -> np.ndarray:
    """n strictly ascending random uint32 values, 0 and 2^32 - 1 among them (0 alone when n == 1)."""
    if n == 1:
        return np.zeros(1, np.uint32)
    vals = np.zeros(0, np.uint32)
    while len(vals) < n - 2:
        vals = np.sort(np.concatenate([vals, rng.integers(1, U32 - 1, size=n - 2 - len(vals) + n // 64 + 16, dtype=np.uint32)]))
        vals = vals[np.concatenate([[True], vals[1:] != vals[:-1]])]
    vals = np.delete(vals, rng.choice(len(vals), size=len(vals) - (n - 2), replace=False))
    return np.concatenate([[0], vals, [U32 - 1]]).astype(np.uint32)


def length_for_r(k: int, r_length: int, r: float) -> int:
    """The smallest query length lq in [1, 2^64 - 1] with pair_r(k, lq, r_length) >= r (2^64 - 1 when none): pair_r is
    non-decreasing in lq, so lq - 1 and lq sit one length step either side of r."""
    lo, hi = 1, U64MAX
    while lo < hi:
        mid = (lo + hi) // 2
        if pair_r(k, mid, r_length) >= r:
            hi = mid
        else:
            lo = mid + 1
    return lo


def merge_counts(A, B, s: int):
    """(common, denom) of two strictly ascending uint32 arrays by set operations: the denom = min(s, |A u B|) smallest
    union values, and how many of them both rows hold.  The same definition as compare, for rows of millions."""
    both = np.sort(np.concatenate([np.asarray(A, np.uint32), np.asarray(B, np.uint32)]))
    if len(both) == 0 or s < 1:
        return 0, 0
    twice = both[1:] == both[:-1]  # a value of both rows appears twice in a row
    union, shared = both[np.concatenate([[True], ~twice])], both[1:][twice]
    denom = min(s, len(union))
    return int(np.searchsorted(shared, union[denom - 1], side="right")), denom


def dist(q_rows, q_count, r_rows, r_count, k: int, q_length=None, r_length=None):
    """(common, denom, distance, p_value or None), each [nq, nr], as pg_mash_dist defines them."""
    s = int(np.asarray(q_rows).shape[1])
    Q = [[int(v) for v in q_rows[i][: int(q_count[i])]] for i in range(len(q_count))]
    R = [[int(v) for v in r_rows[i][: int(r_count[i])]] for i in range(len(r_count))]
    nq, nr = len(Q), len(R)
    common, denom = np.zeros((nq, nr), np.uint32), np.zeros((nq, nr), np.uint32)
    dst = np.zeros((nq, nr), np.float64)
    p = np.zeros((nq, nr), np.float64) if q_length is not None else None
    for x in range(nq):
        for y in range(nr):
            c, d = compare(Q[x], R[y], s)
            common[x, y], denom[x, y], dst[x, y] = c, d, distance(c, d, k)
            if p is not None:
                p[x, y] = p_value(c, d, k, int(q_length[x]), int(r_length[y]))
    return common, denom, dst, p
