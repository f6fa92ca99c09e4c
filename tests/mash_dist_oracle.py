"""Plain restatement of the Mash distance between grouped sketches (pg_mash_dist), for checking its device path.  TEST
INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and tools/bench_mash_dist.py.

common and denom come from Mash's compareSketches loop, literally, in plain Python; the distance from math.log with
the same branches; the p-value from scipy.stats.binom.sf.  Nothing here follows the device design: no merge path, no
warp, no incomplete beta function."""
from __future__ import annotations

import math

import numpy as np


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
