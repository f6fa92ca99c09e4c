"""CPU tier of the Mash distance's numeric limits (test_gpu_mash_dist_limits.py): the exact binomial tail and its
r-sensitivity that the GPU p-values are held to, the device's Stirling table against mpmath, and the two
constructions the GPU tier builds its pairs with: prefix rows that set (common, denom) and query lengths that set r,
and the NumPy merge it checks rows of 2^21 values against."""
import math
import os
import re
from fractions import Fraction

import mpmath
import numpy as np
import pytest

import mash_dist_oracle as O
from test_mash_dist_host import exact_tail

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def as_mpf(f: Fraction):
    with mpmath.workdps(80):
        return mpmath.mpf(f.numerator) / f.denominator


@pytest.mark.parametrize("r", [O.pair_r(21, 5 * 10 ** 6, 5 * 10 ** 6), O.pair_r(8, 10 ** 4, 10 ** 5), 0.5, 0.37, 0.9921875, 1e-3, 1 - 1e-7])
def test_exact_tail_against_fractions(r):
    for n in (1, 2, 3, 17, 60, 121, 200):
        for c in sorted(c for c in {0, 1, 2, n // 4, n // 2, int(n * r), int(n * r) + 1, n - 1, n} if 0 <= c <= n):
            want = as_mpf(exact_tail(c, n, r)) if c else mpmath.mpf(1)
            got = O.p_value_exact(c, n, r)
            if want == 0:
                assert got == 0
            else:
                assert abs(got - want) <= mpmath.mpf(10) ** -44 * want, (n, c, r, got, want)
    assert O.p_value_exact(5, 4, 0.5) == 0 and O.p_value_exact(0, 4, 0.5) == 1


@pytest.mark.parametrize("c,n,r", [(1, 1, 0.3), (3, 10, 0.2), (500, 1000, 0.5), (520, 1000, 0.5), (1, 10 ** 5, 1e-6), (99_990, 10 ** 5, 1 - 1e-4),
                                   (40, 3418, 0.01), (3418, 3418, 0.999)])
def test_kappa_is_the_log_derivative(c, n, r):
    with mpmath.workdps(60):
        R, h = mpmath.mpf(r), mpmath.mpf(10) ** -15
        fd = (mpmath.log(O.p_value_exact(c, n, R * (1 + h))) - mpmath.log(O.p_value_exact(c, n, R * (1 - h)))) / (2 * h)
    got = O.p_value_kappa(c, n, r)
    assert got > 0 and abs(got - float(fd)) <= 1e-12 * abs(float(fd)), (got, float(fd))
    assert O.p_value_kappa(0, n, r) == 0.0


def test_device_stirling_table_is_mpmath():
    src = open(os.path.join(ROOT, "poly_b200", "csrc", "mash_dist.cu")).read()
    body = re.search(r"STIRLERR_SMALL\[15\] = \{([^}]*)\}", src).group(1)
    vals = [float(v) for v in body.replace("\n", " ").split(",") if v.strip()]
    assert len(vals) == 15
    with mpmath.workdps(40):
        for n, v in enumerate(vals, 1):
            want = mpmath.loggamma(n + 1) - (n + mpmath.mpf(1) / 2) * mpmath.log(n) + n - mpmath.log(2 * mpmath.pi) / 2
            assert v == float(want), (n, v, float(want))


@pytest.mark.parametrize("n", [1, 2, 31, 33, 1000, 3419])
def test_prefix_rows_set_common_and_denom(n):
    master = O.master_list(np.random.default_rng(n), n)
    assert len(master) == n and master.dtype == np.uint32 and (np.diff(master.astype(np.int64)) > 0).all()
    if n > 1:
        assert master[0] == 0 and master[-1] == O.U32 - 1
    B = master.tolist()
    for c in sorted({0, 1, n // 2, n - 1, n}):
        assert O.compare(B[:c], B, n) == (c, n) and O.compare(B, B[:c], n) == (c, n)
        assert O.merge_counts(master[:c], master, n) == (c, n)


@pytest.mark.parametrize("k,r_length", [(30, O.U64MAX), (16, O.U64MAX), (21, 10 ** 6)])
def test_lengths_set_r(k, r_length):
    top = O.pair_r(k, O.U64MAX, r_length)
    for target in (1e-9, 3.3e-7, 1e-3, 0.25, 0.5, 0.75, 1 - 1e-6, 1 - 1e-9):
        if not O.pair_r(k, 1, r_length) < target <= top:
            continue
        lq = O.length_for_r(k, r_length, target)
        assert O.pair_r(k, lq - 1, r_length) < target <= O.pair_r(k, lq, r_length)
        # one length step moves r by a relative 1 / lq at most, and below an ulp once lq is large
        assert O.pair_r(k, lq, r_length) - target <= max(target / lq, math.ulp(target)) * 1.01
    # the ranges the GPU grid draws on: k = 30 reaches 1e-9 .. 0.5, k = 16 reaches 0.5 .. 1 - 1e-9
    if r_length == O.U64MAX:
        assert O.pair_r(k, 1, r_length) < (1e-9 if k == 30 else 0.5) and top > (0.5 if k == 30 else 1 - 1e-9)


def test_numpy_merge_is_compare():
    rng = np.random.default_rng(41)
    for trial in range(300):
        s = int(rng.integers(1, 40))
        pool = np.unique(rng.integers(0, O.U32, size=int(rng.integers(1, 90)), dtype=np.uint64)).astype(np.uint32)
        if trial % 5 == 0:
            pool = np.union1d(pool, np.array([0, O.U32 - 1], np.uint32))
        a = np.sort(rng.choice(pool, size=int(rng.integers(0, min(s, len(pool)) + 1)), replace=False))
        b = np.sort(rng.choice(pool, size=int(rng.integers(0, min(s, len(pool)) + 1)), replace=False))
        if trial % 7 == 0:
            b = a[: int(rng.integers(0, len(a) + 1))]
        assert O.merge_counts(a, b, s) == O.compare(a.tolist(), b.tolist(), s), (a, b, s)
        assert O.merge_counts(b, a, s) == O.compare(b.tolist(), a.tolist(), s)
