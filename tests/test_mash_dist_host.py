"""CPU tier of the Mash distance between grouped sketches (pg_mash_dist, pg_mash_dist_within): every argument rule, in
its order, before any device work, for the host and _dev forms; the Python mirror's rules; and the oracle on
hand-worked cases, its p-value against an exact binomial tail."""
import ctypes as C
import math
from fractions import Fraction

import numpy as np
import pytest

from poly_b200 import _lib, mash

import mash_dist_oracle as O

ARG = _lib.PG_ERR_ARG
U32MAX = (1 << 32) - 1


def dense(dev, q, qc, nq, r, rc, nr, stride=4, s=4, k=21, ql=None, rl=None, p=False):
    L = _lib.lib()
    n = max(min(nq * nr, 64), 1)  # the rule tests never reach the outputs
    out = [np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(n, np.float64), np.zeros(n, np.float64) if p else None]
    args = (_lib.ptr(q), _lib.ptr(qc), nq, _lib.ptr(r), _lib.ptr(rc), nr, stride, s, k, _lib.ptr(ql), _lib.ptr(rl), *[_lib.ptr(o) for o in out])
    return L.pg_mash_dist_dev(*args, None) if dev else L.pg_mash_dist(*args)


def within(dev, q, qc, nq, r, rc, nr, stride=4, s=4, k=21, ql=None, rl=None, max_d=1.0, max_p=1.0, flags=0, pairs=True, n_pairs=True, p=False):
    L = _lib.lib()
    pq, pr = np.zeros(8, np.uint32), np.zeros(8, np.uint32)
    dist = np.zeros(8, np.float64)
    pv = np.zeros(8, np.float64) if p else None
    cnt, d_cnt = C.c_uint64(0), np.zeros(1, np.uint64)
    args = (_lib.ptr(q), _lib.ptr(qc), nq, _lib.ptr(r), _lib.ptr(rc), nr, stride, s, k, _lib.ptr(ql), _lib.ptr(rl), max_d, max_p, flags,
            pq.ctypes.data if pairs else None, pr.ctypes.data, None, None, dist.ctypes.data, _lib.ptr(pv), 8)
    if dev:
        return L.pg_mash_dist_within_dev(*args, d_cnt.ctypes.data if n_pairs else None, None)
    return L.pg_mash_dist_within(*args, C.byref(cnt) if n_pairs else None)


ROWS = np.array([[1, 5, 9, 0], [2, 5, 0, 0]], np.uint32)
CNT = np.array([3, 2], np.uint32)
LEN = np.array([1000, 2000], np.uint64)


@pytest.mark.parametrize("dev", [False, True])
@pytest.mark.parametrize("form", [dense, within])
def test_rules_in_order(dev, form):
    R, C_ = ROWS, CNT
    # every rule broken at once: the first one decides, then each is fixed in turn
    assert form(dev, None, None, 1 << 32, None, None, 2, stride=0, s=0, k=0, p=True) == ARG and "2^32" in _lib.last_error()
    assert form(dev, None, None, 2, None, None, 1 << 32, stride=0, s=0, k=0, p=True) == ARG and "2^32" in _lib.last_error()
    assert form(dev, None, None, 2, None, None, 2, stride=0, s=0, k=0, p=True) == ARG and "kmerSize" in _lib.last_error()
    assert form(dev, None, None, 2, None, None, 2, stride=0, s=0, p=True) == ARG and "sketchSize" in _lib.last_error()
    assert form(dev, None, None, 2, None, None, 2, stride=3, p=True) == ARG and "row_stride" in _lib.last_error()
    assert form(dev, None, C_, 2, R, C_, 2, p=True) == ARG and "null rows" in _lib.last_error()
    assert form(dev, R, None, 2, R, C_, 2, p=True) == ARG and "null rows" in _lib.last_error()
    assert form(dev, R, C_, 2, None, C_, 2, p=True) == ARG and "null rows" in _lib.last_error()
    assert form(dev, R, C_, 2, R, None, 2, p=True) == ARG and "null rows" in _lib.last_error()
    assert form(dev, R, C_, 2, R, C_, 2, p=True) == ARG and "lengths" in _lib.last_error()
    assert form(dev, R, C_, 2, R, C_, 2, ql=LEN, p=True) == ARG and "lengths" in _lib.last_error()
    assert form(dev, R, C_, 2, R, C_, 2, rl=LEN, p=True) == ARG and "lengths" in _lib.last_error()
    if form is within:
        # a p-value limit below 1 needs the lengths too, even without a p_value output
        assert form(dev, R, C_, 2, R, C_, 2, max_p=0.5) == ARG and "lengths" in _lib.last_error()
        kw = dict(ql=LEN, rl=LEN, p=True)
        assert form(dev, R, C_, 2, R, C_, 1, max_d=math.nan, flags=6, pairs=False, n_pairs=False, **kw) == ARG and "NaN" in _lib.last_error()
        assert form(dev, R, C_, 2, R, C_, 2, max_p=math.nan, **kw) == ARG and "NaN" in _lib.last_error()
        assert form(dev, R, C_, 2, R, C_, 1, flags=2, pairs=False, n_pairs=False, **kw) == ARG and "flag" in _lib.last_error()
        assert form(dev, R, C_, 2, R, C_, 1, flags=1, pairs=False, n_pairs=False, **kw) == ARG and "PG_PAIRS_UPPER" in _lib.last_error()
        assert form(dev, R, C_, 2, R, C_, 2, flags=1, pairs=False, **kw) == ARG and "null pair_q" in _lib.last_error()
        assert form(dev, R, C_, 2, R, C_, 2, flags=1, n_pairs=False, **kw) == ARG and "null pair_q" in _lib.last_error()
    if not dev:
        kw = dict(ql=LEN, rl=LEN, p=True)
        big = np.array([5, 2], np.uint32)
        assert form(dev, R, big, 2, R, C_, 2, **kw) == ARG and "query row 0 holds 5" in _lib.last_error()
        assert form(dev, R, C_, 2, R, big, 2, **kw) == ARG and "reference row 0" in _lib.last_error()
        for bad in ([[1, 1, 9, 0], [2, 5, 0, 0]], [[1, 5, 9, 0], [5, 2, 0, 0]]):
            b = np.array(bad, np.uint32)
            assert form(dev, b, C_, 2, R, C_, 2, **kw) == ARG and "ascending" in _lib.last_error()
            assert form(dev, R, C_, 2, b, C_, 2, **kw) == ARG and "ascending" in _lib.last_error()
        # the words past count are not read: a descending tail is fine as far as the rules go, and so is a 0 length
        # when no p-value is asked for (checked here only through the next rule firing)
        zero = np.array([1000, 0], np.uint64)
        assert form(dev, R, C_, 2, R, C_, 2, ql=zero, rl=LEN, p=True) == ARG and "length 1 is 0" in _lib.last_error()
        assert form(dev, R, C_, 2, R, C_, 2, ql=LEN, rl=zero, p=True) == ARG and "length 1 is 0" in _lib.last_error()


@pytest.mark.parametrize("dev", [False, True])
def test_empty_sides_are_valid(dev):
    # nq == 0 or nr == 0 needs no buffer on the empty side; the dense forms then touch no device
    assert dense(dev, None, None, 0, ROWS, CNT, 2, p=True, rl=LEN) == _lib.PG_OK
    assert dense(dev, ROWS, CNT, 2, None, None, 0, p=True, ql=LEN) == _lib.PG_OK
    assert dense(dev, None, None, 0, None, None, 0) == _lib.PG_OK
    if not dev:
        assert within(dev, None, None, 0, None, None, 0, flags=1) == _lib.PG_OK
    # the scalar rules still hold on empty sides
    assert dense(dev, None, None, 0, None, None, 0, k=0) == ARG
    assert dense(dev, None, None, 0, None, None, 0, s=5) == ARG


def test_python_mirror_rules():
    R, C_ = ROWS, CNT
    for kw in (dict(k=0), dict(k=1 << 31)):
        with pytest.raises(_lib.PolyError) as e:
            mash.dist(R, C_, R, C_, **kw)
        assert e.value.code == ARG
    with pytest.raises(ValueError):
        mash.dist(R, C_, np.zeros((2, 5), np.uint32), C_, 21)  # two sketch sizes
    with pytest.raises(ValueError):
        mash.dist(R, C_[:1], R, C_, 21)
    with pytest.raises(ValueError):
        mash.dist(R, C_, R, C_, 21, q_length=LEN)  # one side's lengths only
    with pytest.raises(_lib.PolyError) as e:
        mash.dist(R, np.array([9, 1], np.uint32), R, C_, 21)
    assert e.value.code == ARG
    with pytest.raises(_lib.PolyError) as e:
        mash.dist_within(R, C_, R, C_, 21, max_p_value=0.5)
    assert e.value.code == ARG
    with pytest.raises(_lib.PolyError) as e:
        mash.dist_within(R, C_, R[:1], C_[:1], 21, upper=True)
    assert e.value.code == ARG
    c, d, dist, p = mash.dist(np.zeros((0, 4), np.uint32), np.zeros(0, np.uint32), R, C_, 21)
    assert c.shape == (0, 2) and dist.shape == (0, 2) and p is None
    out = mash.dist_within(np.zeros((0, 4), np.uint32), np.zeros(0, np.uint32), R, C_, 21)
    assert all(len(o) == 0 for o in out[:5]) and out[5] is None


# ---- the oracle on hand-worked cases ----------------------------------------------------------------------------
@pytest.mark.parametrize("A,B,s,common,denom", [
    ([1, 2, 3], [4, 5, 6], 10, 0, 6),                 # disjoint ranges, union below s
    ([1, 2, 3], [4, 5, 6], 4, 0, 4),                  # disjoint ranges, union above s
    ([10, 20], [1, 2, 3, 4], 3, 0, 3),                # B ends (at s) before A starts
    ([1, 2, 3, 4], [1, 2, 3, 4], 4, 4, 4),            # identical rows
    ([1, 2, 3], [1, 2, 3, 4, 5], 5, 3, 5),            # A a prefix of B
    ([1, 2, 3, 4, 5], [1, 2, 3], 5, 3, 5),            # and the other way round
    ([], [], 5, 0, 0),                                # empty rows
    ([], [1, 2], 5, 0, 2),                            # one empty row
    ([1, 3, 5, 7], [2, 3, 6, 7], 10, 2, 6),           # |A u B| < s
    ([1, 3, 5, 7], [2, 3, 6, 7], 4, 1, 4),            # the shared 7 lies past the s-th union value
    ([1, 3, 5, 7], [2, 3, 6, 7], 6, 2, 6),            # union rank of 7 is exactly s - 1
    ([5], [5], 1, 1, 1),                              # s = 1
    ([5], [6], 1, 0, 1),
    ([6], [5, 6], 1, 0, 1),
    ([0, U32MAX], [0, U32MAX], 2, 2, 2),              # unsigned extremes
])
def test_oracle_counts(A, B, s, common, denom):
    assert O.compare(A, B, s) == (common, denom)
    assert O.compare(B, A, s) == (common, denom)
    assert O.compare(A, A, s) == (len(A), len(A))


def test_oracle_distance_branches():
    assert O.distance(0, 0, 21) == 0.0 and math.copysign(1, O.distance(0, 0, 21)) == 1
    assert O.distance(5, 5, 21) == 0.0
    assert O.distance(0, 5, 21) == 1.0
    j = 3 / 7
    assert O.distance(3, 7, 21) == -math.log(2 * j / (1 + j)) / 21
    # the clamp at 1: with k = 1, J = 1/1000 gives -ln(2/1001) = 6.2 > 1
    assert O.distance(1, 1000, 1) == 1.0
    assert O.distance(999, 1000, 1) < 1.0
    # two strains at 1 % substitutions, k = 21: (1 - p)^k agree of the union's share -> D near p
    a = 0.99 ** 21
    jj = a / (2 - a)
    assert abs(-math.log(2 * jj / (1 + jj)) / 21 + math.log(0.99)) < 1e-12


def test_oracle_p_value_branches():
    assert O.p_value(0, 100, 21, 10 ** 6, 10 ** 6) == 1.0
    assert O.p_value(5, 100, 600, 10 ** 6, 10 ** 6) == 0.0  # 4^k overflows: r = 0
    four_k = 4.0 ** 21
    pq, pr = 1 / (1 + four_k / 5e6), 1 / (1 + four_k / 2e6)
    assert O.pair_r(21, 5 * 10 ** 6, 2 * 10 ** 6) == pq * pr / (pq + pr - pq * pr)
    assert O.p_value(10, 10, 1, 10 ** 6, 10 ** 6) > 0.99  # k = 1: every k-mer is everywhere


def exact_tail(c: int, n: int, r: float) -> Fraction:
    x = Fraction(r)
    return sum((Fraction(math.comb(n, i)) * x ** i * (1 - x) ** (n - i) for i in range(c, n + 1)), Fraction(0))


@pytest.mark.parametrize("k,lq,lr", [(21, 5 * 10 ** 6, 5 * 10 ** 6), (16, 3 * 10 ** 6, 10 ** 5), (8, 10 ** 4, 10 ** 5), (4, 1000, 50), (12, 1, 10 ** 9)])
def test_oracle_p_value_against_exact_tail(k, lq, lr):
    r = O.pair_r(k, lq, lr)
    for n in (1, 2, 7, 30, 60):
        for c in sorted({1, 2, n // 3 or 1, n // 2 or 1, n - 1 or 1, n}):
            want = exact_tail(c, n, r)
            got = O.p_value(c, n, k, lq, lr)
            if want < Fraction(10) ** -290:
                assert got <= 1e-280
            else:
                assert abs(Fraction(got) - want) <= Fraction(1, 10 ** 9) * want, (c, n, got, float(want))
