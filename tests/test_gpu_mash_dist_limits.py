"""GPU tier of the Mash distance at its numeric limits (pg_mash_dist): the p-value against an exact binomial tail
(mash_dist_oracle.p_value_exact) for sketch sizes 1 .. 2^24, r from 1e-9 to 1 - 1e-9, common across each tail and on
both sides of the incomplete beta's branch switch; the edges of r (exactly 1, tiny, subnormal, 4^k overflowing) and of
the lengths; and the merge and the distance at s = 2^21, where both rows are read from global memory.

Pairs are chosen through the real entry point: for a target denom n the reference row B is a strictly ascending list
of n values (0 and 2^32 - 1 among them) and query row A_i is its first c_i values, so with s = n every pair has
common = c_i and denom = n; r is set per pair by the query length (mash_dist_oracle.length_for_r) against a reference
of length 2^64 - 1.

Where the exact tail p >= 1e-300 the device must hold |p_gpu - p| <= (tol(n) + 4 eps kappa) p, with
tol(n) = 4e-12 max(1, sqrt(n / 10^4)) and kappa = |d ln p / d ln r|, which covers an ulp of difference between the
device's r and the oracle's (the device may fuse pq + pr - pq pr into one FMA).  Below 1e-300 it must give
0 <= p_gpu <= 2e-300.  Every p-value is finite, in [0, 1] and never -0.0."""
import math

import numpy as np
import pytest

import mash_dist_oracle as O
from poly_b200 import mash

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -52
RL = O.U64MAX  # every reference row's length
K_LOW, K_HIGH = 30, 16  # against length 2^64 - 1, query lengths reach r in (1e-10, 0.94) at k = 30, (2.3e-10, 1 - 4.6e-10) at k = 16
R_SIDE = [float(x) for x in np.logspace(-9, math.log10(0.5), 7)]  # r, and 1 - r, from 1e-9 to 0.5
Z = (-6, -2, -0.5, 0, 0.5, 2, 5, 8)


def tol(n: int) -> float:
    return 4e-12 * max(1.0, math.sqrt(n / 1e4))


def branch_switch(c: int, n: int) -> float:
    """The r at which mash_p_value changes branch, in the device's arithmetic: r < (a + 1) / (a + b + 2)."""
    a, b = float(c), float(n) - c + 1.0
    return (a + 1.0) / (a + b + 2.0)


def grid(n: int):
    """{k: [(common, query length)]}: r on both log scales with common at Z standard deviations around n r and at
    1, 2, n - 1, n; and, for common spread over [1, n], the two lengths one step either side of the branch switch."""
    out = {K_LOW: set(), K_HIGH: set()}
    ends = {1, 2, n - 1, n}
    for k, target in [(K_LOW, r) for r in R_SIDE] + [(K_HIGH, 1.0 - r) for r in R_SIDE]:
        lq = O.length_for_r(k, RL, target)
        r = O.pair_r(k, lq, RL)
        sd = math.sqrt(n * r * (1.0 - r))
        for c in ends | {int(round(n * r + z * sd)) for z in Z}:
            if 1 <= c <= n:
                out[k].add((c, lq))
    for c in {1, 2, n // 10, n // 3, n // 2, n - n // 10, n - 10, n - 2, n - 1, n}:
        if 1 <= c <= n:
            sw = branch_switch(c, n)
            k = K_LOW if sw <= 0.5 else K_HIGH
            lq = O.length_for_r(k, RL, sw)
            out[k] |= {(c, lq - 1), (c, lq)}
    return {k: sorted(v) for k, v in out.items() if v}


def device_counts(master_t, k: int, pairs, torch):
    """(common, denom, distance, p) of query rows master[:c] of length lq, for (c, lq) in pairs, against B = master of
    length RL, s = len(master), through pg_mash_dist_dev."""
    n = int(master_t.numel())
    nq = len(pairs)
    rows = master_t.unsqueeze(0).expand(nq, n).contiguous()
    qc = torch.tensor([c for c, _ in pairs], dtype=torch.int32, device="cuda")
    ql = torch.from_numpy(np.array([lq for _, lq in pairs], np.uint64).view(np.int64)).cuda()
    rl = torch.from_numpy(np.array([RL], np.uint64).view(np.int64)).cuda()
    rc = torch.tensor([n], dtype=torch.int32, device="cuda")
    out = mash.dist(rows, qc, master_t.unsqueeze(0), rc, k, ql, rl)
    torch.cuda.synchronize()
    del rows
    c, d, dist, p = (t[:, 0].cpu().numpy() for t in out)
    return c.view(np.uint32), d.view(np.uint32), dist, p


def p_errors(n: int, k: int, pairs, p_dev):
    """[(err / bound, common, length, r)] of each pair whose exact p >= 1e-300; asserts the rest and the range rules."""
    ratios = []
    for (c, lq), p in zip(pairs, p_dev):
        p = float(p)
        assert math.isfinite(p) and 0.0 <= p <= 1.0 and not math.copysign(1.0, p) < 0, (n, c, lq, p)
        r = O.pair_r(k, lq, RL)
        pe = O.p_value_exact(c, n, r)
        if pe < 1e-300:
            assert p <= 2e-300, (n, c, lq, r, p, float(pe))
            continue
        bound = tol(n) + 4 * EPS * O.p_value_kappa(c, n, r, pe)
        ratios.append((float(abs(p - pe) / pe) / bound, c, lq, r))
    return ratios


def master_on_device(n: int, torch):
    master = O.master_list(np.random.default_rng(1000 + n), n)
    return master, torch.from_numpy(master.view(np.int32)).cuda()


def check_grid(n: int, torch):
    master, master_t = master_on_device(n, torch)
    ratios = []
    for k, pairs in grid(n).items():
        c, d, dist, p = device_counts(master_t, k, pairs, torch)
        want_c = np.array([cc for cc, _ in pairs], np.uint32)
        assert np.array_equal(c, want_c) and (d == n).all()
        ratios += p_errors(n, k, pairs, p)
    worst = sorted(ratios, reverse=True)[:5]
    assert worst[0][0] <= 1.0, f"n = {n}: worst |p - exact| / bound (err/bound, common, query length, r): {worst}"


@pytest.mark.parametrize("n", [1, 2, 31, 32, 33, 1000, 3418, 3419, 10 ** 4, 10 ** 5, 1 << 21])
def test_p_value_grid_against_exact_tail(gpu, n):
    import torch

    check_grid(n, torch)


def test_p_value_at_s_2_24(gpu):
    # a row of 2^24 values is 64 MiB: a few pairs, at r = 0.5 around the mean and in the far tail, near r = 1, and at
    # the branch switch of a common near n
    import torch

    n = 1 << 24
    master, master_t = master_on_device(n, torch)
    lq_half = O.length_for_r(K_LOW, RL, 0.5)
    r = O.pair_r(K_LOW, lq_half, RL)
    sd = math.sqrt(n * r * (1 - r))
    low = [(int(round(n * r + z * sd)), lq_half) for z in (-2, 0, 2, 8)]
    lq_hi = O.length_for_r(K_HIGH, RL, 1 - 1e-6)
    sw = O.length_for_r(K_HIGH, RL, branch_switch(n - 10, n))
    high = [(n - 20, lq_hi), (n - 10, sw - 1), (n - 10, sw)]
    ratios = []
    for k, pairs in ((K_LOW, low), (K_HIGH, high)):
        c, d, _, p = device_counts(master_t, k, pairs, torch)
        assert np.array_equal(c, [cc for cc, _ in pairs]) and (d == n).all()
        ratios += p_errors(n, k, pairs, p)
    worst = max(ratios)
    assert worst[0] <= 1.0, f"n = 2^24: worst |p - exact| / bound (err/bound, common, query length, r): {worst}"


@pytest.mark.parametrize("n", [1000, 3418])
def test_p_value_sweeps_every_common(gpu, n):
    # common = 0 .. n at three r: every p against the exact tail, and p never rises with common
    import torch

    master, master_t = master_on_device(n, torch)
    for target in (0.01, 0.5, 0.97):
        lq = O.length_for_r(K_HIGH, RL, target)
        pairs = [(c, lq) for c in range(n + 1)]
        c, d, _, p = device_counts(master_t, K_HIGH, pairs, torch)
        assert np.array_equal(c, np.arange(n + 1)) and (d == n).all()
        assert p[0] == 1.0 and (np.diff(p) <= 0).all(), target
        ratios = p_errors(n, K_HIGH, pairs, p)
        worst = max(ratios)
        assert worst[0] <= 1.0, f"n = {n}: worst |p - exact| / bound (err/bound, common, query length, r): {worst}"


def test_p_value_small_denoms_sweep_every_common(gpu):
    # n <= 16, every common, five r: reaches every entry of the device's Stirling table, and the first of its series
    import torch

    for n in range(1, 17):
        master, master_t = master_on_device(n, torch)
        pairs = [(c, O.length_for_r(K_HIGH, RL, t)) for t in (1e-3, 0.3, 0.5, 0.8, 0.999) for c in range(n + 1)]
        c, d, _, p = device_counts(master_t, K_HIGH, pairs, torch)
        assert np.array_equal(c, [cc for cc, _ in pairs]) and (d == n).all()
        worst = max(p_errors(n, K_HIGH, pairs, p))
        assert worst[0] <= 1.0, (n, worst)


# ---- edges of r and of the lengths ------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 16, 21, 32, 268, 269, 509, 510, 511, 512])
def test_r_and_length_edges(gpu, k):
    # r == 1 exactly (k = 1, both lengths >= 2^56: p = 1); r tiny (k = 32, length 1: 2.7e-20); pq pr subnormal
    # (k = 268: r = 2^-537) or underflowing to 0 (k = 269, lengths 1); pq at the smallest normal doubles
    # (k = 509 .. 511, length 1), where pq pr underflows for any lengths: r = 0, p = 0, never NaN; 4^k overflowing
    # (k = 512: r = 0, p = 0, as the header states); lengths 1, 2, 2^56 and 2^64 - 1 on both sides
    n = 40
    master = O.master_list(np.random.default_rng(k), n)
    cs = [0, 1, 2, 20, 39, 40]
    lens = [1, 2, 1 << 56, O.U64MAX]
    q = np.tile(master, (len(cs) * len(lens), 1))
    qc = np.array([c for c in cs for _ in lens], np.uint32)
    ql = np.array([ln for _ in cs for ln in lens], np.uint64)
    r_rows, rc, rl = np.tile(master, (len(lens), 1)), np.full(len(lens), n, np.uint32), np.array(lens, np.uint64)
    c, d, dist, p = mash.dist(q, qc, r_rows, rc, k, ql, rl)
    assert np.array_equal(c, np.repeat(qc[:, None], len(lens), 1)) and (d == n).all()
    assert (dist == np.array([[O.distance(int(x), n, k) for x in row] for row in c])).all()
    for i in range(len(qc)):
        for j in range(len(lens)):
            common, pv = int(qc[i]), float(p[i, j])
            assert math.isfinite(pv) and 0.0 <= pv <= 1.0 and math.copysign(1.0, pv) > 0, (k, common, ql[i], rl[j], pv)
            r = O.pair_r(k, int(ql[i]), int(rl[j]))
            if common == 0 or r >= 1.0:
                assert pv == 1.0, (k, common, ql[i], rl[j], r, pv)
                continue
            if r == 0.0:
                assert pv == 0.0, (k, common, r, pv)
                continue
            pe = O.p_value_exact(common, n, r)
            if pe < 1e-300:
                assert pv <= 2e-300, (k, common, ql[i], rl[j], r, pv)
            else:
                bound = tol(n) + 4 * EPS * O.p_value_kappa(common, n, r, pe)
                assert abs(pv - pe) <= bound * pe, (k, common, ql[i], rl[j], r, pv, float(pe))
    if k == 1:
        assert O.pair_r(1, 1 << 56, 1 << 56) == 1.0 and (p[np.ix_((qc > 0) & (ql >= 1 << 56), [2, 3])] == 1.0).all()
    if k >= 509:
        assert all(O.pair_r(k, a, b) == 0.0 for a in lens for b in lens) and (p[qc > 0] == 0.0).all()


# ---- the merge and the distance at s = 2^21 --------------------------------------------------------------------
def test_merge_and_distance_at_s_2_21(gpu):
    # partial overlaps whose union reaches s inside one lane's range of the merge, a short row, an empty row against
    # a full one, and common = s - 1: common and denom against the NumPy restatement, distance within 2 ulp of the
    # oracle's literal formula
    s = 1 << 21
    rng = np.random.default_rng(2021)
    pool = O.master_list(rng, 3 * s)
    in_base = np.zeros(len(pool), bool)
    in_base[rng.choice(len(pool) - 1, size=s, replace=False)] = True  # 2^32 - 1, the pool's last value, stays out
    base, rest = pool[in_base], pool[~in_base]
    rows = [base]
    for share in (0.1, 0.5, 0.9, 0.999):
        keep = base[rng.random(s) < share]
        rows.append(np.sort(np.concatenate([keep, rng.choice(rest, size=s - len(keep), replace=False)])))
    rows.append(base[: s // 3])  # a short row
    rows.append(np.zeros(0, np.uint32))  # an empty row
    rows.append(np.delete(base, s // 2))  # common = s - 1 against base
    rows.append(np.append(np.delete(base, 7), np.uint32(O.U32 - 1)))  # the same with a full row
    m = len(rows)
    mat, cnt = np.zeros((m, s), np.uint32), np.array([len(x) for x in rows], np.uint32)
    for i, x in enumerate(rows):
        mat[i, : len(x)] = x
    # the merge's 32 lanes split P = min(a + b, 2 s) items evenly; the s-th union value of these pairs is inside a
    # lane's range, not on its edge
    for i in range(1, 5):
        merged = np.sort(np.concatenate([base, rows[i]]))
        first = np.ones(len(merged), bool)
        first[1:] = merged[1:] != merged[:-1]
        at = int(np.searchsorted(np.cumsum(first), s))  # the merge item holding the s-th union value
        assert at % (2 * s // 32) not in (0, 2 * s // 32 - 1)
    k = 21
    c, d, dist, _ = mash.dist(mat, cnt, mat, cnt, k)
    for i in range(m):
        for j in range(m):
            wc, wd = O.merge_counts(rows[i], rows[j], s)
            assert (c[i, j], d[i, j]) == (wc, wd), (i, j)
            want = O.distance(wc, wd, k)
            if want in (0.0, 1.0):
                assert dist[i, j] == want and not np.signbit(dist[i, j])
            else:
                assert abs(dist[i, j] - want) <= 2 * np.spacing(want), (i, j, dist[i, j], want)
    assert (c[0, 7], d[0, 7]) == (s - 1, s) and (c[0, 8], d[0, 8]) == (s - 1, s)
    assert (c[0, 6], d[0, 6], dist[0, 6]) == (0, s, 1.0)
