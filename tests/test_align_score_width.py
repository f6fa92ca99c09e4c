"""CPU tier: the score-width rule of the alignment kernels (score_bound and score_packed16 in
poly_b200/csrc/align_core.cuh), compiled on the host with nvcc.  Every alignment kernel runs its DP in 2 x int16,
int32 or int64 cells as this rule says, so the bound must hold for every value a kernel computes: here it is checked
against an exact restatement of the DP in Python integers over small shapes, then the chosen width is checked just
below and just above each threshold."""
import itertools
import os
import shutil
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "poly_b200", "csrc")

# one call per input line "global max|S| gap short_len sum_len n_queries" -> "bound int32 packed16"; PACKED is
# score_packed16, or 0 for the bound alone
PROGRAM = r"""
#include <cstdio>
#include "align_core.cuh"

int main() {
    int global;
    long long amax, gap;
    unsigned long long short_len, sum_len, nq;
    while (std::scanf("%d %lld %lld %llu %llu %llu", &global, &amax, &gap, &short_len, &sum_len, &nq) == 6) {
        const long double bound = pg::score_bound(global, amax, gap, short_len, sum_len);
        std::printf("%.0Lf %d %d\n", bound, bound < pg::SCORE32_LIMIT, (int)(PACKED));
    }
    return 0;
}
"""


def nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    pytest.fail("nvcc not found: the width rule is checked by compiling its header")


def compile_rule(d, packed):
    """[(bound, int32, packed16)] of [(global, max|S|, gap, short_len, sum_len, n_queries)], from the header itself."""
    src, exe = d / "width.cu", d / "width"
    src.write_text(PROGRAM.replace("PACKED", packed))
    r = subprocess.run([nvcc(), "-std=c++17", "-O1", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC,
                        str(src), "-o", str(exe)], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr

    def run(cases):
        out = subprocess.run([str(exe)], input="".join("%d %d %d %d %d %d\n" % c for c in cases), capture_output=True, text=True,
                             check=True).stdout.split("\n")
        return [(int(b), bool(int(w)), bool(int(p))) for b, w, p in (line.split() for line in out if line)]

    return run


@pytest.fixture(scope="module")
def bound_rule(tmp_path_factory):
    return compile_rule(tmp_path_factory.mktemp("score_bound"), "0")


@pytest.fixture(scope="module")
def width_rule(tmp_path_factory):
    return compile_rule(tmp_path_factory.mktemp("score_width"), "pg::score_packed16(global, gap, bound, nq)")


def dp_extremes(a, b, S, gap, global_alignment):
    """align.go's fill (NW :113-135, SW :180-196) in exact integers: the largest |H| over every cell, boundaries
    included, and the largest |x| over every add a cell makes (diag + S, up + gap, left + gap)."""
    prev = [j * gap if global_alignment else 0 for j in range(len(b) + 1)]
    big = max(abs(x) for x in prev)
    for i in range(1, len(a) + 1):
        cur = [i * gap if global_alignment else 0]
        for j in range(1, len(b) + 1):
            d, u, l = prev[j - 1] + S[a[i - 1]][b[j - 1]], prev[j] + gap, cur[j - 1] + gap
            cur.append(max(d, u, l) if global_alignment else max(0, d, u, l))
            big = max(big, abs(d), abs(u), abs(l), abs(cur[j]))
        prev = cur
    return big


TABLES = {
    "one_large": [[1, -1, -1], [-1, 1, -1], [-1, -1, 40]],
    "one_large_negative": [[1, -45, -1], [-1, 1, -1], [-1, -1, 1]],
    "all_negative": [[-2, -5, -1], [-3, -4, -6], [-1, -2, -7]],
    "mixed": [[3, -3, 0], [-3, 3, -1], [0, -1, 2]],
}
MAX_LEN = 12


def strings(S, la, lb, rng):
    """Pairs that reach the extremes: repeats of the largest entry's symbols, of the smallest's, and a random pair."""
    S = np.asarray(S)
    hi = np.unravel_index(S.argmax(), S.shape)
    lo = np.unravel_index(S.argmin(), S.shape)
    yield [hi[0]] * la, [hi[1]] * lb
    yield [lo[0]] * la, [lo[1]] * lb
    yield list(rng.integers(0, 3, la)), list(rng.integers(0, 3, lb))


@pytest.mark.parametrize("gap", [-9, -1, 0, 1, 7])
@pytest.mark.parametrize("global_alignment", [False, True], ids=["local", "global"])
def test_bound_covers_every_value(bound_rule, global_alignment, gap):
    """Lengths 0..12 on either side (the shorter string as a and as b): score_bound is at least every |H| and
    every add's result, so a width that holds the bound holds the DP."""
    rng = np.random.default_rng(gap + 100 + 1000 * global_alignment)
    cases, need = [], []
    for (name, S), la, lb in itertools.product(TABLES.items(), range(MAX_LEN + 1), range(MAX_LEN + 1)):
        amax = int(np.abs(S).max())
        for a, b in strings(S, la, lb, rng):
            cases.append((int(global_alignment), amax, gap, min(la, lb), la + lb, 2))
            need.append((dp_extremes(a, b, S, gap, global_alignment), name, la, lb))
    got = bound_rule(cases)
    short = [(name, la, lb, bound, v) for (bound, _, _), (v, name, la, lb) in zip(got, need) if bound < v]
    assert not short, short[:5]


def test_width_edges(width_rule):
    """Each threshold from just below and just above: (case) -> (bound, int32, packed int16)."""
    lim = 2_000_000_000
    cases = {
        # packed int16: local, gap <= 0, bound < 16000, |gap| < 16000, two queries
        (0, 615, -1, 25, 10025, 2): (15990, True, True),       # 26 * 615: the headline primer shape scaled up
        (0, 616, -1, 25, 10025, 2): (16016, True, False),
        (0, 3, -2, 25, 10025, 2): (78, True, True),            # the headline primer shape itself
        (0, 3, -2, 25, 10025, 1): (78, True, False),           # one query
        (0, 3, 0, 25, 10025, 2): (78, True, True),
        (0, 3, 1, 25, 10025, 2): (30081, True, False),         # a positive gap: never packed
        (0, 3, 1, 2, 3, 2): (15, True, False),
        (1, 3, -2, 25, 10025, 2): (30081, True, False),        # global: never packed
        (0, 0, -15999, 5, 10, 2): (15999, True, True),
        (0, 0, -16000, 5, 10, 2): (16000, True, False),
        (0, 666, -1, 23, 10023, 2): (15984, True, True),
        (0, 667, -1, 23, 10023, 2): (16008, True, False),
        # int32: bound < 2e9
        (0, 76_923_076, -1, 25, 10025, 2): (1_999_999_976, True, False),
        (0, 76_923_077, -1, 25, 10025, 2): (2_000_000_002, False, False),
        (0, 80_000_000, -1, 24, 10024, 2): (lim, False, False),  # exactly the limit: int64
        (0, 79_999_999, -1, 24, 10024, 2): (lim - 25, True, False),
        (1, 3, -664_451, 8, 3008, 2): (664_451 * 3010, True, False),
        (1, 3, -664_452, 8, 3008, 2): (664_452 * 3010, False, False),
        (1, 1_999_999_999, 0, 0, 0, 2): (2 * 1_999_999_999, False, False),
        (1, 999_999_999, 0, 0, 0, 2): (1_999_999_998, True, False),
        # a positive gap takes the global form: values grow with the longer string
        (0, 3, 2**20, 10, 3010, 2): (2**20 * 3012, False, False),
        (0, 3, 664_010, 10, 3010, 2): (664_010 * 3012, True, False),
        (0, 3, 664_011, 10, 3010, 2): (664_011 * 3012, False, False),
        (0, 3, 1, 10, 3010, 2): (3 * 3012, True, False),
    }
    got = dict(zip(cases, width_rule(list(cases))))
    bad = {c: (got[c], w) for c, w in cases.items() if got[c] != w}
    assert not bad, bad
