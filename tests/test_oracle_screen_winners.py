"""CPU tier of the screen's winner-take-all restatement (tests/screen_winners_oracle.py): hand-worked
cases, a second, word-for-word Python restatement on small random inputs, and the properties the device tests lean
on (won counts never exceed the first pass, n = 1 and isolated references keep their results)."""
from collections import Counter

import numpy as np
import pytest

import oracle_ffi
import screen_oracle
import screen_winners_oracle

K = 4


def h(kmer: bytes) -> int:
    return oracle_ffi.murmur3_32(kmer)


def restate(sk, reads, k):
    """The definition, word for word: first-pass shared, each pool value's winner by (shared, -index) among the
    references holding it, then the multiset of won values per reference."""
    sk = np.asarray(sk, np.uint32)
    pool = Counter(h(r[p:p + k]) for r in reads for p in range(max(len(r) - k, 0)))
    n, s = sk.shape
    held = [Counter(int(x) for x in row) for row in sk]
    first = [sum(min(c, pool[v]) for v, c in held[i].items()) for i in range(n)]
    shared, cont, mult = np.zeros(n, np.uint32), np.zeros(n, np.float64), np.zeros(n, np.uint64)
    for i in range(n):
        ms = []
        for v, c_r in held[i].items():
            if pool[v] and all(first[j] < first[i] or (first[j] == first[i] and j > i) for j in range(n) if j != i and held[j][v]):
                ms += [pool[v]] * min(c_r, pool[v])
        ms.sort()
        shared[i], cont[i] = len(ms), len(ms) / s
        mult[i] = ms[(len(ms) - 1) // 2] if ms else 0
    return shared, cont, mult


def check(sk, reads, k, want_shared=None, want_mult=None):
    sk = np.asarray(sk, np.uint32)
    got = screen_winners_oracle.mash_screen_winners(sk, reads, k)
    want = restate(sk, reads, k)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.tobytes() == w.tobytes(), (g, w)
    if want_shared is not None:
        assert got[0].tolist() == want_shared
    if want_mult is not None:
        assert got[2].tolist() == want_mult
    first = screen_oracle.mash_screen(sk, reads, k)
    assert (got[0] <= first[0]).all() and int(got[0].sum()) <= int(first[0].sum())
    return got


def test_two_references_sharing_values():
    a, c, g = h(b"AAAA"), h(b"CCCC"), h(b"GGGG")
    reads = [b"A" * 7, b"C" * 5, b"G" * 6]  # pool counts a 3, c 1, g 2
    sk = [[a, c, 1, 2],  # first pass 1 + 1 = 2
          [a, g, g, 3]]  # first pass 1 + 2 = 3: takes a
    assert screen_oracle.mash_screen(np.array(sk, np.uint32), reads, K)[0].tolist() == [2, 3]
    # 0 keeps c alone: {1}; 1 keeps a and g: {3, 2, 2} -> lower median 2
    check(sk, reads, K, want_shared=[1, 3], want_mult=[1, 2])


def test_an_exact_tie_goes_to_the_lower_index():
    a, c, g = h(b"AAAA"), h(b"CCCC"), h(b"GGGG")
    reads = [b"A" * 7, b"C" * 5, b"G" * 6]
    row = [a, c, g, 5]
    check([row, row], reads, K, want_shared=[3, 0], want_mult=[2, 0])
    other = [a, 7, 8, 9]  # first pass 1: loses a to both copies
    check([other, row, row], reads, K, want_shared=[0, 3, 0], want_mult=[0, 2, 0])
    # the same first-pass shared through different values: a goes with the lower index, whichever row that is
    x, y = [a, c, 1, 2], [a, g, 4, 5]  # 1 + 1 and 1 + min(1, 2)
    check([x, y], reads, K, want_shared=[2, 1], want_mult=[1, 2])
    check([y, x], reads, K, want_shared=[2, 1], want_mult=[2, 1])


def test_a_reference_holding_a_value_several_times():
    a, c = h(b"AAAA"), h(b"CCCC")
    reads = [b"A" * 7, b"C" * 5]  # a 3, c 1
    sk = [[a, c, c, 0],   # first pass 1 + 1 = 2
          [a, a, a, a]]   # first pass min(4, 3) = 3: takes a with all three copies
    check(sk, reads, K, want_shared=[1, 3], want_mult=[1, 3])


def test_zero_tails_shared_by_several_references():
    z = screen_winners_oracle.window_hashing_to(0, K, b"ACGT")
    a, c = h(b"AAAA"), h(b"CCCC")
    reads = [z + b"T", z + b"G", b"A" * 7, b"C" * 5]  # c_pool(0) = 2, a 3, c 1
    sk = [[a, 0, 0, 0],   # 1 + 2 = 3
          [a, c, 0, 0],   # 1 + 1 + 2 = 4: takes 0 and a
          [0, 0, 0, 0],   # 2
          [c, 0, 5, 6]]   # 1 + 1 = 2
    # 1: {3, 1, 2, 2} -> 2; the others keep nothing
    check(sk, reads, K, want_shared=[0, 4, 0, 0], want_mult=[0, 2, 0, 0])
    # without a pool window that hashes to 0, zero tails share nothing
    check(sk, reads[2:], K, want_shared=[0, 2, 0, 0])


def test_n_one_equals_the_first_pass():
    rng = np.random.default_rng(3)
    reads = [bytes(rng.choice(list(b"ACGT"), 40)) for _ in range(20)]
    ph = [h(r[p:p + K]) for r in reads for p in range(len(r) - K)]
    sk = np.where(rng.random((1, 30)) < 0.7, rng.choice(ph, (1, 30)), 0).astype(np.uint32)
    got = check(sk, reads, K)
    for g, w in zip(got, screen_oracle.mash_screen(sk, reads, K)):
        assert g.tobytes() == w.tobytes()
    assert got[0][0] > 0


def test_an_empty_pool_gives_zeros():
    a = h(b"AAAA")
    for reads in ([], [b"", b"ACG"]):
        got = check([[a, 0], [a, 1]], reads, K, want_shared=[0, 0], want_mult=[0, 0])
        assert got[1].tolist() == [0.0, 0.0]


def test_a_reference_sharing_nothing_with_the_others_keeps_its_results():
    a, c, g, t = h(b"AAAA"), h(b"CCCC"), h(b"GGGG"), h(b"TTTT")
    reads = [b"A" * 7, b"C" * 5, b"G" * 6, b"T" * 9]
    sk = np.array([[a, c, 1, 2], [a, c, a, 3], [g, t, t, 0]], np.uint32)  # 2 shares no value with 0 or 1
    got = check(sk, reads, K)
    first = screen_oracle.mash_screen(sk, reads, K)
    assert [x[2] for x in got] == [x[2] for x in first] and got[0][2] == 3


@pytest.mark.parametrize("seed", range(8))
def test_random_inputs_match_the_restatement(seed):
    rng = np.random.default_rng(100 + seed)
    k = int(rng.choice([0, 1, 3, 4, 5]))
    reads = [bytes(rng.choice(list(b"ACGT"[: int(rng.integers(1, 5))]), int(rng.integers(0, 40)))) for _ in range(int(rng.integers(0, 30)))]
    ph = [h(r[p:p + k]) for r in reads for p in range(max(len(r) - k, 0))] or [7]
    n, s = int(rng.integers(1, 14)), int(rng.integers(1, 20))
    # families: rows copied from a few bases with some words replaced, so values are contended and ties occur
    base = np.where(rng.random((3, s)) < 0.7, rng.choice(ph, (3, s)), rng.choice([0, 1, 0xFFFFFFFF], (3, s)))
    sk = base[rng.integers(0, 3, n)]
    swap = rng.random((n, s)) < 0.3
    sk = np.where(swap, rng.choice(ph + [0], (n, s)), sk).astype(np.uint32)
    got = check(sk, reads, k)
    # reordering the rows moves each winner with its index, up to the ties
    perm = rng.permutation(n)
    first = screen_oracle.mash_screen(sk, reads, k)[0]
    if len(set(first.tolist())) == n:  # no tie: the winners follow their rows
        again = screen_winners_oracle.mash_screen_winners(sk[perm], reads, k)
        assert all(a.tobytes() == b[perm].tobytes() for a, b in zip(again, got))
