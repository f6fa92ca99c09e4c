"""CPU tier of the screen's restatement (tests/screen_oracle.py): hand-worked cases, and a second, word-for-word
Python restatement of the definition (one murmur3 call per window, Counter arithmetic) on small random inputs."""
from collections import Counter

import numpy as np
import pytest

import oracle_ffi
import screen_oracle

K = 4


def h(kmer: bytes) -> int:
    return oracle_ffi.murmur3_32(kmer)


def restate(sk, reads, k):
    """The definition, word for word: pool counts over windows 0 .. L - k - 1, then per reference the multiset
    min(c_r, c_pool) and the lower median of the shared hashes' pool counts."""
    pool = Counter(h(r[p:p + k]) for r in reads for p in range(max(len(r) - k, 0)))
    n, s = sk.shape
    shared, cont, mult = np.zeros(n, np.uint32), np.zeros(n, np.float64), np.zeros(n, np.uint64)
    for i in range(n):
        ms = []
        for v, c_r in Counter(int(x) for x in sk[i]).items():
            ms += [pool[v]] * min(c_r, pool[v])
        ms.sort()
        shared[i], cont[i] = len(ms), len(ms) / s
        mult[i] = ms[(len(ms) - 1) // 2] if ms else 0
    return shared, cont, mult


def check(sk, reads, k, want_shared=None, want_mult=None):
    got = screen_oracle.mash_screen(sk, reads, k)
    want = restate(np.asarray(sk, np.uint32), reads, k)
    for g, w in zip(got, want):
        assert np.array_equal(g, w) and g.tobytes() == w.tobytes(), (g, w)
    if want_shared is not None:
        assert got[0].tolist() == want_shared
    if want_mult is not None:
        assert got[2].tolist() == want_mult
    return got


def test_duplicate_words_and_pool_counts_on_either_side():
    a, c, g = h(b"AAAA"), h(b"CCCC"), h(b"GGGG")
    # pool: AAAA x 3 (read of 7 A: windows 0..2), CCCC x 1 (read of 5 C: window 0)
    reads = [b"A" * 7, b"C" * 5]
    sk = np.array([
        [a, a, c, c, g],  # c_r(a) = 2 < c_pool 3 -> 2; c_r(c) = 2 > c_pool 1 -> 1; g absent
        [a, a, a, a, a],  # min(5, 3) = 3
    ], np.uint32)
    s, _, m = check(sk, reads, K, want_shared=[3, 3])
    # reference 0: multiset {3, 3, 1} -> sorted {1, 3, 3}, lower median element 1 = 3
    assert m.tolist() == [3, 3]


def test_lower_median_of_even_and_odd_counts():
    a, c, t = h(b"AAAA"), h(b"CCCC"), h(b"TTTT")
    reads = [b"A" * 5, b"C" * 6, b"T" * 9]  # pool counts 1, 2, 5
    sk = np.array([
        [a, c, 1, 2],   # {1, 2}: even, lower median = 1
        [a, c, t, 3],   # {1, 2, 5}: odd, median = 2
        [c, c, t, t],   # {2, 2, 5, 5}: even, lower median = 2
        [5, 6, 7, 8],   # nothing shared -> 0
    ], np.uint32)
    check(sk, reads, K, want_shared=[2, 3, 4, 0], want_mult=[1, 2, 2, 0])


def test_zero_tail_words_and_short_reads():
    zero_pool = [bytes(8)]  # every window of zero bytes hashes to one value, not to 0
    z = h(bytes(K))
    sk = np.array([[z, 0, 0, 0], [0, 0, 0, 0]], np.uint32)
    check(sk, zero_pool, K, want_shared=[1, 0])
    # reads with L <= k contribute nothing, L = k + 1 exactly one window
    a = h(b"ACGT")
    sk = np.array([[a, 0]], np.uint32)
    check(sk, [b"", b"ACG", b"ACGT"], K, want_shared=[0])
    check(sk, [b"ACGTA"], K, want_shared=[1], want_mult=[1])


def test_k_zero_hashes_every_position_to_the_empty_hash():
    e = h(b"")
    sk = np.array([[e, e, 9]], np.uint32)
    check(sk, [b"ACG", b"T"], 0, want_shared=[2], want_mult=[4])


def test_no_references_and_no_reads():
    assert [len(x) for x in screen_oracle.mash_screen(np.zeros((0, 4), np.uint32), [b"ACGTACGT"], K)] == [0, 0, 0]
    check(np.array([[1, 2, 3]], np.uint32), [], K, want_shared=[0])


@pytest.mark.parametrize("seed", range(6))
def test_random_inputs_match_the_restatement(seed):
    rng = np.random.default_rng(seed)
    k = int(rng.choice([0, 1, 3, 4, 5, 8]))
    reads = [bytes(rng.choice(list(b"ACGT"[: int(rng.integers(1, 5))]), int(rng.integers(0, 40)))) for _ in range(int(rng.integers(0, 30)))]
    pool_hashes = [h(r[p:p + k]) for r in reads for p in range(max(len(r) - k, 0))] or [7]
    n, s = int(rng.integers(1, 12)), int(rng.integers(1, 24))
    # reference words: pool hashes (some repeated), zeros and random values, in any order
    sk = np.where(rng.random((n, s)) < 0.6, rng.choice(pool_hashes, (n, s)), rng.choice([0, 1, 0xFFFFFFFF], (n, s)))
    check(sk.astype(np.uint32), reads, k)
    bases, off = oracle_ffi.ragged(reads)
    assert sorted(screen_oracle.pool_hashes(bases, off, k).tolist()) == sorted(h(r[p:p + k]) for r in reads for p in range(max(len(r) - k, 0)))
    for threads in (2, 7):
        a = screen_oracle.mash_screen(sk, reads, k, nthreads=threads)
        b = screen_oracle.mash_screen(sk, reads, k)
        assert all(np.array_equal(x, y) for x, y in zip(a, b))
