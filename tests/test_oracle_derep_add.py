"""CPU tier: a growing dereplication, restated batch by batch (tests/derep_add_oracle.py: links from the kept
representatives seed a batch, then the greedy rule runs inside it), equals the dereplication oracle of the
concatenated set for any split.  This is the decomposition pg_mash_dereplicator_add relies on."""
import numpy as np
import pytest

import derep_add_oracle
import derep_oracle
import oracle_ffi
from poly_b200 import mash, synth


def counts(sk):
    rc, same = oracle_ffi.similarity_block(sk, 0, len(sk), 0, len(sk))
    assert rc == 0
    return same


@pytest.fixture(scope="module")
def survey_sample():
    """The 8-read, R = 4 family sample of SURVEY 8d (10 kbp, k = 31, s = 2000)."""
    n, L, k, s = 8, 10000, 31, 2000
    rc, sk = oracle_ffi.sketch_batch(synth.family_reads(n, L, family=4), synth.uniform_offsets(n, L), k, s, variant=1)
    assert rc == 0
    return sk


@pytest.fixture(scope="module")
def families():
    """48 reads of 2 kbp in families of 8, k = 21, s = 400."""
    n, L, k, s = 48, 2000, 21, 400
    rc, sk = oracle_ffi.sketch_batch(synth.family_reads(n, L, family=8), synth.uniform_offsets(n, L), k, s, variant=1)
    assert rc == 0
    return sk


def random_cuts(rng, n, k):
    return sorted(int(c) for c in rng.integers(0, n + 1, size=k))  # repeats give empty batches


def test_random_splits_equal_the_whole(survey_sample, families):
    rng = np.random.default_rng(7)
    for sk in (survey_sample, families):
        n, s = sk.shape
        same = counts(sk)
        off = sorted({int(c) for c in np.triu(same, 1).ravel()} - {0} | {1, s})
        for c in off[:: max(1, len(off) // 10)] + off[-2:]:
            d = 1.0 - np.float64(c) / np.float64(s)  # exactly on the Distance of the pairs that count c
            assert mash.min_same_for_distance(d, s) == c
            for nearest in (False, True):
                want = derep_oracle.dereplicate(sk, c, nearest)
                splits = [[], list(range(1, n)), [0, 0, n, n]] + [random_cuts(rng, n, k) for k in (1, 2, 3, 6)]
                for cuts in splits:
                    got = derep_add_oracle.dereplicate_in_batches(sk, cuts, c, nearest)
                    assert np.array_equal(got[0], want[0]) and got[1] == want[1], (c, nearest, cuts)


def test_only_the_representatives_are_kept(families):
    g = derep_add_oracle.GrowingDereplication(400, 150, nearest=True)
    first = g.add(families[:20])
    rep, n_reps = derep_oracle.dereplicate(families[:20], 150, True)
    assert np.array_equal(first[0], rep) and first[1] == n_reps
    assert g.rep_ids == [int(i) for i in np.nonzero(rep == np.arange(20))[0]]
    assert np.array_equal(g.rep_rows, families[:20][rep == np.arange(20)])


def hand_sets(n_a, n_b):
    """Sketches 0 (the even values 2..40) and 1 (the odd values 1..39) share nothing; sketch 2 takes n_a of 0's
    values and n_b of 1's, and is padded above both with its own."""
    s = 20
    a, b = np.arange(2, 41, 2, dtype=np.uint32), np.arange(1, 40, 2, dtype=np.uint32)
    c = np.sort(np.r_[a[:n_a], b[:n_b], 100 + np.arange(s - n_a - n_b, dtype=np.uint32)])
    return np.stack([a, b, c])


def test_cross_batch_tie_goes_to_the_kept_representative():
    """Row 2 is as close to 0 (kept by the first batch) as to 1 (a representative of its own batch): the kept
    one, the smaller id, wins in both modes."""
    sk = hand_sets(9, 9)
    same = counts(sk)
    assert (same[0, 1], same[2, 0], same[2, 1]) == (0, 9, 9)
    for nearest in (False, True):
        for cuts in ([1], [1, 2], [2]):
            got = derep_add_oracle.dereplicate_in_batches(sk, cuts, 5, nearest)
            assert list(got[0]) == [0, 1, 0] and got[1] == 2, (nearest, cuts)
    # 1 closer than 0: nearest moves row 2 to the batch's own representative, first keeps the kept one
    sk = hand_sets(7, 12)
    for cuts in ([1], [2]):
        assert list(derep_add_oracle.dereplicate_in_batches(sk, cuts, 5)[0]) == [0, 1, 0]
        assert list(derep_add_oracle.dereplicate_in_batches(sk, cuts, 5, True)[0]) == [0, 1, 1]


def test_empty_batches():
    g = derep_add_oracle.GrowingDereplication(16, 1)
    rep, n_new = g.add(np.zeros((0, 16), np.uint32))
    assert (len(rep), n_new, g.n) == (0, 0, 0)
