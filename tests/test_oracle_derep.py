"""CPU tier: the dereplication oracle (tests/derep_oracle.py) -- greedy representatives over the restated
Similarity, first or nearest assignment -- against values worked out by hand, its pair-list and literal-loop forms,
the single-linkage groups of the cluster oracle, and the threshold arithmetic of mash.dereplicate that needs no
device."""
import numpy as np
import pytest

import cluster_oracle
import derep_oracle
import oracle_ffi
from poly_b200 import mash, synth


def counts(sk):
    rc, same = oracle_ffi.similarity_block(sk, 0, len(sk), 0, len(sk))
    assert rc == 0
    return same


def as_mashes(sk, k=21):
    out = []
    for row in sk:
        m = oracle_ffi.OracleMash(k, sk.shape[1])
        m.Sketches[:] = row
        out.append(m)
    return out


@pytest.fixture(scope="module")
def survey_sample():
    """The 8-read, R = 4 family sample of SURVEY 8d (10 kbp, k = 31, s = 2000) and its count matrix."""
    n, L, k, s = 8, 10000, 31, 2000
    reads = synth.family_reads(n, L, family=4)
    rc, sk = oracle_ffi.sketch_batch(reads, synth.uniform_offsets(n, L), k, s, variant=1)
    assert rc == 0
    same = counts(sk)
    assert list(same[0]) == [2000, 758, 793, 714, 0, 0, 0, 0]
    return sk, same


@pytest.fixture(scope="module")
def families():
    """48 reads of 2 kbp in families of 8, k = 21, s = 400: enough links for both modes to differ."""
    n, L, k, s = 48, 2000, 21, 400
    rc, sk = oracle_ffi.sketch_batch(synth.family_reads(n, L, family=8), synth.uniform_offsets(n, L), k, s, variant=1)
    assert rc == 0
    return sk


# Worked out from the count matrix of the sample: row 0 = [2000, 758, 793, 714], rows 1..3 link each other at
# 733, 733, 732; row 4 = [737, 755, 712] towards 5, 6, 7; 5-6 at 787, 5-7 at 693, 6-7 at 704.
SURVEY_PINS = {
    1: [0, 0, 0, 0, 4, 4, 4, 4],  # every pair of a family links: the first member represents it
    700: [0, 0, 0, 0, 4, 4, 4, 4],
    715: [0, 0, 0, 3, 4, 4, 4, 7],  # 0-3 (714) and 4-7 (712) are cut: 3 and 7 are kept
    760: [0, 1, 0, 3, 4, 5, 5, 7],  # 0 keeps only 2 (793); 6 joins 5 (787) and not 4 (755)
    794: list(range(8)),  # above every off-diagonal count
}


@pytest.mark.parametrize("nearest", [False, True])
def test_survey_sample_pins(survey_sample, nearest):
    sk, _ = survey_sample
    for min_same, want in SURVEY_PINS.items():
        rep, n_reps = derep_oracle.dereplicate(sk, min_same, nearest)
        assert list(rep) == want and n_reps == len(set(want)), min_same


def test_three_forms_agree_over_a_threshold_sweep(survey_sample, families):
    for sk in (survey_sample[0], families):
        s = sk.shape[1]
        same = counts(sk)
        i, j = np.nonzero(np.triu(same, 1))
        mashes = as_mashes(sk)
        off = sorted({int(c) for c in same[i, j]} | {1, s})
        for c in off[:: max(1, len(off) // 12)] + off[-2:]:
            d = 1.0 - np.float64(c) / np.float64(s)  # exactly on the Distance of the pairs that count c
            assert mash.min_same_for_distance(d, s) == c
            for nearest in (False, True):
                want = derep_oracle.dereplicate(sk, c, nearest)
                got = derep_oracle.dereplicate_pairs(i, j, same[i, j], len(sk), c, nearest)
                assert np.array_equal(got[0], want[0]) and got[1] == want[1], (c, nearest)
                got = derep_oracle.dereplicate_literal(mashes, d, nearest)
                assert np.array_equal(got[0], want[0]) and got[1] == want[1], (c, nearest)
                for threads in (1, 3):
                    assert np.array_equal(derep_oracle.dereplicate(sk, c, nearest, nthreads=threads)[0], want[0])


def test_pair_list_order_and_direction_do_not_matter(survey_sample):
    sk, same = survey_sample
    i, j = np.nonzero(np.triu(same, 1))
    perm = np.random.default_rng(1).permutation(len(i))
    for min_same in (715, 760):
        want = derep_oracle.dereplicate(sk, min_same, True)
        # reversed triples, a diagonal entry and every pair listed twice
        pi, pj, ps = np.r_[j[perm], 3, i], np.r_[i[perm], 3, j], np.r_[same[i, j][perm], 2000, same[i, j]]
        got = derep_oracle.dereplicate_pairs(pi, pj, ps, 8, min_same, True)
        assert np.array_equal(got[0], want[0]) and got[1] == want[1]


def test_modes_share_the_representatives(survey_sample, families):
    differ = 0
    for sk in (survey_sample[0], families):
        same = counts(sk)
        for c in sorted({int(x) for x in np.triu(same, 1).ravel()} - {0}):
            first, nf = derep_oracle.dereplicate(sk, c)
            near, nn = derep_oracle.dereplicate(sk, c, True)
            idx = np.arange(len(sk))
            assert nf == nn and np.array_equal(first == idx, near == idx)
            # first takes the smallest linked representative, nearest one at least as close
            assert (first <= near).all() and (same[first, idx] <= same[near, idx]).all()
            differ += not np.array_equal(first, near)
    assert differ > 0


def hand_sets(n_a, n_b):
    """Sketches 0 (the even values 2..40) and 1 (the odd values 1..39) share nothing; sketch 2 takes n_a of 0's
    values and n_b of 1's, and is padded above both with its own."""
    s = 20
    a, b = np.arange(2, 41, 2, dtype=np.uint32), np.arange(1, 40, 2, dtype=np.uint32)
    c = np.sort(np.r_[a[:n_a], b[:n_b], 100 + np.arange(s - n_a - n_b, dtype=np.uint32)])
    return np.stack([a, b, c])


def test_nearest_and_first_differ_on_a_hand_built_set():
    sk = hand_sets(7, 12)
    same = counts(sk)
    assert (same[0, 1], same[0, 2], same[1, 2]) == (0, 7, 12)
    assert list(derep_oracle.dereplicate(sk, 5)[0]) == [0, 1, 0]
    assert list(derep_oracle.dereplicate(sk, 5, True)[0]) == [0, 1, 1]
    assert list(derep_oracle.dereplicate(sk, 8)[0]) == [0, 1, 1]  # 0-2 cut: only 1 is linked to 2
    for nearest in (False, True):
        assert list(derep_oracle.dereplicate(sk, 13, nearest)[0]) == [0, 1, 2]  # nothing links
    # a tie goes to the smaller index
    sk = hand_sets(9, 9)
    same = counts(sk)
    assert (same[0, 2], same[1, 2]) == (9, 9)
    for nearest in (False, True):
        assert list(derep_oracle.dereplicate(sk, 5, nearest)[0]) == [0, 1, 0]
        assert list(derep_oracle.dereplicate_literal(as_mashes(sk), 1 - 5 / 20, nearest)[0]) == [0, 1, 0]


def chain(n, step, s=16):
    """Sketch i = the s ascending values step * i ... step * i + s - 1."""
    return (np.arange(n, dtype=np.uint32)[:, None] * step + np.arange(s, dtype=np.uint32)).astype(np.uint32)


def test_chains():
    sk = chain(11, 8)  # neighbours share 8 values, i and i + 2 none
    same = counts(sk)
    assert (same[0, 1], same[0, 2]) == (8, 0)
    for nearest in (False, True):
        rep, n_reps = derep_oracle.dereplicate(sk, 8, nearest)
        assert list(rep) == [i - i % 2 for i in range(11)] and n_reps == 6
    sk = chain(11, 4)  # i ~ i + 1 (12), i + 2 (8); i + 3 shares 4
    same = counts(sk)
    assert (same[0, 1], same[0, 2], same[0, 3]) == (12, 8, 4)
    for nearest in (False, True):
        rep, n_reps = derep_oracle.dereplicate(sk, 8, nearest)
        assert list(rep) == [i - i % 3 for i in range(11)] and n_reps == 4
    # every sketch in one single-linkage group, yet not one within the cut of the first
    assert cluster_oracle.cluster(sk, 8)[1] == 1


def test_representatives_cover_and_are_unlinked(survey_sample, families):
    for sk in (survey_sample[0], families, chain(40, 4)):
        same = counts(sk)
        n = len(sk)
        idx = np.arange(n)
        for c in sorted({int(x) for x in np.triu(same, 1).ravel()} - {0})[::3]:
            label = cluster_oracle.cluster(sk, c)[0]
            for nearest in (False, True):
                rep, n_reps = derep_oracle.dereplicate(sk, c, nearest)
                is_rep = rep == idx
                assert n_reps == is_rep.sum() and (rep <= idx).all() and is_rep[rep].all()
                others = ~is_rep
                assert (same[rep[others], idx[others]] >= c).all()  # linked to its representative
                reps = idx[is_rep]
                assert not (np.triu(same[np.ix_(reps, reps)], 1) >= c).any()  # representatives pairwise unlinked
                assert (label[rep] == label).all()  # within i's single-linkage group


def test_empty_set():
    for nearest in (False, True):
        rep, n_reps = derep_oracle.dereplicate(np.zeros((0, 4), np.uint32), 1, nearest)
        assert (len(rep), n_reps) == (0, 0)
        rep, n_reps = derep_oracle.dereplicate_pairs([], [], [], 0, 1, nearest)
        assert (len(rep), n_reps) == (0, 0)


def test_mirror_thresholds_that_need_no_launch():
    sk = np.arange(12, dtype=np.uint32).reshape(3, 4)
    with pytest.raises(ValueError):
        mash.dereplicate(sk)
    with pytest.raises(ValueError):
        mash.dereplicate(sk, min_same=1, max_distance=0.5)
    with pytest.raises(ValueError, match="every pair"):
        mash.dereplicate(sk, max_distance=1.0, nearest=True)
    # no count reaches a negative distance: every sketch represents itself, without touching the library
    for nearest in (False, True):
        rep, n_reps = mash.dereplicate(sk, max_distance=-0.25, nearest=nearest)
        assert list(rep) == [0, 1, 2] and rep.dtype == np.uint32 and n_reps == 3
