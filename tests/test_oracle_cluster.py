"""CPU tier: the cluster oracle (tests/cluster_oracle.py) -- single-linkage groups over the restated
Similarity, labels = smallest index of the group -- against pinned values, a brute-force union-find in
Python and hand-built sketches; and the threshold arithmetic of mash.cluster that needs no device."""
import numpy as np
import pytest

import cluster_oracle
import oracle_ffi
from poly_b200 import mash, synth


def brute_labels(same: np.ndarray, min_same: int):
    """Labels, group count and link count from a dense count matrix (row = receiver), entries i < j only."""
    n = len(same)
    parent = list(range(n))

    def find(x):
        while parent[x] != x:
            x = parent[x]
        return x

    links = 0
    for i in range(n):
        for j in range(i + 1, n):
            if same[i, j] >= min_same:
                links += 1
                parent[find(i)] = find(j)  # any root: the labels below do not depend on it
    groups = {}
    for i in range(n):
        groups.setdefault(find(i), []).append(i)
    label = np.zeros(n, np.uint32)
    for members in groups.values():
        label[members] = min(members)
    return label, len(groups), links


@pytest.fixture(scope="module")
def survey_sample():
    """The 8-read, R = 4 family sample of SURVEY 8d (10 kbp, k = 31, s = 2000) and its count matrix."""
    n, L, k, s = 8, 10000, 31, 2000
    reads = synth.family_reads(n, L, family=4)
    rc, sk = oracle_ffi.sketch_batch(reads, synth.uniform_offsets(n, L), k, s, variant=1)
    assert rc == 0
    rc, same = oracle_ffi.similarity_block(sk, 0, n, 0, n)
    assert rc == 0 and list(same[0]) == [2000, 758, 793, 714, 0, 0, 0, 0]
    return sk, same


def test_survey_sample_groups_are_its_families(survey_sample):
    sk, _ = survey_sample
    for min_same in (1, 700):
        label, n_groups, n_links = cluster_oracle.cluster(sk, min_same)
        assert list(label) == [0, 0, 0, 0, 4, 4, 4, 4] and n_groups == 2
    assert cluster_oracle.cluster(sk, 1)[2] == 12  # 2 families x C(4, 2) pairs, none across


def test_threshold_sweep_matches_brute_force(survey_sample):
    sk, same = survey_sample
    cut_but_joined = 0
    for min_same in range(700, 801):
        want = brute_labels(same, min_same)
        label, n_groups, n_links, links = cluster_oracle.cluster(sk, min_same, want_links=True)
        assert (list(label), n_groups, n_links) == (list(want[0]), want[1], want[2]), min_same
        assert [tuple(p) for p in links] == [(i, j) for i in range(8) for j in range(i + 1, 8) if same[i, j] >= min_same]
        # single linkage: members whose direct link is cut stay together through a third member
        cut_but_joined += any(same[i, j] < min_same and label[i] == label[j] for i in range(8) for j in range(i + 1, 8))
        for threads in (1, 3):
            assert np.array_equal(cluster_oracle.cluster(sk, min_same, nthreads=threads)[0], label)
    assert cut_but_joined > 0


def test_pair_list_form_agrees(survey_sample):
    sk, same = survey_sample
    i, j = np.nonzero(np.triu(same, 1))
    for min_same in (1, 700, 760, 800, 2000):
        want = cluster_oracle.cluster(sk, min_same)
        got = cluster_oracle.cluster_pairs(i, j, same[i, j], 8, min_same)
        assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
    # order and direction of the triples do not matter; the diagonal is ignored
    perm = np.random.default_rng(1).permutation(len(i))
    got = cluster_oracle.cluster_pairs(np.r_[j[perm], 3], np.r_[i[perm], 3], np.r_[same[i, j][perm], 2000], 8, 700)
    assert list(got[0]) == [0, 0, 0, 0, 4, 4, 4, 4] and got[2] == int((same[i, j] >= 700).sum()) == 11


def test_chain_is_one_group():
    """0-1 and 1-2 share two hashes each, 0-2 share none: single linkage still joins all three; 3 stands alone."""
    sk = np.array([[10, 20, 30, 40], [10, 20, 50, 60], [5, 50, 60, 70], [1, 2, 3, 4]], np.uint32)
    rc, same = oracle_ffi.similarity_block(sk, 0, 4, 0, 4)
    assert rc == 0 and (same[0, 1], same[1, 2], same[0, 2]) == (2, 2, 0)
    label, n_groups, n_links = cluster_oracle.cluster(sk, 2)
    assert (list(label), n_groups, n_links) == ([0, 0, 0, 3], 2, 2)
    assert list(cluster_oracle.cluster(sk, 3)[0]) == [0, 1, 2, 3]
    # the smallest index labels the group wherever it sits in the chain
    label, _, _ = cluster_oracle.cluster(sk[[2, 1, 3, 0]], 2)
    assert list(label) == [0, 0, 2, 0]


def test_empty_set():
    label, n_groups, n_links = cluster_oracle.cluster(np.zeros((0, 4), np.uint32), 1)
    assert (len(label), n_groups, n_links) == (0, 0, 0)


def test_distance_threshold_on_a_count_includes_it():
    """A max_distance that is exactly 1 - c/s for some count c admits c; the next double below it does not."""
    s = 400
    a = np.arange(1, s + 1, dtype=np.uint32) * 2
    for c in (1, 123, 399, 400):
        b = a.copy()
        b[c:] += 1  # exactly c common values, both still ascending
        sk = np.stack([a, b])
        assert oracle_ffi.similarity_block(sk, 0, 1, 1, 2)[1][0, 0] == c
        d = 1.0 - np.float64(c) / np.float64(s)
        m = mash.min_same_for_distance(d, s)
        assert m == c and list(cluster_oracle.cluster(sk, m)[0]) == [0, 0]
        m = mash.min_same_for_distance(np.nextafter(d, -1.0), s)
        assert m == c + 1
        if m <= s:
            assert list(cluster_oracle.cluster(sk, m)[0]) == [0, 1]


def test_mirror_thresholds_that_need_no_launch():
    sk = np.arange(12, dtype=np.uint32).reshape(3, 4)
    with pytest.raises(ValueError):
        mash.cluster(sk)
    with pytest.raises(ValueError):
        mash.cluster(sk, min_same=1, max_distance=0.5)
    with pytest.raises(ValueError, match="every pair"):
        mash.cluster(sk, max_distance=1.0)
    # no count reaches a negative distance: the identity labelling, without touching the library
    label, n_groups, n_links = mash.cluster(sk, max_distance=-0.25)
    assert list(label) == [0, 1, 2] and label.dtype == np.uint32 and (n_groups, n_links) == (3, 0)
