"""CPU tier: a growing clustering, restated batch by batch (tests/cluster_add_oracle.py: the prefix's groups, the
batch's links to every earlier sketch and the links inside the batch, united), equals the cluster oracle of the
prefix after every add, for any split.  This is the decomposition pg_mash_clusterer_add relies on."""
import numpy as np
import pytest

import cluster_add_oracle
import cluster_oracle
import oracle_ffi
from poly_b200 import mash, synth


def counts(sk):
    rc, same = oracle_ffi.similarity_block(sk, 0, len(sk), 0, len(sk))
    assert rc == 0
    return same


@pytest.fixture(scope="module")
def survey_sample():
    """The 16-read, R = 4 family sample of SURVEY 8d (10 kbp, k = 31, s = 2000)."""
    n, L, k, s = 16, 10000, 31, 2000
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


def check_every_add(sk, cuts, min_same):
    """After each add: all labels against the oracle of the prefix, the batch labels as its slice; the link counts
    summed over the adds against the whole set's."""
    edges = [0, *cuts, len(sk)]
    links = 0
    for (label, batch, n_groups, n_links, _), end, start in zip(cluster_add_oracle.cluster_in_batches(sk, cuts, min_same), edges[1:], edges[:-1]):
        want = cluster_oracle.cluster(sk[:end], min_same)
        assert np.array_equal(label, want[0]) and n_groups == want[1], (min_same, cuts, end)
        assert np.array_equal(batch, want[0][start:end])
        links += n_links
        assert links == want[2], (min_same, cuts, end)


def test_random_splits_equal_the_prefix(survey_sample, families):
    rng = np.random.default_rng(5)
    for sk in (survey_sample, families):
        n, s = sk.shape
        same = counts(sk)
        off = sorted({int(c) for c in np.triu(same, 1).ravel()} - {0} | {1, s})
        for c in off[:: max(1, len(off) // 10)] + off[-2:]:
            d = 1.0 - np.float64(c) / np.float64(s)  # exactly on the Distance of the pairs that count c
            assert mash.min_same_for_distance(d, s) == c
            splits = [[], list(range(1, n)), [0, 0, n, n]] + [random_cuts(rng, n, k) for k in (1, 2, 3, 6)]
            for cuts in splits:
                check_every_add(sk, cuts, c)


def hand_sets(n_a, n_b):
    """Sketches 0 (the even values 2..40) and 1 (the odd values 1..39) share nothing; sketch 2 takes n_a of 0's
    values and n_b of 1's, and is padded above both with its own."""
    s = 20
    a, b = np.arange(2, 41, 2, dtype=np.uint32), np.arange(1, 40, 2, dtype=np.uint32)
    c = np.sort(np.r_[a[:n_a], b[:n_b], 100 + np.arange(s - n_a - n_b, dtype=np.uint32)])
    return np.stack([a, b, c])


def test_a_batch_row_bridges_two_earlier_groups():
    """Row 2 links both 0 and 1: the earlier group of 1 is absorbed and its label retired."""
    sk = hand_sets(9, 9)
    same = counts(sk)
    assert (same[0, 1], same[2, 0], same[2, 1]) == (0, 9, 9)
    g = cluster_add_oracle.GrowingClustering(20, 5)
    labels, n_groups, n_links, n_merged = g.add(sk[:2])
    assert list(labels) == [0, 1] and (n_groups, n_links, n_merged) == (2, 0, 0)
    labels, n_groups, n_links, n_merged = g.add(sk[2:])
    assert list(labels) == [0] and list(g.label) == [0, 0, 0] and (n_groups, n_links, n_merged) == (1, 2, 1)
    # a row linked to one earlier group only absorbs nothing
    g = cluster_add_oracle.GrowingClustering(20, 5)
    g.add(hand_sets(9, 2)[:2])
    assert g.add(hand_sets(9, 2)[2:])[1:] == (2, 1, 0)


def chain(n):
    """n sketches of s = 16: sketch i holds 8 i .. 8 i + 15, so neighbours share 8 values and nothing else links."""
    return (np.arange(n, dtype=np.uint32)[:, None] * 8 + np.arange(16, dtype=np.uint32)).astype(np.uint32)


def test_bridging_sketches_arriving_last_merge_many_groups():
    """The even links of a chain first (each its own group), then every odd one in one batch: that add joins them
    all, and every earlier group but the first is absorbed."""
    n = 40
    ck = chain(n)
    order = np.r_[np.arange(0, n, 2), np.arange(1, n, 2)]
    sk = ck[order]
    g = cluster_add_oracle.GrowingClustering(16, 8)
    labels, n_groups, n_links, n_merged = g.add(sk[: n // 2])
    assert list(labels) == list(range(n // 2)) and (n_groups, n_links, n_merged) == (n // 2, 0, 0)
    labels, n_groups, n_links, n_merged = g.add(sk[n // 2:])
    assert (labels == 0).all() and (g.label == 0).all()
    assert (n_groups, n_links, n_merged) == (1, n - 1, n // 2 - 1)
    want = cluster_oracle.cluster(sk, 8)
    assert np.array_equal(g.label, want[0]) and (want[1], want[2]) == (1, n - 1)


def test_empty_batches():
    g = cluster_add_oracle.GrowingClustering(16, 1)
    assert g.add(np.zeros((0, 16), np.uint32))[1:] == (0, 0, 0) and g.n == 0
    g.add(chain(3))
    assert g.add(np.zeros((0, 16), np.uint32))[1:] == (1, 0, 0) and g.n == 3
