"""pg_mash_cluster on the GPU against the cluster oracle: labels element for element, and both counts."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import cluster_oracle
import oracle_ffi
from poly_b200 import _lib, mash, sketchfile, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def sketches_of(reads, n, L, k, s):
    rc, sk = oracle_ffi.sketch_batch(reads, synth.uniform_offsets(n, L), k, s, variant=1, nthreads=len(os.sched_getaffinity(0)))
    assert rc == 0
    return sk


def check_against_oracle(sk, min_same):
    want = cluster_oracle.cluster(sk, min_same)
    label, n_groups, n_links = mash.cluster(sk, min_same=min_same)
    assert label.dtype == np.uint32 and np.array_equal(label, want[0])
    assert (n_groups, n_links) == want[1:]
    return label, n_groups, n_links


@pytest.fixture(scope="module")
def family(gpu):
    """2 048 family reads of 2 kbp, 16 per family, k = 21, s = 400: members share 137..273 hashes."""
    n, L, k, s = 2048, 2000, 21, 400
    return sketches_of(synth.family_reads(n, L, family=16), n, L, k, s)


def test_families_whole_split_and_chance_links(family):
    n = len(family)
    fam = (np.arange(n) // 16 * 16).astype(np.uint32)
    label, n_groups, n_links = check_against_oracle(family, 100)  # below every in-family count
    assert np.array_equal(label, fam) and n_groups == n // 16
    label, n_groups, _ = check_against_oracle(family, 200)  # cuts about half of the direct links: families split
    assert n // 16 < n_groups < n and (label // 16 == fam // 16).all()
    label, n_groups, _ = check_against_oracle(family, 1)  # single 32-bit hashes shared by chance join whole families
    assert n_groups < n // 16


def test_only_identical_sketches_link_at_the_sketch_size(family):
    sk = family[:512].copy()
    sk[[7, 100, 511]] = sk[3]
    sk[300] = sk[20]
    label, n_groups, n_links = check_against_oracle(sk, sk.shape[1])
    want = np.arange(512, dtype=np.uint32)
    want[[7, 100, 511]] = 3
    want[300] = 20
    assert np.array_equal(label, want) and (n_groups, n_links) == (508, 6 + 1)


def test_link_count_is_the_filtered_sparse_pair_count(family):
    _, _, ps = mash.distance_sparse(family, upper=True)
    for min_same in (1, 150, 200):
        assert mash.cluster(family, min_same=min_same)[2] == int((ps >= min_same).sum())


def test_max_distance_is_the_count_cut(family):
    d = 1.0 - 200.0 / 400.0
    assert mash.min_same_for_distance(d, 400) == 200
    got, want = mash.cluster(family, max_distance=d), mash.cluster(family, min_same=200)
    assert np.array_equal(got[0], want[0]) and got[1:] == want[1:]
    assert got[1] < mash.cluster(family, max_distance=float(np.nextafter(d, -1.0)))[1]  # count 200 no longer links
    as_mashes = []
    for row in family[:64]:
        m = mash.New(21, 400)
        m.Sketches[:] = row
        as_mashes.append(m)
    assert np.array_equal(mash.cluster(as_mashes, max_distance=d)[0], cluster_oracle.cluster(family[:64], 200)[0])


def test_unsorted_regime_links_by_the_literal_walk(gpu):
    """150 bp reads, k = 21, s = 1000: 129 positional hashes and a zero tail, so Similarity's range check
    (Sketches[s-1] = 0 below the other's first hash) counts 0 for every pair: every read is its own group."""
    n, L, k, s = 512, 150, 21, 1000
    sk = sketches_of(synth.independent_reads(n, L), n, L, k, s)
    label, n_groups, n_links = check_against_oracle(sk, 1)
    assert np.array_equal(label, np.arange(n)) and (n_groups, n_links) == (n, 0)
    # an unsorted pair with the same four values: the walk counts 2, a set intersection would count 4
    pair = np.array([[3, 1, 2, 9], [1, 2, 3, 9]], np.uint32)
    rc, same = oracle_ffi.similarity_block(pair, 0, 2, 0, 2)
    assert rc == 0 and same[0, 1] == same[1, 0] == 2
    for sk2 in (pair, pair[::-1].copy()):
        assert list(check_against_oracle(sk2, 2)[0]) == [0, 0]
        assert list(check_against_oracle(sk2, 3)[0]) == [0, 1]


def test_shuffled_input_gives_the_same_partition(family):
    perm = np.random.default_rng(7).permutation(len(family))
    for min_same in (100, 200):
        base = mash.cluster(family, min_same=min_same)
        label, n_groups, n_links = check_against_oracle(family[perm], min_same)
        assert (n_groups, n_links) == base[1:]

        def partition(lab, ids):
            groups = {}
            for pos, l in enumerate(lab):
                groups.setdefault(int(l), set()).add(int(ids[pos]))
            return {frozenset(g) for g in groups.values()}

        assert partition(label, perm) == partition(base[0], np.arange(len(family)))
        # labels are still the smallest position of each group
        assert (label <= np.arange(len(label))).all() and np.array_equal(label[label], label)
        for rep in np.unique(label):
            assert rep == np.nonzero(label == rep)[0][0]


def test_row_length_not_a_multiple_of_four(family):
    for n in (2045, 2046, 2047, 5, 1):
        check_against_oracle(family[:n], 150)


def test_more_than_one_row_tile(gpu):
    """49 152 sketches: the dense pass runs in two row tiles, and families that straddle the cut are joined
    by links whose row is in the first tile and whose column is a row of the second."""
    n, L, k, s, min_same = 49152, 80, 21, 16, 4
    rows_per = ((2 << 30) // n) & ~7  # distance_tile_rows
    assert 0 < rows_per < n
    sk = sketches_of(synth.family_reads(n, L, family=16), n, L, k, s)
    want_label, want_groups, want_links, links = cluster_oracle.cluster(sk, min_same, want_links=True)
    across = links[(links[:, 0] < rows_per) & (links[:, 1] >= rows_per)]
    assert len(across) > 0 and rows_per % 16 != 0
    label, n_groups, n_links = mash.cluster(sk, min_same=min_same)
    assert np.array_equal(label, want_label) and (n_groups, n_links) == (want_groups, want_links)
    assert (label[across[:, 0]] == label[across[:, 1]]).all()


def test_device_path_equals_host_path(family):
    import torch

    d_sk = torch.from_numpy(family.view(np.int32)).cuda()
    for min_same in (100, 200, 400):
        want = mash.cluster(family, min_same=min_same)
        label, n_groups, n_links = mash.cluster(d_sk, min_same=min_same)
        assert label.is_cuda and label.dtype == torch.int32
        assert np.array_equal(label.cpu().numpy().view(np.uint32), want[0]) and (int(n_groups), int(n_links)) == want[1:]
    # the counts are optional
    label = torch.empty(len(family), dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().pg_mash_cluster_dev(d_sk.data_ptr(), len(family), 400, 100, label.data_ptr(), None, None,
                                              torch.cuda.current_stream().cuda_stream))
    assert np.array_equal(label.cpu().numpy().view(np.uint32), mash.cluster(family, min_same=100)[0])
    label, n_groups, n_links = mash.cluster(d_sk, max_distance=-1.0)  # nothing can link: no launch
    assert label.is_cuda and label.cpu().tolist() == list(range(len(family))) and (int(n_groups), int(n_links)) == (len(family), 0)


def test_empty_set_and_argument_errors(family):
    label, n_groups, n_links = mash.cluster(np.zeros((0, 400), np.uint32), min_same=1)
    assert (len(label), n_groups, n_links) == (0, 0, 0)
    sk = family[:32]
    lab = np.zeros(32, np.uint32)
    ng, nl = C.c_uint64(9), C.c_uint64(9)
    for bad in (0, 401):
        assert _lib.lib().pg_mash_cluster(sk.ctypes.data, 32, 400, bad, lab.ctypes.data, C.byref(ng), C.byref(nl)) == _lib.PG_ERR_ARG
        assert "min_same" in _lib.last_error() and (ng.value, nl.value) == (0, 0)
        with pytest.raises(_lib.PolyError) as e:
            mash.cluster(sk, min_same=bad)
        assert e.value.code == _lib.PG_ERR_ARG
    assert _lib.lib().pg_mash_cluster(sk.ctypes.data, 32, 0, 1, lab.ctypes.data, None, None) == _lib.PG_ERR_PANIC
    with pytest.raises(_lib.GoPanic):
        mash.cluster(np.zeros((3, 0), np.uint32), min_same=1)
    with pytest.raises(_lib.GoPanic):
        mash.cluster(np.zeros((3, 0), np.uint32), max_distance=0.5)
    assert _lib.lib().pg_mash_cluster(None, 1 << 32, 400, 1, None, None, None) == _lib.PG_ERR_ARG


def test_cpp_mirror_agrees_with_python(family):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "cluster_tests"])
    sk = family[:512]
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "set.pgsketch")
        sketchfile.save(path, sk, np.full(len(sk), 400, np.uint32), 21, 400)
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "cluster_tests"), path, "200"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: cluster tests pass"
    label, n_groups, n_links = cluster_oracle.cluster(sk, 200)
    assert lines[0] == f"{n_groups} {n_links}" and lines[1] == " ".join(str(int(x)) for x in label)
