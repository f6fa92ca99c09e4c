"""Growing a clustering on the GPU (pg_mash_clusterer_*): after every add, the labels of everything added so far
against mash.cluster of that prefix and against the cluster oracle, the batch's labels against their slice, and
the counts (groups, links summed over the adds, earlier groups absorbed) against the oracle; the borrowed index
against a SketchIndex built over every sketch."""
import ctypes as C
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

import cluster_add_oracle
import cluster_oracle
import oracle_ffi
from poly_b200 import _lib, mash, sketchfile, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def sketches_of(reads, n, L, k, s):
    rc, sk = oracle_ffi.sketch_batch(reads, synth.uniform_offsets(n, L), k, s, variant=1, nthreads=len(os.sched_getaffinity(0)))
    assert rc == 0
    return sk


@pytest.fixture(scope="module")
def family(gpu):
    """2 048 family reads of 2 kbp, 16 per family, k = 21, s = 400: members share 137..273 hashes."""
    n, L, k, s = 2048, 2000, 21, 400
    return sketches_of(synth.family_reads(n, L, family=16), n, L, k, s)


def chain(n):
    """n sketches of s = 16: sketch i holds 8 i .. 8 i + 15, so neighbours share 8 values and nothing else links."""
    return (np.arange(n, dtype=np.uint32)[:, None] * 8 + np.arange(16, dtype=np.uint32)).astype(np.uint32)


class Prefixes:
    """The oracle's answer for every prefix of one set, from its links listed once."""

    def __init__(self, sk, min_same):
        self.i, self.j, _ = cluster_oracle.links_of(sk, min_same)

    def at(self, end):
        """(labels, n_groups, n_links) of sketches [0, end)"""
        keep = self.j < end
        label, n_groups = cluster_oracle.labels_of(end, self.i[keep], self.j[keep])
        return label, n_groups, int(keep.sum())


def grow(sk, cuts, min_same):
    """Adds the batches between the cut points and checks every add; returns the final labels."""
    want = Prefixes(sk, min_same)
    edges = [0, *cuts, len(sk)]
    prev = np.zeros(0, np.uint32)
    with mash.Clusterer(sk.shape[1], min_same=min_same) as c:
        for a, b in zip(edges[:-1], edges[1:]):
            labels, n_groups, n_links, n_merged = c.add(sk[a:b])
            assert labels.dtype == np.uint32 and len(labels) == b - a and c.n == b
            w_label, w_groups, w_links = want.at(b)
            got = c.labels()
            assert np.array_equal(got, w_label) and n_groups == w_groups == c.n_groups, (min_same, cuts, b)
            assert np.array_equal(labels, w_label[a:b])
            assert c.n_links == w_links, (min_same, cuts, b)
            roots = np.nonzero(prev == np.arange(a))[0]
            assert n_merged == int((w_label[roots] != roots).sum()), (min_same, cuts, b)
            whole = mash.cluster(sk[:b], min_same=min_same)
            assert np.array_equal(whole[0], got) and whole[1:] == (w_groups, w_links)
            prev = got
    return prev


def random_splits(rng, n, count):
    return [sorted(int(c) for c in rng.integers(0, n + 1, size=int(rng.integers(0, 7)))) for _ in range(count)]


def test_family_reads_in_random_batches(family):
    rng = np.random.default_rng(13)
    for min_same in (1, 100, 200, 400):
        for cuts in random_splits(rng, len(family), 3):
            grow(family, cuts, min_same)


def test_single_row_adds(family):
    grow(family[:64], list(range(1, 64)), 150)
    grow(chain(40), list(range(1, 40)), 8)


def test_query_in_several_row_blocks(family, monkeypatch):
    """The batch's query against the earlier sketches runs in blocks of 7 and 1 rows."""
    for rows in ("7", "1"):
        monkeypatch.setenv("PG_INDEX_QUERY_ROWS", rows)
        grow(family[:600], [100, 350], 150)


def test_batch_pass_in_several_row_tiles(gpu):
    """49 152 sketches: the second batch's own pass runs in several row tiles, and its cross query (24 569 x 24 583
    counts) in two 2 GiB row blocks; families and chain links straddle every cut."""
    n = 49152
    sk = chain(n)
    rows_per = ((2 << 30) // (n - 101)) & ~7  # distance_tile_rows of the second batch
    assert rows_per < n - 101
    with mash.Clusterer(16, min_same=8) as c:
        assert c.add(sk[:101])[1:] == (1, 100, 0)
        labels, n_groups, n_links, n_merged = c.add(sk[101:])
        assert (labels == 0).all() and (n_groups, n_links, n_merged) == (1, n - 101, 0) and (c.labels() == 0).all()
    fam = sketches_of(synth.family_reads(n, 80, family=16), n, 80, 21, 16)
    grow(fam, [24583], 4)


def test_late_bridges_merge_many_groups(gpu):
    """Chained windows fed evens first: the later batches bridge the earlier groups, and each add's n_merged
    reports how many were absorbed."""
    n = 4000
    ck = chain(n)
    order = np.r_[np.arange(0, n, 2), np.arange(1, n, 4), np.arange(3, n, 4)]
    sk = ck[order]
    labels = grow(sk, [n // 2, 3 * n // 4], 8)
    assert (labels == 0).all()
    with mash.Clusterer(16, min_same=8) as c:
        assert c.add(sk[: n // 2])[1:] == (n // 2, 0, 0)
        _, n_groups, n_links, n_merged = c.add(sk[n // 2: 3 * n // 4])  # each odd row 4 t + 1 joins evens 4 t and 4 t + 2
        assert (n_groups, n_links, n_merged) == (n // 4, n // 2, n // 4)
        _, n_groups, n_links, n_merged = c.add(sk[3 * n // 4:])
        assert (n_groups, n_links, n_merged) == (1, n // 2 - 1, n // 4 - 1)


def test_identical_sketches_across_batches(family):
    sk = family[:512].copy()
    sk[[7, 100, 511]] = sk[3]
    sk[300] = sk[20]
    for cuts in ([5], [50, 200, 400], [301]):
        grow(sk, cuts, 400)
    grow(sk, [4, 8], 150)


def test_unsorted_batches(family):
    """150 bp reads under s = 400 are in the fill regime (unsorted, zero tails): alone every one is its own group,
    and after ascending sketches they drop the index's join while the labels stay exact."""
    n, L, k, s = 512, 150, 21, 400
    short = sketches_of(synth.independent_reads(n, L), n, L, k, s)
    assert (grow(short, [100, 300], 1) == np.arange(n)).all()
    mixed = np.concatenate([family[:256], short[:128], family[256:512]])
    for cuts in ([256, 384], [100, 300, 400]):
        grow(mixed, cuts, 150)


def test_unsorted_batch_whose_tile_does_not_fit(gpu):
    """6000-word sketches: an unsorted batch needs the pairwise tile for its query, which does not fit.  The add
    fails with PG_ERR_UNSUPPORTED and the clusterer is unchanged; the next ascending batch is exact."""
    rng = np.random.default_rng(3)
    refs = np.sort(rng.integers(0, 1 << 32, size=(40, 6000), dtype=np.uint32), axis=1)
    refs[[5, 17]] = refs[2]
    refs[33] = refs[30]
    unsorted = rng.integers(0, 1 << 32, size=(2, 6000), dtype=np.uint32)
    with mash.Clusterer(6000, min_same=3000) as c:
        c.add(refs[:30])
        before = c.labels()
        with pytest.raises(_lib.PolyError) as e:
            c.add(unsorted)
        assert e.value.code == _lib.PG_ERR_UNSUPPORTED
        assert c.n == 30 and np.array_equal(c.labels(), before) and c.index.nearest(refs[:1], 1)[0][0, 0] == 0
        labels, n_groups, n_links, n_merged = c.add(refs[30:])
        want = cluster_oracle.cluster(refs, 3000)
        assert np.array_equal(c.labels(), want[0]) and (n_groups, c.n_links) == want[1:]
        assert list(labels) == list(want[0][30:]) and n_merged == 0


def test_empty_batches(family):
    sk = family[:300]
    grow(sk, [0, 0, 150, 150, 300], 150)
    L = _lib.lib()
    with mash.Clusterer(400, min_same=150) as c:
        first, ng, nl, nm = (C.c_uint64(9) for _ in range(4))
        assert L.pg_mash_clusterer_add(c._h, None, 0, 400, None, C.byref(first), C.byref(ng), C.byref(nl), C.byref(nm)) == _lib.PG_OK
        assert (first.value, ng.value, nl.value, nm.value) == (0, 0, 0, 0)
        _, n_groups, _, _ = c.add(sk[:10])
        assert L.pg_mash_clusterer_add(c._h, None, 0, -1, None, C.byref(first), C.byref(ng), C.byref(nl), C.byref(nm)) == _lib.PG_OK
        assert (first.value, ng.value, nl.value, nm.value) == (10, n_groups, 0, 0)
        assert L.pg_mash_clusterer_add_dev(c._h, None, 0, 7, None, C.byref(first), None, None, None, None) == _lib.PG_OK and first.value == 10
        labels, g2, l2, m2 = c.add(np.zeros((0, 400), np.uint32))
        assert len(labels) == 0 and (g2, l2, m2) == (n_groups, 0, 0)


def test_device_path_equals_host_path(family):
    import torch

    st = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    want = mash.cluster(family, min_same=150)
    host = []
    with mash.Clusterer(400, min_same=150) as c:
        for a, b in ((0, 700), (700, 1500), (1500, 2048)):
            host.append(c.add(family[a:b]))
    with mash.Clusterer(400, min_same=150) as c:
        for (a, b), h in zip(((0, 700), (700, 1500), (1500, 2048)), host):
            t = torch.from_numpy(family[a:b].view(np.int32)).cuda()
            labels, *counts = c.add(t)
            assert labels.is_cuda and labels.dtype == torch.int32 and all(isinstance(x, int) for x in counts)
            assert np.array_equal(labels.cpu().numpy().view(np.uint32), h[0]) and tuple(counts) == h[1:]
        assert np.array_equal(c.labels(), want[0]) and (c.n_groups, c.n_links) == want[1:]
        # labels_dev against labels, over slices
        for a, b in ((0, 2048), (100, 101), (1500, 2048), (7, 7)):
            out = torch.full((max(b - a, 1),), -5, dtype=torch.int32, device="cuda")
            _lib.check(L.pg_mash_clusterer_labels_dev(c._h, a, b, out.data_ptr(), st))
            torch.cuda.synchronize()
            assert np.array_equal(out.cpu().numpy().view(np.uint32)[: b - a], c.labels(a, b))
    # the label output and the counts are optional
    with mash.Clusterer(400, min_same=150) as c:
        d_sk = torch.from_numpy(family.view(np.int32)).cuda()
        out = torch.empty(len(family), dtype=torch.int32, device="cuda")
        _lib.check(L.pg_mash_clusterer_add_dev(c._h, d_sk.data_ptr(), 1000, 400, out.data_ptr(), None, None, None, None, st))
        _lib.check(L.pg_mash_clusterer_add_dev(c._h, d_sk[1000:].data_ptr(), 1048, 400, None, None, None, None, None, st))
        _lib.check(L.pg_mash_clusterer_add(c._h, family.ctypes.data, 0, 400, None, None, None, None, None))
        assert np.array_equal(c.labels(0, 2048), want[0])  # c.n counts only the adds made through the wrapper


def test_argument_errors_leave_the_clusterer_unchanged(family):
    L = _lib.lib()
    sk = family[:600]
    want = mash.cluster(sk, min_same=150)
    label = np.zeros(600, np.uint32)
    first, ng, nl, nm = (C.c_uint64(0) for _ in range(4))
    with mash.Clusterer(400, min_same=150) as c:
        c.add(sk[:200])
        h, before = c._h, c.labels()
        # in order: s <= 0, an s other than the clusterer's, the id limit, a null buffer
        assert L.pg_mash_clusterer_add(h, None, 1 << 33, 0, None, None, None, None, None) == _lib.PG_ERR_PANIC
        assert L.pg_mash_clusterer_add(h, None, 1 << 33, 16, None, None, None, None, None) == _lib.PG_ERR_ARG and "size" in _lib.last_error()
        assert L.pg_mash_clusterer_add(h, None, (1 << 32) - 200, 400, None, None, None, None, None) == _lib.PG_ERR_ARG \
            and "2^32" in _lib.last_error()
        assert L.pg_mash_clusterer_add(h, None, 10, 400, label.ctypes.data, None, None, None, None) == _lib.PG_ERR_ARG \
            and "null" in _lib.last_error()
        assert L.pg_mash_clusterer_add_dev(h, None, 10, -1, None, None, None, None, None, None) == _lib.PG_ERR_PANIC
        assert L.pg_mash_clusterer_add_dev(h, None, 10, 400, None, None, None, None, None, None) == _lib.PG_ERR_ARG
        with pytest.raises(_lib.PolyError):
            c.add(np.zeros((3, 16), np.uint32))
        with pytest.raises(_lib.GoPanic):
            c.add(np.zeros((3, 0), np.uint32))
        # labels: begin > end, end > n, a null buffer with end > begin
        assert L.pg_mash_clusterer_labels(h, 5, 4, label.ctypes.data) == _lib.PG_ERR_ARG
        assert L.pg_mash_clusterer_labels(h, 0, 201, label.ctypes.data) == _lib.PG_ERR_ARG
        assert L.pg_mash_clusterer_labels(h, 0, 10, None) == _lib.PG_ERR_ARG
        assert L.pg_mash_clusterer_labels(h, 200, 200, None) == _lib.PG_OK
        assert L.pg_mash_clusterer_labels_dev(h, 0, 201, None, None) == _lib.PG_ERR_ARG
        assert c.n == 200 and np.array_equal(c.labels(), before) and c.index.n == 200
        assert L.pg_mash_clusterer_add(h, sk[200:].ctypes.data, 400, 400, label.ctypes.data, C.byref(first), C.byref(ng), C.byref(nl),
                                       C.byref(nm)) == _lib.PG_OK
        assert first.value == 200 and np.array_equal(label[:400], want[0][200:]) and ng.value == want[1]
        assert np.array_equal(c.labels(0, 600), want[0])  # c.n counts only the adds made through the wrapper


def test_borrowed_index_answers_as_a_sketch_index(family):
    import torch

    sk, queries = family[:1500], family[1500:1700]
    with mash.Clusterer(400, min_same=200) as c:
        for a, b in ((0, 400), (400, 1100), (1100, 1500)):
            c.add(sk[a:b])
        with pytest.raises(ValueError, match="Clusterer.add"):
            c.index.add(queries)
        with mash.SketchIndex(sk) as ix:
            for k in (1, 10):
                got, want = c.index.nearest(queries, k), ix.nearest(queries, k)
                assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want))
            got, want = c.index.within(queries, min_same=150), ix.within(queries, min_same=150)
            assert all(g.tobytes() == w.tobytes() for g, w in zip(got, want))
            dq = torch.from_numpy(queries.view(np.int32)).cuda()
            got = c.index.nearest(dq, 10, max_distance=0.6)
            want = ix.nearest(queries, 10, max_distance=0.6)
            assert np.array_equal(got[0].cpu().numpy().view(np.uint32), want[0])
        # "which group would this sketch join": the top hit's label, as the clustering of the grown set says
        ref = c.index.nearest(queries, 1, min_same=200)[0][:, 0]
        hit = ref != mash.NO_REF
        grown = mash.cluster(np.concatenate([sk, queries]), min_same=200)[0]
        assert hit.any() and (grown[1500:][hit] == grown[c.labels()[ref[hit]]]).all()
        labels, *_ = c.add(family[1700:])  # after device queries: the add waits for them
        assert np.array_equal(labels, mash.cluster(np.concatenate([sk, family[1700:]]), min_same=200)[0][1500:])


def test_two_threads_add_to_one_clusterer(family):
    """Each call's first is the number of sketches added before it; the final labels equal mash.cluster of the
    batches in the order their first values give."""
    L = _lib.lib()
    batches = [family[i * 128:(i + 1) * 128] for i in range(16)]
    with mash.Clusterer(400, min_same=150) as c:
        done = []  # (first, batch index, n_links)
        lock = threading.Lock()

        def worker(idx):
            for i in idx:
                label, first, nl = np.zeros(128, np.uint32), C.c_uint64(0), C.c_uint64(0)
                _lib.check(L.pg_mash_clusterer_add(c._h, batches[i].ctypes.data, 128, 400, label.ctypes.data, C.byref(first), None,
                                                   C.byref(nl), None))
                with lock:
                    done.append((first.value, i, nl.value))

        th = [threading.Thread(target=worker, args=(range(t, 16, 2),)) for t in range(2)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        done.sort()
        assert [f for f, _, _ in done] == [128 * j for j in range(16)]
        order = np.concatenate([batches[i] for _, i, _ in done])
        want = mash.cluster(order, min_same=150)
        got = np.zeros(2048, np.uint32)
        _lib.check(L.pg_mash_clusterer_labels(c._h, 0, 2048, got.ctypes.data))
        assert np.array_equal(got, want[0]) and sum(x for _, _, x in done) == want[2]


def test_oracle_restatement_agrees_on_the_device(family):
    sk = family[:400]
    want = cluster_add_oracle.cluster_in_batches(sk, [90, 250], 150)
    with mash.Clusterer(400, min_same=150) as c:
        for (a, b), (label, batch, n_groups, n_links, n_merged) in zip(((0, 90), (90, 250), (250, 400)), want):
            got = c.add(sk[a:b])
            assert np.array_equal(got[0], batch) and got[1:] == (n_groups, n_links, n_merged)
            assert np.array_equal(c.labels(), label)


def test_cpp_mirror_agrees_with_the_oracle(family):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "cluster_add_tests"])
    sk = family[:512]
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "set.pgsketch")
        sketchfile.save(path, sk, np.full(len(sk), 400, np.uint32), 21, 400)
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "cluster_add_tests"), path, "200", "3"], capture_output=True, text=True,
                             timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: cluster add tests pass"
    label, n_groups, n_links = cluster_oracle.cluster(sk, 200)
    assert lines[0] == f"{n_groups} {n_links}" and lines[1] == " ".join(str(int(x)) for x in label)
