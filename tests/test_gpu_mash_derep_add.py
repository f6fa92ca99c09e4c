"""Growing a dereplication on the GPU (pg_mash_dereplicator_*): the concatenated adds against mash.dereplicate
of the whole set and against the dereplication oracle, in both modes, and the representative index against a
SketchIndex built over the representatives."""
import ctypes as C
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

import derep_add_oracle
import derep_oracle
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


def grow(sk, cuts, min_same, nearest):
    """(rep, n_reps, representatives) of the sketches added as the batches between the cut points."""
    edges = [0, *cuts, len(sk)]
    with mash.Dereplicator(sk.shape[1], min_same=min_same, nearest=nearest) as d:
        parts, total = [], 0
        for a, b in zip(edges[:-1], edges[1:]):
            rep, n_new = d.add(sk[a:b])
            assert rep.dtype == np.uint32 and len(rep) == b - a and d.n == b
            parts.append(rep)
            total += n_new
        reps = d.representatives()
    return np.concatenate(parts), total, reps


def check_splits(sk, splits, min_same, modes=(False, True)):
    """Every split against the one-shot call and the oracle, in both modes."""
    links = derep_oracle.links_of(sk, min_same)
    for nearest in modes:
        want = derep_oracle.dereplicate_pairs(*links, len(sk), min_same, nearest)
        whole = mash.dereplicate(sk, min_same=min_same, nearest=nearest)
        assert np.array_equal(whole[0], want[0]) and whole[1] == want[1]
        for cuts in splits:
            rep, n_reps, reps = grow(sk, cuts, min_same, nearest)
            assert np.array_equal(rep, want[0]) and n_reps == want[1], (min_same, nearest, cuts)
            assert np.array_equal(reps, np.nonzero(rep == np.arange(len(sk)))[0])


def random_splits(rng, n, count):
    return [sorted(int(c) for c in rng.integers(0, n + 1, size=int(rng.integers(0, 7)))) for _ in range(count)]


def test_family_reads_in_random_batches(family):
    rng = np.random.default_rng(11)
    for min_same in (1, 100, 200, 400):
        check_splits(family, random_splits(rng, len(family), 4), min_same)


def test_single_row_adds(family):
    sk = family[:64]
    check_splits(sk, [list(range(1, 64))], 150)


def test_batches_straddle_a_sub_block(family):
    check_splits(family, [[1000], [1023, 1025], [5, 1030, 2040]], 150)


def test_chain_batch_in_two_row_tiles(gpu):
    """49 152 chained sketches (s = 16, neighbours share 8 values): the second batch's own pass runs in several row
    tiles, and the first cut sits inside a link."""
    n = 49152
    sk = (np.arange(n, dtype=np.uint32)[:, None] * 8 + np.arange(16, dtype=np.uint32)).astype(np.uint32)
    rows_per = ((2 << 30) // (n - 101)) & ~7  # distance_tile_rows of the second batch
    assert rows_per < n - 101
    want = np.arange(n, dtype=np.uint32)
    want -= want % 2
    for nearest in (False, True):
        for cuts in ([101], [101, 30001]):
            rep, n_reps, _ = grow(sk, cuts, 8, nearest)
            assert np.array_equal(rep, want) and n_reps == n // 2, (nearest, cuts)


def test_families_across_batches_in_row_tiles(gpu):
    n, L, k, s = 49152, 80, 21, 16
    sk = sketches_of(synth.family_reads(n, L, family=16), n, L, k, s)
    check_splits(sk, [[24583]], 4)


def test_identical_sketches_across_batches(family):
    sk = family[:512].copy()
    sk[[7, 100, 511]] = sk[3]
    sk[300] = sk[20]
    check_splits(sk, [[5], [50, 200, 400], [301]], 400)
    check_splits(sk, [[4, 8]], 150)


def test_unsorted_batches(family):
    """150 bp reads under s = 400 are in the fill regime (unsorted, zero tails): alone every one is kept, and after
    ascending representatives they drop the index's join while the answers stay equal."""
    n, L, k, s = 512, 150, 21, 400
    short = sketches_of(synth.independent_reads(n, L), n, L, k, s)
    rep, n_reps, _ = grow(short, [100, 300], 1, False)
    assert np.array_equal(rep, np.arange(n)) and n_reps == n
    mixed = np.concatenate([family[:256], short[:128], family[256:512]])
    check_splits(mixed, [[256, 384], [100, 300, 400]], 150)


def test_empty_batches(family):
    sk = family[:300]
    check_splits(sk, [[0, 0, 150, 150, 300]], 150)
    L = _lib.lib()
    for nearest in (False, True):
        with mash.Dereplicator(400, min_same=150, nearest=nearest) as d:
            first, n_new = C.c_uint64(9), C.c_uint64(9)
            assert L.pg_mash_dereplicator_add(d._h, None, 0, 400, None, C.byref(first), C.byref(n_new)) == _lib.PG_OK
            assert (first.value, n_new.value) == (0, 0)
            d.add(sk[:10])
            assert L.pg_mash_dereplicator_add(d._h, None, 0, -1, None, C.byref(first), C.byref(n_new)) == _lib.PG_OK
            assert (first.value, n_new.value) == (10, 0)
            assert L.pg_mash_dereplicator_add_dev(d._h, None, 0, 7, None, C.byref(first), None, None) == _lib.PG_OK and first.value == 10


def test_device_path_equals_host_path(family):
    import torch

    st = torch.cuda.current_stream().cuda_stream
    L = _lib.lib()
    for nearest in (False, True):
        want = mash.dereplicate(family, min_same=150, nearest=nearest)
        with mash.Dereplicator(400, min_same=150, nearest=nearest) as d:
            reps = []
            for a, b in ((0, 700), (700, 1500), (1500, 2048)):
                t = torch.from_numpy(family[a:b].view(np.int32)).cuda()
                rep, n_new = d.add(t)
                assert rep.is_cuda and rep.dtype == torch.int32 and isinstance(n_new, int)
                reps.append(rep.cpu().numpy().view(np.uint32))
            assert np.array_equal(np.concatenate(reps), want[0]) and d._ix.n == want[1]
        # the counters are optional
        with mash.Dereplicator(400, min_same=150, nearest=nearest) as d:
            d_sk = torch.from_numpy(family.view(np.int32)).cuda()
            out = torch.empty(len(family), dtype=torch.int32, device="cuda")
            _lib.check(L.pg_mash_dereplicator_add_dev(d._h, d_sk.data_ptr(), 1000, 400, out.data_ptr(), None, None, st))
            _lib.check(L.pg_mash_dereplicator_add_dev(d._h, d_sk[1000:].data_ptr(), 1048, 400, out[1000:].data_ptr(), None, None, st))
            assert np.array_equal(out.cpu().numpy().view(np.uint32), want[0])


def test_argument_errors_leave_the_dereplicator_unchanged(family):
    import torch

    L = _lib.lib()
    sk = family[:600]
    want = mash.dereplicate(sk, min_same=150)[0]
    rep = np.zeros(600, np.uint32)
    first, n_new = C.c_uint64(0), C.c_uint64(0)
    with mash.Dereplicator(400, min_same=150) as d:
        d.add(sk[:200])
        h = d._h
        # in order: s <= 0, an s other than the dereplicator's, the id limit, a null buffer
        assert L.pg_mash_dereplicator_add(h, None, 1 << 33, 0, None, None, None) == _lib.PG_ERR_PANIC
        assert L.pg_mash_dereplicator_add(h, None, 1 << 33, 16, None, None, None) == _lib.PG_ERR_ARG and "size" in _lib.last_error()
        assert L.pg_mash_dereplicator_add(h, None, (1 << 32) - 200, 400, None, None, None) == _lib.PG_ERR_ARG and "2^32" in _lib.last_error()
        assert L.pg_mash_dereplicator_add(h, None, 10, 400, rep.ctypes.data, None, None) == _lib.PG_ERR_ARG and "null" in _lib.last_error()
        assert L.pg_mash_dereplicator_add(h, sk.ctypes.data, 10, 400, None, None, None) == _lib.PG_ERR_ARG
        assert L.pg_mash_dereplicator_add_dev(h, None, 10, -1, None, None, None, None) == _lib.PG_ERR_PANIC
        assert L.pg_mash_dereplicator_add_dev(h, None, 10, 400, None, None, None, None) == _lib.PG_ERR_ARG
        with pytest.raises(_lib.PolyError):
            d.add(np.zeros((3, 16), np.uint32))
        with pytest.raises(_lib.GoPanic):
            d.add(np.zeros((3, 0), np.uint32))
        assert L.pg_mash_dereplicator_add(h, sk[200:].ctypes.data, 400, 400, rep.ctypes.data, C.byref(first), C.byref(n_new)) == _lib.PG_OK
        assert first.value == 200 and np.array_equal(rep[:400], want[200:])
        assert d.representatives().tolist() == np.nonzero(want == np.arange(600))[0].tolist()
    # reps: a short buffer keeps the first ids and reports the total
    with mash.Dereplicator(400, min_same=400) as d:
        d.add(torch.from_numpy(sk[:50].view(np.int32)).cuda())
        ids, cnt = np.zeros(50, np.uint32), C.c_uint64(0)
        assert L.pg_mash_dereplicator_reps(d._h, ids.ctypes.data, 10, C.byref(cnt)) == _lib.PG_ERR_ARG and cnt.value == 50
        assert ids[:10].tolist() == list(range(10))
        assert L.pg_mash_dereplicator_reps(d._h, None, 0, C.byref(cnt)) == _lib.PG_ERR_ARG and cnt.value == 50


def test_representative_index_answers_as_a_sketch_index(family):
    import torch

    sk, queries = family[:1500], family[1500:1700]
    for nearest in (False, True):
        with mash.Dereplicator(400, min_same=200, nearest=nearest) as d:
            for a, b in ((0, 400), (400, 1100), (1100, 1500)):
                rep, _ = d.add(sk[a:b])
            reps = d.representatives()
            with mash.SketchIndex(sk[reps]) as ix:
                for k in (1, 10):
                    got, want = d.nearest(queries, k), ix.nearest(queries, k)
                    mapped = np.where(want[0] == mash.NO_REF, mash.NO_REF, reps[np.minimum(want[0], len(reps) - 1)])
                    assert np.array_equal(got[0], mapped) and all(np.array_equal(g, w) for g, w in zip(got[1:], want[1:]))
                got, want = d.within(queries, min_same=150), ix.within(queries, min_same=150)
                assert np.array_equal(got[1], reps[want[1]]) and all(g.tobytes() == w.tobytes() for g, w in zip(got[2:], want[2:]))
                assert got[0].tobytes() == want[0].tobytes()
                dq = torch.from_numpy(queries.view(np.int32)).cuda()
                got = d.nearest(dq, 10, max_distance=0.6)
                want = ix.nearest(queries, 10, max_distance=0.6)
                mapped = np.where(want[0] == mash.NO_REF, mash.NO_REF, reps[np.minimum(want[0], len(reps) - 1)])
                assert np.array_equal(got[0].cpu().numpy().view(np.uint32), mapped)
            rep, _ = d.add(family[1700:])  # after device queries: the add waits for them
            assert np.array_equal(rep, mash.dereplicate(np.concatenate([sk, family[1700:]]), min_same=200, nearest=nearest)[0][1500:])
    with mash.Dereplicator(400, min_same=200) as d:  # no representative yet: every slot empty
        ref, same, _, nh = d.nearest(queries[:4], 3)
        assert (ref == mash.NO_REF).all() and (nh == 0).all()


def test_two_threads_add_to_one_dereplicator(family):
    """Each call's first is the number of sketches added before it; the result equals sequential adds in the
    order the calls took."""
    L = _lib.lib()
    batches = [family[i * 128:(i + 1) * 128] for i in range(16)]
    for nearest in (False, True):
        with mash.Dereplicator(400, min_same=150, nearest=nearest) as d:
            done = []  # (first, batch index, rep)
            lock = threading.Lock()

            def worker(idx):
                for i in idx:
                    rep, first, n_new = np.zeros(128, np.uint32), C.c_uint64(0), C.c_uint64(0)
                    _lib.check(L.pg_mash_dereplicator_add(d._h, batches[i].ctypes.data, 128, 400, rep.ctypes.data, C.byref(first), C.byref(n_new)))
                    with lock:
                        done.append((first.value, i, rep))

            th = [threading.Thread(target=worker, args=(range(t, 16, 2),)) for t in range(2)]
            for t in th:
                t.start()
            for t in th:
                t.join()
            done.sort()
            assert [f for f, _, _ in done] == [128 * j for j in range(16)]
            order = np.concatenate([batches[i] for _, i, _ in done])
            want = mash.dereplicate(order, min_same=150, nearest=nearest)[0]
            assert np.array_equal(np.concatenate([r for _, _, r in done]), want)


def test_oracle_restatement_agrees_on_the_device(family):
    sk = family[:400]
    for nearest in (False, True):
        want = derep_add_oracle.dereplicate_in_batches(sk, [90, 250], 150, nearest)
        rep, n_reps, _ = grow(sk, [90, 250], 150, nearest)
        assert np.array_equal(rep, want[0]) and n_reps == want[1]


@pytest.mark.parametrize("mode", ["first", "nearest"])
def test_cpp_mirror_agrees_with_the_oracle(family, mode):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "derep_add_tests"])
    sk = family[:512]
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "set.pgsketch")
        sketchfile.save(path, sk, np.full(len(sk), 400, np.uint32), 21, 400)
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "derep_add_tests"), path, "200", mode, "3"], capture_output=True, text=True,
                             timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: derep add tests pass"
    rep, n_reps = derep_oracle.dereplicate(sk, 200, mode == "nearest")
    assert lines[0] == f"{n_reps}" and lines[1] == " ".join(str(int(x)) for x in rep)
