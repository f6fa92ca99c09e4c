"""GPU tier of growing a sketch index (pg_mash_index_add*): after any sequence of adds, top-k queries at k = 10 and
1024 and radius queries answer byte for byte as an index created over the concatenated reference set."""
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

from poly_b200 import _lib, mash, sketchfile
from test_gpu_mash_index import _fill_sets
from test_gpu_mash_index_within import assert_same_lists, family, host, long_lists  # noqa: F401 (fixtures)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def answers(ix, queries, min_same=1):
    return ix.nearest(queries, 10), ix.nearest(queries, mash.INDEX_MAX_TOP_K), ix.within(queries, min_same=min_same)


def assert_same_answers(got, want):
    for g_top, w_top in zip(got[:2], want[:2]):
        for g, w, name in zip(g_top, w_top, ("ref", "same", "distance", "n_hits")):
            assert host(g).tobytes() == host(w).tobytes(), name
    assert_same_lists(got[2], [host(x) for x in want[2]])


def fresh_answers(refs, queries, min_same=1):
    with mash.SketchIndex(refs) as ix:
        return answers(ix, queries, min_same)


def grown(first, batches):
    ix = mash.SketchIndex(first)
    for b in batches:
        assert ix.add(b) == ix.n - len(b)
    return ix


def check_grown(refs, queries, cuts, min_same=1):
    parts = np.split(refs, cuts)
    with grown(parts[0], parts[1:]) as ix:
        assert ix.n == len(refs)
        assert_same_answers(answers(ix, queries, min_same), fresh_answers(refs, queries, min_same))


@pytest.fixture(scope="module")
def fill_sets(gpu):
    return _fill_sets()


@pytest.mark.parametrize("cuts", [[613], [1], [1599], [50, 51], [800, 1200], [3, 4, 300, 301, 900, 1598]])
def test_family_splits_equal_create(family, cuts):
    refs, queries = family
    check_grown(refs, queries, cuts, min_same=60)


def test_family_single_row_adds(family):
    refs, queries = family
    check_grown(refs[:800], queries, list(range(736, 800)), min_same=60)  # 64 adds of one row


def test_bucket_count_changes(family):
    """1600 x 500 entries take twice the buckets of 800 x 500: the merge rebuckets the joined entries."""
    refs, queries = family
    check_grown(refs, queries, [800], min_same=1)


def test_empty_index_grows(family):
    import torch

    refs, queries = family
    want = fresh_answers(refs, queries)
    dev = torch.device("cuda", torch.cuda.current_device())
    for empty in (np.zeros((0, 0), np.uint32), torch.zeros((0, 0), dtype=torch.int32, device=dev)):
        with mash.SketchIndex(empty) as ix:
            assert ix.add(refs[:700]) == 0 and (ix.n, ix.s) == (700, 500)
            assert ix.add(refs[700:]) == 700
            assert_same_answers(answers(ix, queries), want)
    asc300 = np.ascontiguousarray(refs[:, :300])
    with mash.SketchIndex(np.zeros((0, 500), np.uint32)) as ix:  # created with s = 500, holding nothing
        ix.add(asc300[:5])
        assert ix.s == 300
        ix.add(asc300[5:])
        assert_same_answers(answers(ix, queries), fresh_answers(asc300, queries))
        with pytest.raises(_lib.PolyError) as e:
            ix.add(refs[:2])
        assert e.value.code == _lib.PG_ERR_ARG


def test_unsorted_batch_drops_join(fill_sets):
    asc, fill_full, _, _, _ = fill_sets
    queries = np.concatenate([asc[200:], fill_full[200:]])
    refs = np.concatenate([asc[:150], fill_full[7:8], asc[150:200]])
    check_grown(refs, queries, [150])       # the unsorted sketch opens the batch
    check_grown(refs, queries, [150, 151])  # alone, then an ascending batch onto the unjoined index


def test_unsorted_batch_tile_does_not_fit():
    """6000-word sketches: once the join is dropped, queries need the pairwise tile, which does not fit -- as for
    the index created over the whole set."""
    rng = np.random.default_rng(3)
    refs = np.sort(rng.integers(0, 1 << 32, size=(40, 6000), dtype=np.uint32), axis=1)
    queries = np.sort(rng.integers(0, 1 << 32, size=(6, 6000), dtype=np.uint32), axis=1)
    queries[:2] = refs[[3, 31]]
    unsorted = rng.integers(0, 1 << 32, size=(1, 6000), dtype=np.uint32)
    with mash.SketchIndex(refs[:30]) as ix:
        ix.add(refs[30:])  # merged: the probe serves these queries
        assert_same_answers(answers(ix, queries), fresh_answers(refs, queries))
        ix.add(unsorted)
        with mash.SketchIndex(np.concatenate([refs, unsorted])) as fresh:
            for index in (ix, fresh):
                for call in (lambda: index.nearest(queries, 10), lambda: index.within(queries)):
                    with pytest.raises(_lib.PolyError) as e:
                        call()
                    assert e.value.code == _lib.PG_ERR_UNSUPPORTED


def test_unjoined_indexes_take_ascending_batches(fill_sets, long_lists):
    asc, fill_full, _, _, _ = fill_sets
    queries = np.concatenate([asc[200:], fill_full[200:]])
    check_grown(np.concatenate([fill_full[:100], asc[:140]]), queries, [100, 170])  # unsorted references
    refs, lq = long_lists
    check_grown(refs, lq, [1000, 2500], min_same=20)                    # merged buckets outgrow the join kernel's
    check_grown(np.concatenate([refs, lq[:20]]), lq, [3200], min_same=20)  # the join declines the first 3200


def test_values_above_old_vmax():
    rng = np.random.default_rng(17)
    low = np.sort(rng.integers(0, 1 << 20, size=(300, 64), dtype=np.uint32), axis=1)
    high = np.sort(rng.integers(1 << 31, 1 << 32, size=(200, 64), dtype=np.uint32), axis=1)
    mixed = np.sort(np.concatenate([low[:100, :32], high[:100, 32:]], axis=1), axis=1)
    refs = np.concatenate([low, high, mixed])
    queries = np.concatenate([low[::10], high[::10], mixed[::10],
                              np.sort(rng.integers(0, 1 << 32, size=(20, 64), dtype=np.uint32), axis=1)])
    check_grown(refs, queries, [300, 500])
    check_grown(refs, queries, [300, 301, 302])


def test_mixed_host_and_device_adds(family):
    import torch

    refs, queries = family
    dev = torch.device("cuda", torch.cuda.current_device())
    d_refs = torch.from_numpy(refs.view(np.int32)).to(dev)
    d_q = torch.from_numpy(np.ascontiguousarray(queries).view(np.int32)).to(dev)
    want = fresh_answers(refs, queries)
    with mash.SketchIndex(refs[:900]) as ix:        # host-built index, device batch, device queries
        ix.nearest(d_q, 10)
        assert ix.add(d_refs[900:1300]) == 900
        ix.add(refs[1300:])                           # host add after device queries
        assert_same_answers(answers(ix, d_q), want)
    with mash.SketchIndex(d_refs[:500]) as ix:      # device-built index, host batch, then a device batch
        ix.add(refs[500:1100])
        ix.add(d_refs[1100:])
        got = answers(ix, d_q)
        assert all(x.is_cuda for part in got for x in part)
        assert_same_answers(got, want)


def test_batch_ids_follow_old_n(family):
    refs, _ = family
    with mash.SketchIndex(refs[:1000]) as ix:
        assert ix.add(refs[1000:1300]) == 1000
        ref, same, _, _ = ix.nearest(refs[1000:1300], 1)
        assert (ref[:, 0] >= 1000).all() and (same[:, 0] == 500).all()
        off, lref, _, _ = ix.within(refs[1000:1300], min_same=500)
        assert (lref >= 1000).all() and len(lref) >= 300


def test_errors_leave_index_unchanged(family):
    import torch

    refs, queries = family
    L = _lib.lib()
    dev = torch.device("cuda", torch.cuda.current_device())
    st = torch.cuda.current_stream(dev).cuda_stream
    d_b = torch.from_numpy(refs[:4].view(np.int32)).to(dev)
    b = np.ascontiguousarray(refs[:4])
    # a null index is an argument error before anything else, m == 0 included
    assert L.pg_mash_index_add(None, None, 0, 0) == _lib.PG_ERR_ARG
    assert L.pg_mash_index_add_dev(None, None, 0, 0, None) == _lib.PG_ERR_ARG
    with mash.SketchIndex(refs[:1000]) as ix:
        before = answers(ix, queries)
        for add, buf in ((lambda *a: L.pg_mash_index_add(ix._h, *a), b.ctypes.data), (lambda *a: L.pg_mash_index_add_dev(ix._h, *a, st), d_b.data_ptr())):
            assert add(None, 0, -5) == _lib.PG_OK                   # m == 0 before s
            assert add(None, 4, 0) == _lib.PG_ERR_PANIC             # s <= 0 before the size and the buffer
            assert add(buf, 4, 499) == _lib.PG_ERR_ARG and "size" in _lib.last_error()
            assert add(None, 4, 499) == _lib.PG_ERR_ARG and "size" in _lib.last_error()  # size before the buffer
            assert add(None, (1 << 32) - 1000, 500) == _lib.PG_ERR_ARG and "2^32" in _lib.last_error()
            assert add(None, (1 << 32) - 1001, 500) == _lib.PG_ERR_ARG and "null" in _lib.last_error()
            assert ix.n == 1000
            assert_same_answers(answers(ix, queries), before)
        assert ix.add(np.zeros((0, 7), np.uint32)) == 1000 and ix.s == 500
        with pytest.raises(_lib.GoPanic):
            ix.add(np.zeros((3, 0), np.uint32))
        assert_same_answers(answers(ix, queries), before)


def test_queries_are_atomic_with_adds(family):
    refs, queries = family
    cuts = [600, 800, 1000, 1200, 1400, 1600]
    b1, b2 = queries[:120], queries[120:]
    prefix = []
    for c in cuts:
        with mash.SketchIndex(refs[:c]) as ix:
            prefix.append((ix.nearest(b1, 10), ix.within(b2, min_same=50)))
    ix = mash.SketchIndex(refs[:cuts[0]])
    results, errors = [[] for _ in range(8)], []

    def query(t):
        try:
            for _ in range(6):
                results[t].append(ix.nearest(b1, 10) if t % 2 == 0 else ix.within(b2, min_same=50))
        except Exception as e:  # surfaced below
            errors.append(e)

    def grow():
        try:
            for a, b in zip(cuts, cuts[1:]):
                ix.add(refs[a:b])
        except Exception as e:
            errors.append(e)

    threads = [threading.Thread(target=query, args=(t,)) for t in range(8)] + [threading.Thread(target=grow)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    assert ix.n == cuts[-1]
    for t in range(8):
        for got in results[t]:
            assert any(all(host(g).tobytes() == host(w).tobytes() for g, w in zip(got, p[t % 2])) for p in prefix), t
    ix.close()


def test_cpp_mirror_agrees_with_python(family):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "index_add_tests"])
    refs, queries = family
    with tempfile.TemporaryDirectory() as td:
        rp, qp = os.path.join(td, "refs.pgsketch"), os.path.join(td, "queries.pgsketch")
        sketchfile.save(rp, refs, np.full(len(refs), 500, np.uint32), 21, 500)
        sketchfile.save(qp, queries, np.full(len(queries), 500, np.uint32), 21, 500)
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "index_add_tests"), rp, qp, "100", "7"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: index add tests pass"
    with mash.SketchIndex(refs) as ix:
        off, ref, same, dist = ix.within(queries, min_same=100)
    bits = dist.view(np.uint64)
    want = [" ".join([str(q), str(int(off[q + 1] - off[q]))] + [f"{int(ref[h])}:{int(same[h])}:{int(bits[h]):016x}" for h in range(int(off[q]), int(off[q + 1]))])
            for q in range(len(queries))]
    assert lines[:-1] == want


@pytest.mark.parametrize("piece", ["1", "4099", "100003"])
def test_merge_in_pieces_equals_create(family, piece):
    """The merge runs in pieces of at most 2^31 - 1 keys cut at merge-path points; smaller pieces put the cuts
    inside these sets: every cut position for piece 1, cuts inside and between value runs for the others."""
    refs, queries = family
    rng = np.random.default_rng(23)
    low = np.sort(rng.integers(0, 1 << 12, size=(20, 64), dtype=np.uint32), axis=1)
    high = np.sort(rng.integers(1 << 11, 1 << 32, size=(10, 64), dtype=np.uint32), axis=1)
    small = np.concatenate([low, high, low[:3]])  # repeated rows: equal values across old and new ids
    os.environ["PG_JOIN_MERGE_PIECE"] = piece
    try:
        check_grown(small, np.concatenate([low[::4], high[::3]]), [20, 27])
        if piece != "1":
            check_grown(refs, queries, [800, 1300], min_same=60)
    finally:
        del os.environ["PG_JOIN_MERGE_PIECE"]
