"""GPU tier of the sketch index's radius query (pg_mash_index_query_within*): offsets, reference ids, counts and the
bytes of the f64 distances equal the CSR lists built from the CPU oracle (tests/within_oracle.py)."""
import ctypes as C
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

import oracle_ffi
import within_oracle
from poly_b200 import _lib, mash, sketchfile, synth
from test_gpu_mash_index import _fill_sets

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def host(x):
    x = x.cpu().numpy() if hasattr(x, "cpu") else x
    return x.view(np.uint32) if x.dtype == np.int32 else x.view(np.uint64) if x.dtype == np.int64 else x


def assert_same_lists(got, want):
    for g, w, name in zip(got, want, ("offsets", "ref", "same", "distance")):
        g, w = host(g), np.ascontiguousarray(w)
        assert g.dtype == w.dtype and g.tobytes() == w.tobytes(), name


def check(refs, queries, min_same, ix=None):
    own = ix is None
    ix = ix or mash.SketchIndex(refs)
    try:
        got = ix.within(queries, min_same=min_same)
    finally:
        if own:
            ix.close()
    assert_same_lists(got, within_oracle.within(refs, queries, min_same))
    return got


def check_distances(refs, queries, lists, samples=64):
    """Sampled hits: the listed distance equals the oracle's po_mash_distance bit for bit."""
    off, ref, _, dist = (host(x) for x in lists)
    q_of = np.repeat(np.arange(len(off) - 1), np.diff(off.astype(np.int64)))
    L = oracle_ffi.lib()
    d = C.c_double(0)
    for h in np.random.default_rng(1).permutation(len(ref))[:samples]:
        a, b = np.ascontiguousarray(queries[q_of[h]], np.uint32), np.ascontiguousarray(refs[int(ref[h])], np.uint32)
        assert L.po_mash_distance(a.ctypes.data, len(a), b.ctypes.data, len(b), C.byref(d)) == oracle_ffi.PO_OK
        assert np.float64(d.value).tobytes() == np.float64(dist[h]).tobytes(), h


def top_k_of(lists, nq, k):
    """Each list sorted by (same desc, ref asc) and cut to k, in nearest()'s layout."""
    off, ref, same, dist = (host(x) for x in lists)
    o_ref, o_same = np.full((nq, k), mash.NO_REF, np.uint32), np.zeros((nq, k), np.uint32)
    o_dist, nh = np.ones((nq, k), np.float64), np.zeros(nq, np.uint32)
    for q in range(nq):
        a, b = int(off[q]), int(off[q + 1])
        order = np.lexsort((ref[a:b], -same[a:b].astype(np.int64)))[:k] + a
        m = len(order)
        o_ref[q, :m], o_same[q, :m], o_dist[q, :m], nh[q] = ref[order], same[order], dist[order], m
    return o_ref, o_same, o_dist, nh


@pytest.fixture(scope="module")
def family(gpu):
    """2000 x 2 kbp family reads (R = 20), k = 21, s = 500: references are reads with i % R < R - 4."""
    n, L, R = 2000, 2000, 20
    sk = mash.sketch_uniform(synth.family_reads(n, L, family=R), n, L, 21, 500)
    is_ref = np.arange(n) % R < R - 4
    return sk[is_ref], sk[~is_ref]


@pytest.fixture(scope="module")
def long_lists(gpu):
    """3200 references over a small value range: every query hits nearly all of them, beyond the top-k cap."""
    rng = np.random.default_rng(5)
    refs = np.sort(rng.integers(0, 50, size=(3200, 64), dtype=np.uint32), axis=1)
    queries = np.sort(rng.integers(0, 50, size=(24, 64), dtype=np.uint32), axis=1)
    return refs, queries


@pytest.fixture(scope="module")
def fill_sets(gpu):
    return _fill_sets()


@pytest.mark.parametrize("min_same", [1, 100, 501])
def test_family_reads_match_oracle(family, min_same):
    refs, queries = family
    got = check(refs, queries, min_same)
    if min_same == 501:
        assert int(host(got[0])[-1]) == 0  # above min(sq, s): empty lists
    else:
        check_distances(refs, queries, got)


def test_lists_longer_than_top_k_cap(long_lists):
    refs, queries = long_lists
    off = host(check(refs, queries, 1)[0])
    assert (np.diff(off.astype(np.int64)) > mash.INDEX_MAX_TOP_K).all()
    check(refs, queries, 20)


@pytest.mark.parametrize("k", [10, mash.INDEX_MAX_TOP_K])
def test_sorted_lists_cut_to_k_equal_nearest(family, long_lists, k):
    for refs, queries in (family, long_lists):
        with mash.SketchIndex(refs) as ix:
            lists = ix.within(queries, min_same=1)
            want = ix.nearest(queries, k, min_same=1)
        for g, w, name in zip(top_k_of(lists, len(queries), k), want, ("ref", "same", "distance", "n_hits")):
            assert np.asarray(g).tobytes() == np.ascontiguousarray(w).tobytes(), name


def test_ties_and_multisets():
    rng = np.random.default_rng(7)
    refs = np.sort(rng.integers(0, 40, size=(300, 64), dtype=np.uint32), axis=1)
    queries = np.sort(rng.integers(0, 40, size=(60, 64), dtype=np.uint32), axis=1)
    queries[:5] = refs[:5]
    with mash.SketchIndex(refs) as ix:
        for min_same in (1, 30, 64, 65):
            check(refs, queries, min_same, ix)


def test_skewed_values_take_pairwise_path():
    rng = np.random.default_rng(11)
    refs = np.sort(np.concatenate([np.full((5000, 4), 7, np.uint32), rng.integers(0, 1 << 20, size=(5000, 12), dtype=np.uint32)], axis=1), axis=1)
    queries = np.sort(np.concatenate([np.full((40, 2), 7, np.uint32), rng.integers(0, 1 << 20, size=(40, 14), dtype=np.uint32)], axis=1), axis=1)
    queries[:3] = refs[[0, 1234, 4999]]
    with mash.SketchIndex(refs) as ix:
        for min_same in (1, 3, 16):
            check(refs, queries, min_same, ix)


def test_unsorted_and_unequal_sizes(fill_sets):
    asc, fill_full, fill_half, c150, c200 = fill_sets
    sel_r, sel_q = np.arange(240) % 5 != 0, np.arange(240) % 5 == 0
    asc300 = np.ascontiguousarray(asc[:, :300])
    cases = [
        (fill_full[sel_r], fill_full[sel_q]),  # zero-padded both sides
        (fill_full[sel_r], asc[sel_q]),        # unsorted references, ascending queries
        (asc[sel_r], fill_full[sel_q]),        # ascending references, unsorted queries
        (c150[sel_r], c150[sel_q]),            # unsorted without zero tail
        (fill_full[sel_r], fill_half[sel_q]),  # s_q < s_r, unsorted
        (fill_half[sel_r], fill_full[sel_q]),  # s_q > s_r, unsorted
        (c200[sel_r], c150[sel_q]),            # s_q < s_r, no zero tails
        (c150[sel_r], c200[sel_q]),            # s_q > s_r
        (asc[sel_r], asc300[sel_q]),           # ascending, s_q < s_r (probe)
        (asc300[sel_r], asc[sel_q]),           # ascending, s_q > s_r (probe)
    ]
    for refs, queries in cases:
        got = check(refs, queries, 1)
        check_distances(refs, queries, got, samples=16)
        check(refs, queries, 40)


@pytest.mark.parametrize("rows", ["1", "7"])
def test_forced_small_query_blocks_equal_unforced(family, fill_sets, rows):
    refs, queries = family
    _, _, _, c150, c200 = fill_sets
    sets = [(refs, queries), (c200, c150)]
    base = []
    for r, q in sets:
        with mash.SketchIndex(r) as ix:
            base.append(ix.within(q, min_same=1))
    os.environ["PG_INDEX_QUERY_ROWS"] = rows
    try:
        for (r, q), want in zip(sets, base):
            with mash.SketchIndex(r) as ix:
                assert_same_lists(ix.within(q, min_same=1), want)
    finally:
        del os.environ["PG_INDEX_QUERY_ROWS"]


def _host_call(ix, queries, min_same, cap, lists=True):
    nq, sq = queries.shape
    off = np.zeros(nq + 1, np.uint64)
    ref, same, dist = np.zeros(max(cap, 1), np.uint32), np.zeros(max(cap, 1), np.uint32), np.zeros(max(cap, 1), np.float64)
    cnt = C.c_uint64(0)
    q = np.ascontiguousarray(queries)
    rc = _lib.lib().pg_mash_index_query_within(ix._h, q.ctypes.data, nq, sq, min_same, off.ctypes.data, ref.ctypes.data if lists else None,
                                               same.ctypes.data if lists else None, dist.ctypes.data if lists else None, cap, C.byref(cnt))
    return rc, int(cnt.value), off, ref, same, dist


def test_capacity(family):
    import torch

    refs, queries = family
    want = within_oracle.within(refs, queries, 1)
    total = int(want[0][-1])
    with mash.SketchIndex(refs) as ix:
        cap = total // 3
        rc, cnt, off, ref, same, dist = _host_call(ix, queries, 1, cap)  # too small: the prefix and the whole offsets
        assert rc == _lib.PG_ERR_ARG and cnt == total
        assert off.tobytes() == want[0].tobytes()
        assert ref[:cap].tobytes() == want[1][:cap].tobytes() and same[:cap].tobytes() == want[2][:cap].tobytes()
        assert dist[:cap].tobytes() == want[3][:cap].tobytes()
        rc, cnt, off, *_ = _host_call(ix, queries, 1, 0, lists=False)  # counting call
        assert rc == _lib.PG_OK and cnt == total and off.tobytes() == want[0].tobytes()
        # _dev: never past the cap, the true total on the device
        dev = torch.device("cuda", torch.cuda.current_device())
        d_q = torch.from_numpy(queries.view(np.int32)).to(dev)
        d_off = torch.zeros(len(queries) + 1, dtype=torch.int64, device=dev)
        d_n = torch.zeros((), dtype=torch.int64, device=dev)
        sentinel = 0x5A5A5A5A
        d_ref = torch.full((cap + 64,), sentinel, dtype=torch.int32, device=dev)
        d_same = torch.full((cap + 64,), sentinel, dtype=torch.int32, device=dev)
        d_dist = torch.full((cap + 64,), 7.0, dtype=torch.float64, device=dev)
        st = torch.cuda.current_stream(dev).cuda_stream
        rc = _lib.lib().pg_mash_index_query_within_dev(ix._h, d_q.data_ptr(), len(queries), queries.shape[1], 1, d_off.data_ptr(), d_ref.data_ptr(),
                                                       d_same.data_ptr(), d_dist.data_ptr(), cap, d_n.data_ptr(), st)
        assert rc == _lib.PG_OK
        torch.cuda.synchronize(dev)
        assert int(d_n.item()) == total and host(d_off).tobytes() == want[0].tobytes()
        assert (d_ref[cap:] == sentinel).all() and (d_same[cap:] == sentinel).all() and (d_dist[cap:] == 7.0).all()
        assert host(d_ref[:cap]).tobytes() == want[1][:cap].tobytes() and host(d_dist[:cap]).tobytes() == want[3][:cap].tobytes()


def test_device_entry_points_and_threads(family):
    import torch

    refs, queries = family
    b1, b2 = queries[:150], queries[150:]
    with mash.SketchIndex(refs) as fresh:
        w1, w2 = fresh.within(b1, min_same=50), fresh.within(b2, min_same=50)
        n1, n2 = fresh.nearest(b1, 10), fresh.nearest(b2, 10)
    ix = mash.SketchIndex(refs)
    results, errors = [None] * 8, []

    def work(t):
        try:
            b = b1 if t % 4 < 2 else b2
            results[t] = ix.nearest(b, 10) if t % 2 == 0 else ix.within(b, min_same=50)
        except Exception as e:  # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t in range(8):
        want = (n1, w1, n2, w2)[t % 4]
        for g, w in zip(results[t], want):
            assert host(g).tobytes() == np.ascontiguousarray(w).tobytes(), t
    dev = torch.device("cuda", torch.cuda.current_device())
    d_refs = torch.from_numpy(refs.view(np.int32)).to(dev)
    d_q = torch.from_numpy(np.ascontiguousarray(b1).view(np.int32)).to(dev)
    got = ix.within(d_q, min_same=50)                         # host-built index, device queries
    assert all(x.is_cuda for x in got)
    assert_same_lists(got, w1)
    with mash.SketchIndex(d_refs) as dix:                     # device-built index
        assert_same_lists(dix.within(d_q, min_same=50), w1)
        assert_same_lists(dix.within(b2, min_same=50), w2)
    ix.close()


def test_errors_and_edges(family):
    refs, queries = family
    with mash.SketchIndex(refs) as ix:
        with pytest.raises(_lib.PolyError) as e:
            ix.within(queries[:4], min_same=0)
        assert e.value.code == _lib.PG_ERR_ARG
        with pytest.raises(_lib.GoPanic):
            ix.within(np.zeros((2, 0), np.uint32))
        off, ref, same, dist = ix.within(np.zeros((0, 500), np.uint32))
        assert off.tolist() == [0] and len(ref) == len(same) == len(dist) == 0
        for md in (1.0, 1.5):
            with pytest.raises(ValueError):
                ix.within(queries[:4], max_distance=md)
        assert_same_lists(ix.within(queries[:50], max_distance=0.9), within_oracle.within(refs, queries[:50], mash.min_same_for_distance(0.9, 500)))
        unsorted = np.random.default_rng(9).integers(0, 1 << 32, size=(4, 6000), dtype=np.uint32)
        with pytest.raises(_lib.PolyError) as e:
            ix.within(unsorted)
        assert e.value.code == _lib.PG_ERR_UNSUPPORTED
        # the library's own order: min_same == 0 before nq == 0, nq == 0 before sq <= 0 and a null offsets array
        L, cnt = _lib.lib(), C.c_uint64(9)
        assert L.pg_mash_index_query_within(ix._h, None, 0, 500, 0, None, None, None, None, 0, C.byref(cnt)) == _lib.PG_ERR_ARG
        off = np.full(1, 5, np.uint64)
        assert L.pg_mash_index_query_within(ix._h, None, 0, 0, 1, off.ctypes.data, None, None, None, 0, C.byref(cnt)) == _lib.PG_OK
        assert off[0] == 0 and cnt.value == 0
        assert L.pg_mash_index_query_within(ix._h, None, 3, 0, 1, None, None, None, None, 0, C.byref(cnt)) == _lib.PG_ERR_PANIC
        q = np.ascontiguousarray(queries[:3])
        assert L.pg_mash_index_query_within(ix._h, q.ctypes.data, 3, 500, 1, None, None, None, None, 0, C.byref(cnt)) == _lib.PG_ERR_ARG
    with mash.SketchIndex(np.zeros((0, 500), np.uint32)) as empty:
        off, ref, _, _ = empty.within(queries[:7])
        assert off.tolist() == [0] * 8 and len(ref) == 0


def test_cpp_mirror_agrees_with_python(family):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "within_tests"])
    refs, queries = family
    with tempfile.TemporaryDirectory() as td:
        rp, qp = os.path.join(td, "refs.pgsketch"), os.path.join(td, "queries.pgsketch")
        sketchfile.save(rp, refs, np.full(len(refs), 500, np.uint32), 21, 500)
        sketchfile.save(qp, queries, np.full(len(queries), 500, np.uint32), 21, 500)
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "within_tests"), rp, qp, "100"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: within tests pass"
    with mash.SketchIndex(refs) as ix:
        off, ref, same, dist = ix.within(queries, min_same=100)
    bits = dist.view(np.uint64)
    want = [" ".join([str(q), str(int(off[q + 1] - off[q]))] + [f"{int(ref[h])}:{int(same[h])}:{int(bits[h]):016x}" for h in range(int(off[q]), int(off[q + 1]))])
            for q in range(len(queries))]
    assert lines[:-1] == want
