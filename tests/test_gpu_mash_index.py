"""GPU tier of the sketch index (pg_mash_index_*): every result -- reference ids, counts, f64 distances bit for
bit, n_hits -- equals the brute-force ranking over the CPU oracle (tests/index_oracle.py)."""
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

import index_oracle
from poly_b200 import _lib, mash, sketchfile, synth

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def assert_same_result(got, want):
    for g, w, name in zip(got, want, ("ref", "same", "distance", "n_hits")):
        g = g.cpu().numpy() if hasattr(g, "cpu") else g
        if name == "distance":
            assert g.tobytes() == np.ascontiguousarray(w, np.float64).tobytes(), name
        else:
            assert np.array_equal(g.view(np.uint32) if g.dtype == np.int32 else g, w), name


def check(refs, queries, k, min_same, ix=None):
    own = ix is None
    ix = ix or mash.SketchIndex(refs)
    try:
        got = ix.nearest(queries, k, min_same=min_same)
    finally:
        if own:
            ix.close()
    want = index_oracle.nearest(refs, queries, k, min_same)
    assert_same_result(got, want)
    return got


@pytest.fixture(scope="module")
def family(gpu):
    """2000 x 2 kbp family reads (R = 20), k = 21, s = 500: references are reads with i % R < R - 4."""
    n, L, R = 2000, 2000, 20
    reads = synth.family_reads(n, L, family=R)
    sk = mash.sketch_uniform(reads, n, L, 21, 500)
    idx = np.arange(n)
    is_ref = idx % R < R - 4
    return sk[is_ref], sk[~is_ref], idx[is_ref] // R, idx[~is_ref] // R


@pytest.mark.parametrize("k", [1, 10, mash.INDEX_MAX_TOP_K])
@pytest.mark.parametrize("min_same", [0, 1, 501])
def test_family_reads_match_oracle(family, k, min_same):
    refs, queries, _, _ = family
    ref, _, dist, nh = check(refs, queries, k, min_same)
    index_oracle.check_distances(refs, queries, ref, dist, nh)


def test_family_top_k_equals_set_size(family):
    refs, queries, _, _ = family
    check(refs[:640], queries, 640, 0)
    check(refs[:640], queries, 640, 1)


def test_family_top10_lies_in_own_family(family):
    refs, queries, ref_fam, q_fam = family
    with mash.SketchIndex(refs) as ix:
        ref, same, _, nh = ix.nearest(queries, 10)
    assert (nh == 10).all()
    assert (ref_fam[ref] == q_fam[:, None]).all()
    assert (same[:, :-1] >= same[:, 1:]).all()


def test_ties_and_multisets():
    """Ascending sketches over a small value range: repeated values and many equal counts, so the cut falls
    inside runs of ties."""
    rng = np.random.default_rng(7)
    refs = np.sort(rng.integers(0, 40, size=(300, 64), dtype=np.uint32), axis=1)
    queries = np.sort(rng.integers(0, 40, size=(60, 64), dtype=np.uint32), axis=1)
    queries[:5] = refs[:5]  # exact copies as well
    with mash.SketchIndex(refs) as ix:
        for k in (1, 5, 17, 300):
            for min_same in (0, 1, 30, 64, 65):
                check(refs, queries, k, min_same, ix)


def test_skewed_values_take_pairwise_path():
    """One value in every reference: its bucket cannot fit the join's shared-memory sort at any bucketing, so
    the index falls back to the pairwise kernel for ascending queries too."""
    rng = np.random.default_rng(11)
    refs = np.sort(np.concatenate([np.full((5000, 4), 7, np.uint32), rng.integers(0, 1 << 20, size=(5000, 12), dtype=np.uint32)], axis=1), axis=1)
    queries = np.sort(np.concatenate([np.full((40, 2), 7, np.uint32), rng.integers(0, 1 << 20, size=(40, 14), dtype=np.uint32)], axis=1), axis=1)
    queries[:3] = refs[[0, 1234, 4999]]
    with mash.SketchIndex(refs) as ix:
        for k, min_same in ((1, 1), (10, 1), (64, 0), (1024, 3)):
            check(refs, queries, k, min_same, ix)


def _fill_sets():
    """Reads of one set of families at several lengths: 1100 bp give ascending sketches (L - k >= s), 150 / 200 bp
    fill-regime (positional, unsorted) ones; compact rows (SketchSize = L - k) have no zero tail."""
    n, fam = 240, 4
    long_reads = synth.family_reads(n, 1100, family=fam).reshape(n, 1100)
    asc = mash.sketch_uniform(long_reads.reshape(-1), n, 1100, 21, 1000)
    r150 = np.ascontiguousarray(long_reads[:, :150]).reshape(-1)
    r200 = np.ascontiguousarray(long_reads[:, :200]).reshape(-1)
    off150 = synth.uniform_offsets(n, 150)
    fill_full = mash.sketch_arrays(r150, off150, 21, 1000, pad_zero=True)[0]      # [n, 1000], zero tail
    fill_half = mash.sketch_arrays(r150, off150, 21, 500, pad_zero=True)[0]       # [n, 500], zero tail
    compact150 = mash.sketch_uniform(r150, n, 150, 21, 1000)                      # [n, 129]
    compact200 = mash.sketch_uniform(r200, n, 200, 21, 1000)                      # [n, 179]
    return asc, fill_full, fill_half, compact150, compact200


@pytest.fixture(scope="module")
def fill_sets(gpu):
    return _fill_sets()


def test_unsorted_sketches(fill_sets):
    asc, fill_full, fill_half, c150, c200 = fill_sets
    sel_r, sel_q = np.arange(240) % 5 != 0, np.arange(240) % 5 == 0
    cases = [
        (fill_full[sel_r], fill_full[sel_q]),  # zero-padded both sides
        (fill_full[sel_r], asc[sel_q]),        # unsorted references, ascending queries
        (asc[sel_r], fill_full[sel_q]),        # ascending references, unsorted queries
        (c150[sel_r], c150[sel_q]),            # unsorted without zero tail: the literal walk decides
        (asc[sel_r], c150[sel_q]),
    ]
    for refs, queries in cases:
        for k, min_same in ((1, 1), (10, 0), (50, 1)):
            check(refs, queries, k, min_same)


def test_unequal_sizes_receiver_rule(fill_sets):
    asc, fill_full, fill_half, c150, c200 = fill_sets
    sel_r, sel_q = np.arange(240) % 5 != 0, np.arange(240) % 5 == 0
    asc300 = np.ascontiguousarray(asc[:, :300])  # ascending prefixes are ascending sketches of size 300
    cases = [
        (fill_full[sel_r], fill_half[sel_q]),  # s_q < s_r, unsorted
        (fill_half[sel_r], fill_full[sel_q]),  # s_q > s_r, unsorted
        (c200[sel_r], c150[sel_q]),            # s_q < s_r, unsorted without zero tails
        (c150[sel_r], c200[sel_q]),            # s_q > s_r
        (asc[sel_r], asc300[sel_q]),           # ascending, s_q < s_r (probe)
        (asc300[sel_r], asc[sel_q]),           # ascending, s_q > s_r (probe)
    ]
    for refs, queries in cases:
        ref, _, dist, nh = check(refs, queries, 10, 1)
        index_oracle.check_distances(refs, queries, ref, dist, nh, samples=16)
        check(refs, queries, 7, 0)


def test_forced_small_query_blocks_equal_unforced(family, fill_sets):
    refs, queries, _, _ = family
    _, _, _, c150, c200 = fill_sets
    sets = [(refs, queries), (c200, c150)]
    base = []
    for r, q in sets:
        with mash.SketchIndex(r) as ix:
            base.append(ix.nearest(q, 10, min_same=0))
    os.environ["PG_INDEX_QUERY_ROWS"] = "7"
    try:
        for (r, q), want in zip(sets, base):
            with mash.SketchIndex(r) as ix:
                assert_same_result(ix.nearest(q, 10, min_same=0), want)
    finally:
        del os.environ["PG_INDEX_QUERY_ROWS"]


def test_reuse_concurrency_and_device_entry_points(family):
    import torch

    refs, queries, _, _ = family
    b1, b2 = queries[:150], queries[150:]
    with mash.SketchIndex(refs) as fresh:
        want1, want2 = fresh.nearest(b1, 10), fresh.nearest(b2, 10)
    ix = mash.SketchIndex(refs)
    assert_same_result(ix.nearest(b1, 10), want1)
    assert_same_result(ix.nearest(b2, 10), want2)
    results, errors = [None] * 8, []

    def work(t):
        try:
            results[t] = ix.nearest(b1 if t % 2 == 0 else b2, 10)
        except Exception as e:  # surfaced below
            errors.append(e)

    threads = [threading.Thread(target=work, args=(t,)) for t in range(8)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors
    for t in range(8):
        assert_same_result(results[t], want1 if t % 2 == 0 else want2)
    dev = torch.device("cuda", torch.cuda.current_device())
    d_refs = torch.from_numpy(refs.view(np.int32)).to(dev)
    d_q = torch.from_numpy(np.ascontiguousarray(b1).view(np.int32)).to(dev)
    assert_same_result(ix.nearest(d_q, 10), want1)              # host-built index, device queries
    with mash.SketchIndex(d_refs) as dix:                        # device-built index
        assert_same_result(dix.nearest(d_q, 10), want1)
        assert_same_result(dix.nearest(b2, 10), want2)
    ix.close()


def test_errors_and_empty_batches(family):
    refs, queries, _, _ = family
    with pytest.raises(_lib.GoPanic):
        mash.SketchIndex(np.zeros((3, 0), np.uint32))
    with mash.SketchIndex(refs) as ix:
        with pytest.raises(_lib.GoPanic):
            ix.nearest(np.zeros((2, 0), np.uint32), 5)
        for k in (0, mash.INDEX_MAX_TOP_K + 1):
            with pytest.raises(_lib.PolyError) as e:
                ix.nearest(queries[:4], k)
            assert e.value.code == _lib.PG_ERR_ARG
        ref, same, dist, nh = ix.nearest(np.zeros((0, 500), np.uint32), 5)
        assert ref.shape == (0, 5) and nh.shape == (0,)
        ref, same, dist, nh = ix.nearest(queries[:3], 5, min_same=10**6)  # nothing qualifies
        assert (nh == 0).all() and (ref == mash.NO_REF).all() and (same == 0).all() and (dist == 1.0).all()
        assert_same_result(ix.nearest(queries[:50], 10, max_distance=0.9), index_oracle.nearest(refs, queries[:50], 10, mash.min_same_for_distance(0.9, 500)))
        # unsorted queries take the pairwise tile kernel: 8 * (6000 + 500) words of tiles exceed its 200 KB
        unsorted = np.random.default_rng(9).integers(0, 1 << 32, size=(4, 6000), dtype=np.uint32)
        with pytest.raises(_lib.PolyError) as e:
            ix.nearest(unsorted, 5)
        assert e.value.code == _lib.PG_ERR_UNSUPPORTED


def test_sketch_file_index_equals_array_index(family, fill_sets):
    refs, queries, _, _ = family
    _, fill_full, _, c150, _ = fill_sets
    with tempfile.TemporaryDirectory() as td:
        # dense select-regime rows, and fill-regime rows stored without their zero tails
        for sk, cnt, s, full, q in ((refs, np.full(len(refs), 500, np.uint32), 500, refs, queries),
                                    (c150, np.full(len(c150), c150.shape[1], np.uint32), 1000, fill_full, fill_full[:40])):
            path = os.path.join(td, "set.pgsketch")
            sketchfile.save(path, sk, cnt, 21, s)
            with mash.SketchIndex.load(path) as a, mash.SketchIndex(full) as b:
                assert (a.n, a.s) == (len(cnt), s)
                for k, min_same in ((10, 1), (25, 0)):
                    assert_same_result(a.nearest(q, k, min_same=min_same), b.nearest(q, k, min_same=min_same))


def test_cpp_mirror_agrees_with_python(family):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "index_tests"])
    refs, queries, _, _ = family
    with tempfile.TemporaryDirectory() as td:
        rp, qp = os.path.join(td, "refs.pgsketch"), os.path.join(td, "queries.pgsketch")
        sketchfile.save(rp, refs, np.full(len(refs), 500, np.uint32), 21, 500)
        sketchfile.save(qp, queries, np.full(len(queries), 500, np.uint32), 21, 500)
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "index_tests"), rp, qp, "10", "1"], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: index tests pass"
    with mash.SketchIndex(refs) as ix:
        ref, same, dist, nh = ix.nearest(queries, 10)
    want = [" ".join([str(q), str(int(nh[q]))] + [f"{int(ref[q, t])}:{int(same[q, t])}:{int(dist[q:q + 1, t].view(np.uint64)[0]):016x}" for t in range(int(nh[q]))])
            for q in range(len(queries))]
    assert lines[:-1] == want
