"""CPU tier of the sketch index's radius query: argument checks that need no device, and the CSR oracle
(within_oracle.within) against the top-k oracle ranking with k = n."""
import ctypes as C

import numpy as np
import pytest

import index_oracle
import within_oracle
from poly_b200 import _lib


def test_null_index_is_an_argument_error():
    q = np.zeros((2, 16), np.uint32)
    off = np.zeros(3, np.uint64)
    cnt = C.c_uint64(7)
    L = _lib.lib()
    assert L.pg_mash_index_query_within(None, q.ctypes.data, 2, 16, 1, off.ctypes.data, None, None, None, 0, C.byref(cnt)) == _lib.PG_ERR_ARG
    assert L.pg_mash_index_query_within_dev(None, None, 2, 16, 1, None, None, None, None, 0, None, None) == _lib.PG_ERR_ARG


def _sorted_by_rank(offsets, ref, same):
    """Each CSR row reordered by (same descending, reference ascending)."""
    rows = []
    for q in range(len(offsets) - 1):
        a, b = int(offsets[q]), int(offsets[q + 1])
        order = np.lexsort((ref[a:b], -same[a:b].astype(np.int64)))
        rows.append((ref[a:b][order], same[a:b][order]))
    return rows


@pytest.mark.parametrize("min_same", [1, 5, 20, 33])
def test_within_oracle_agrees_with_full_ranking(min_same):
    rng = np.random.default_rng(min_same)
    refs = np.sort(rng.integers(0, 60, size=(90, 32), dtype=np.uint32), axis=1)
    queries = np.sort(rng.integers(0, 60, size=(25, 32), dtype=np.uint32), axis=1)
    queries[:3] = refs[[0, 40, 89]]
    offsets, ref, same, dist = within_oracle.within(refs, queries, min_same)
    assert offsets[0] == 0 and offsets[-1] == len(ref) == len(same) == len(dist)
    assert (np.diff(offsets.astype(np.int64)) >= 0).all()
    r_ref, r_same, r_dist, r_nh = index_oracle.nearest(refs, queries, len(refs), min_same)
    assert np.array_equal(np.diff(offsets.astype(np.int64)), r_nh.astype(np.int64))
    for q, (g_ref, g_same) in enumerate(_sorted_by_rank(offsets, ref, same)):
        m = int(r_nh[q])
        assert np.array_equal(g_ref, r_ref[q, :m]) and np.array_equal(g_same, r_same[q, :m]), q
        a, b = int(offsets[q]), int(offsets[q + 1])
        assert (np.diff(ref[a:b].astype(np.int64)) > 0).all()  # reference order inside a list
    want = 1 - same.astype(np.float64) / np.float64(32)
    assert dist.tobytes() == want.tobytes()
