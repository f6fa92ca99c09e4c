"""The tile loop over a distance plan across its tile cuts: the sparse pairs of a row range that the device pass
produces in two dense tiles, and the host dense rows that are copied out in two 64 Mi-pair blocks."""
import os

import numpy as np
import pytest

import oracle_ffi
from poly_b200 import _lib, mash

pytestmark = pytest.mark.gpu


def chain_pairs(n, lo, hi, upper):
    """distance_sparse of the chain (sketch i = 8 i ... 8 i + 15) over rows [lo, hi), sorted by (i, j): each sketch
    shares 8 values with each neighbour and nothing with any other sketch."""
    pairs = [(r, c) for r in range(lo, hi) for c in (r - 1, r + 1) if 0 <= c < n and (c > r or not upper)]
    i, j = np.array(pairs, np.uint32).reshape(-1, 2).T
    return i, j, np.full(len(i), 8, np.uint32)


@pytest.mark.parametrize("path", ["join", "pairwise"])
def test_sparse_pairs_across_the_tile_cut(gpu, monkeypatch, path):
    n = 49152
    rows_per = ((2 << 30) // n) & ~7  # distance_tile_rows over the whole set
    assert 0 < rows_per < n
    if path == "pairwise":
        monkeypatch.setenv("PG_K3_PAIRWISE", "1")
    sk = (np.arange(n, dtype=np.uint32)[:, None] * 8 + np.arange(16, dtype=np.uint32)).astype(np.uint32)
    # the whole set (cut at rows_per), the rows around that cut, and a range that does not start at row 0 (cut at 3 + rows_per)
    for lo, hi in ((0, n), (rows_per - 5, rows_per + 5), (3, n - 5)):
        for upper in (True, False):
            got = mash.distance_sparse(sk, lo, hi, upper=upper)
            want = chain_pairs(n, lo, hi, upper)
            assert all(np.array_equal(g, w) for g, w in zip(got, want)), (lo, hi, upper)


def test_host_dense_rows_across_blocks(gpu):
    import torch

    n, s = 8200, 32
    lo, hi = 3, n - 5
    rows_per = max(8, ((64 << 20) // n) & ~7)  # rows per 64 Mi-pair block of the host copy
    cut = lo + rows_per
    assert cut < hi  # two blocks
    rng = np.random.default_rng(8200)
    sk = np.sort(rng.integers(0, 8192, size=(n, s), dtype=np.uint32), axis=1)  # ascending, many shared values
    same, dist = mash.distance_block(sk, lo, hi)
    # one call into device buffers writes every row without the host loop
    d_sk = torch.from_numpy(sk.view(np.int32)).cuda()
    d_same = torch.empty((hi - lo, n), dtype=torch.int32, device="cuda")
    d_dist = torch.empty((hi - lo, n), dtype=torch.float64, device="cuda")
    _lib.check(_lib.lib().pg_mash_distance_block_dev(d_sk.data_ptr(), n, s, lo, hi, d_same.data_ptr(), d_dist.data_ptr(),
                                                     torch.cuda.current_stream().cuda_stream))
    assert np.array_equal(same, d_same.cpu().numpy().view(np.uint32))
    assert np.array_equal(dist.view(np.uint64), d_dist.cpu().numpy().view(np.uint64))
    del d_same, d_dist
    # the rows on both sides of the block cut against the oracle
    rc, want = oracle_ffi.similarity_block(sk, cut - 4, cut + 4, 0, n, len(os.sched_getaffinity(0)))
    assert rc == oracle_ffi.PO_OK
    assert (want.sum(axis=1) > s).all()  # every row shares values beyond its own diagonal entry
    assert np.array_equal(same[cut - 4 - lo: cut + 4 - lo], want)
    assert np.array_equal(dist[cut - 4 - lo: cut + 4 - lo], 1 - want / float(s))
