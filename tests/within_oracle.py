"""Brute-force radius queries over the CPU oracle: index_oracle's literal same matrix (query = receiver), kept where
same >= min_same, as the CSR lists of pg_mash_index_query_within.
TEST INFRASTRUCTURE ONLY (tests/, smoke() and tools/bench_within.py's parity check)."""
from __future__ import annotations

import numpy as np

from index_oracle import same_matrix


def within(refs: np.ndarray, queries: np.ndarray, min_same: int, nthreads: int = 0):
    """(offsets, ref, same, distance) in the radius query's CSR layout: every reference with same >= min_same,
    in reference order, for each query."""
    refs = np.ascontiguousarray(refs, dtype=np.uint32)
    queries = np.ascontiguousarray(queries, dtype=np.uint32)
    same = same_matrix(refs, queries, nthreads)
    den = max(min(refs.shape[1], queries.shape[1]), 1)
    q, j = np.nonzero(same >= min_same)  # row-major: query, then reference ascending
    offsets = np.zeros(len(queries) + 1, dtype=np.uint64)
    offsets[1:] = np.cumsum(np.bincount(q, minlength=len(queries)), dtype=np.uint64)
    cnt = same[q, j].astype(np.uint32)
    return offsets, j.astype(np.uint32), cnt, 1 - cnt.astype(np.float64) / np.float64(den)  # mash.go:134,139 in f64
