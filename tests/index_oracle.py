"""Brute-force top-k nearest references over the CPU oracle: the literal po_mash_similarity for every
query x reference pair (query = receiver), a stable sort by (-same, reference index), the cut.
TEST INFRASTRUCTURE ONLY (tests/ and tools/bench_query.py's parity check)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import oracle_ffi

NO_REF = 0xFFFFFFFF


def same_matrix(refs: np.ndarray, queries: np.ndarray, nthreads: int = 0) -> np.ndarray:
    """same[q, j] = queries[q].Similarity(refs[j]) matching count, as the oracle counts it."""
    refs = np.ascontiguousarray(refs, dtype=np.uint32)
    queries = np.ascontiguousarray(queries, dtype=np.uint32)
    nq, sq = queries.shape
    n, sr = refs.shape
    if nq == 0 or n == 0:
        return np.zeros((nq, n), dtype=np.uint32)
    if sq == sr:  # one array, rows = queries, columns = references: the multithreaded block driver
        rc, same = oracle_ffi.similarity_block(np.concatenate([queries, refs]), 0, nq, nq, nq + n, nthreads or os.cpu_count() or 1)
        assert rc == oracle_ffi.PO_OK, rc
        return same
    L = oracle_ffi.lib()
    out = np.zeros((nq, n), dtype=np.uint32)
    cnt, sim = C.c_int64(0), C.c_double(0)
    for q in range(nq):
        a = queries[q].ctypes.data
        for j in range(n):
            rc = L.po_mash_similarity(a, sq, refs[j].ctypes.data, sr, C.byref(cnt), C.byref(sim))
            assert rc == oracle_ffi.PO_OK, rc
            out[q, j] = cnt.value
    return out


def rank(same: np.ndarray, top_k: int, min_same: int, den: int):
    """(ref, same, distance, n_hits) of every row of a same matrix, in the index's output layout."""
    nq, n = same.shape
    ref = np.full((nq, top_k), NO_REF, dtype=np.uint32)
    cnt = np.zeros((nq, top_k), dtype=np.uint32)
    dist = np.ones((nq, top_k), dtype=np.float64)
    nh = np.zeros(nq, dtype=np.uint32)
    idx = np.arange(n)
    for q in range(nq):
        row = same[q].astype(np.int64)
        order = np.lexsort((idx, -row))  # stable: same descending, then index ascending
        order = order[row[order] >= min_same][:top_k]
        m = len(order)
        nh[q] = m
        ref[q, :m] = order
        cnt[q, :m] = row[order]
        dist[q, :m] = 1 - cnt[q, :m].astype(np.float64) / np.float64(den)  # mash.go:134,139 in f64
    return ref, cnt, dist, nh


def nearest(refs: np.ndarray, queries: np.ndarray, top_k: int, min_same: int, nthreads: int = 0):
    refs = np.ascontiguousarray(refs, dtype=np.uint32)
    queries = np.ascontiguousarray(queries, dtype=np.uint32)
    return rank(same_matrix(refs, queries, nthreads), top_k, min_same, min(refs.shape[1], queries.shape[1]))


def check_distances(refs: np.ndarray, queries: np.ndarray, ref: np.ndarray, dist: np.ndarray, nh: np.ndarray, samples: int = 64):
    """The listed distances equal the oracle's po_mash_distance bit for bit (a sample of the hits)."""
    L = oracle_ffi.lib()
    d = C.c_double(0)
    rng = np.random.default_rng(1)
    hits = [(q, t) for q in range(len(nh)) for t in range(int(nh[q]))]
    for i in rng.permutation(len(hits))[:samples]:
        q, t = hits[i]
        a, b = np.ascontiguousarray(queries[q], np.uint32), np.ascontiguousarray(refs[int(ref[q, t])], np.uint32)
        assert L.po_mash_distance(a.ctypes.data, len(a), b.ctypes.data, len(b), C.byref(d)) == oracle_ffi.PO_OK
        assert np.float64(d.value).tobytes() == np.float64(dist[q, t]).tobytes(), (q, t)
