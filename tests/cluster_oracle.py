"""Single-linkage groups of a sketch set on the CPU: the checker of pg_mash_cluster.

The reference has no clustering; the only reference arithmetic here is (*Mash).Similarity, through the
oracle's po_mash_similarity_block (row = receiver).  Sketches i < j are linked iff row i, column j counts at
least min_same; the groups are the connected components of the link graph (scipy's connected_components, which
shares nothing with the device's union-find); label[i] is the smallest index of i's component.
TEST INFRASTRUCTURE ONLY (tests/, __graft_entry__.smoke() and tools/bench_cluster.py)."""
from __future__ import annotations

import os

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

import oracle_ffi

_BLOCK_CELLS = 32 << 20  # counts per row block of the pair scan (128 MB)


def links_of(sketches, min_same: int, nthreads=None):
    """(i, j, same) of the linked pairs i < j of the [n, s] sketches, in (i, j) order."""
    sk = np.ascontiguousarray(sketches, np.uint32)
    n = len(sk)
    nthreads = nthreads or len(os.sched_getaffinity(0))
    out = [(np.zeros(0, np.int64),) * 3]
    rows = max(1, _BLOCK_CELLS // max(n, 1))
    for lo in range(0, n, rows):
        hi = min(n, lo + rows)
        rc, same = oracle_ffi.similarity_block(sk, lo, hi, lo, n, nthreads)  # columns below lo are never above the diagonal
        assert rc == oracle_ffi.PO_OK, rc
        i, j = np.nonzero(same >= min_same)
        keep = j > i
        out.append((i[keep] + lo, j[keep] + lo, same[i[keep], j[keep]].astype(np.int64)))
    return tuple(np.concatenate(c) for c in zip(*out))


def labels_of(n: int, link_i, link_j):
    """(label uint32[n], n_groups) of the graph over n items with the given edges."""
    if n == 0:
        return np.zeros(0, np.uint32), 0
    graph = coo_matrix((np.ones(len(link_i), np.uint8), (link_i, link_j)), shape=(n, n))
    n_groups, comp = connected_components(graph, directed=False)
    first = np.full(n_groups, n, np.int64)
    np.minimum.at(first, comp, np.arange(n))
    return first[comp].astype(np.uint32), int(n_groups)


def cluster(sketches, min_same: int, nthreads=None, want_links: bool = False):
    """(label uint32[n], n_groups, n_links) of the [n, s] sketches at same >= min_same; with want_links also the
    [n_links, 2] array of linked pairs i < j in (i, j) order."""
    i, j, _ = links_of(sketches, min_same, nthreads)
    label, n_groups = labels_of(len(sketches), i, j)
    return (label, n_groups, len(i), np.stack([i, j], axis=1)) if want_links else (label, n_groups, len(i))


def cluster_pairs(pair_i, pair_j, pair_same, n: int, min_same: int):
    """(label uint32[n], n_groups, n_links) from (i, j, same) triples, of which those with same >= min_same and
    i != j are the links: the host half of grouping through a sparse pair list."""
    pi, pj, ps = (np.asarray(a) for a in (pair_i, pair_j, pair_same))
    keep = (ps >= min_same) & (pi != pj)
    label, n_groups = labels_of(n, pi[keep], pj[keep])
    return label, n_groups, int(keep.sum())
