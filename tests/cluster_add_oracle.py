"""A growing clustering on the CPU: the checker of pg_mash_clusterer_add, restated batch by batch.

A batch B added to a clustered prefix P is merged by three things only: the groups of P (its labels, nothing
else about how they were found), every link between a row of B and any sketch of P (counted with the batch row as
the receiver, as a query of the index over P counts it) and every link inside B (counted with the lower row as the
receiver, as cluster counts it).  The groups after the add are the connected components of the union of the three;
labels are the smallest id of each.  Counts come from the oracle's po_mash_similarity_block, components from
scipy through cluster_oracle.labels_of.
TEST INFRASTRUCTURE ONLY (tests/)."""
from __future__ import annotations

import numpy as np

import cluster_oracle
import oracle_ffi


def _block(sk, row_lo, row_hi, col_lo, col_hi):
    rc, same = oracle_ffi.similarity_block(sk, row_lo, row_hi, col_lo, col_hi)
    assert rc == oracle_ffi.PO_OK, rc
    return same.astype(np.int64)


class GrowingClustering:
    """Every sketch added so far, their labels and group count."""

    def __init__(self, s: int, min_same: int):
        self.s, self.min_same = s, min_same
        self.rows = np.zeros((0, s), np.uint32)
        self.label = np.zeros(0, np.uint32)
        self.n_groups = 0

    @property
    def n(self) -> int:
        return len(self.rows)

    def add(self, batch):
        """(labels uint32[m] of the batch's rows, n_groups, n_links, n_merged) of one batch."""
        b = np.ascontiguousarray(batch, np.uint32).reshape(-1, self.s)
        m, n = len(b), self.n
        if m == 0:
            return np.zeros(0, np.uint32), self.n_groups, 0, 0
        joint = np.concatenate([b, self.rows])
        cross = _block(joint, 0, m, m, m + n) if n else np.zeros((m, 0), np.int64)  # batch row = receiver
        inner = _block(b, 0, m, 0, m)  # lower row = receiver
        ci, cj = np.nonzero(cross >= self.min_same)
        ii, ij = np.nonzero(inner >= self.min_same)
        keep = ij > ii
        ii, ij = ii[keep], ij[keep]
        old = np.arange(n)  # each earlier sketch linked to its label: the earlier groups
        src = np.concatenate([old, n + ci, n + ii])
        dst = np.concatenate([self.label.astype(np.int64), cj, n + ij])
        label, n_groups = cluster_oracle.labels_of(n + m, src, dst)
        roots = np.nonzero(self.label == np.arange(n))[0]
        n_merged = int((label[roots] != roots).sum())
        self.rows = np.concatenate([self.rows, b])
        self.label, self.n_groups = label, n_groups
        return label[n:].copy(), n_groups, len(ci) + len(ii), n_merged


def cluster_in_batches(sketches, cuts, min_same: int):
    """Each add's (labels of all sketches so far, batch labels, n_groups, n_links, n_merged) for the [n, s] sketches
    added as the batches between the sorted cut points."""
    sk = np.ascontiguousarray(sketches, np.uint32)
    g = GrowingClustering(sk.shape[1], min_same)
    edges = [0, *cuts, len(sk)]
    out = []
    for a, b in zip(edges[:-1], edges[1:]):
        got = g.add(sk[a:b])
        out.append((g.label.copy(), *got))
    return out
