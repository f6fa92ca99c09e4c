"""A growing dereplication on the CPU: the checker of pg_mash_dereplicator_add, restated batch by batch.

A batch B appended to a dereplicated set is decided by the representatives kept so far that link to its rows
(counted with the batch row as the receiver, as a query of the representative index counts it) and by B's own
representatives before each row (counted with the lower row as the receiver, as dereplicate counts it).  Nothing
else is consulted: not the earlier sketches that are not representatives, and no earlier row is revisited.  Counts
come from the oracle's po_mash_similarity_block; the greedy loop is plain Python over them.
TEST INFRASTRUCTURE ONLY (tests/ and tools/bench_derep_add.py)."""
from __future__ import annotations

import numpy as np

import oracle_ffi


def _block(sk, row_lo, row_hi, col_lo, col_hi):
    rc, same = oracle_ffi.similarity_block(sk, row_lo, row_hi, col_lo, col_hi)
    assert rc == oracle_ffi.PO_OK, rc
    return same.astype(np.int64)


class GrowingDereplication:
    """The kept representatives (ids and rows) and the number of sketches added so far."""

    def __init__(self, s: int, min_same: int, nearest: bool = False):
        self.s, self.min_same, self.nearest = s, min_same, nearest
        self.rep_ids: list[int] = []
        self.rep_rows = np.zeros((0, s), np.uint32)
        self.n = 0

    def add(self, batch):
        """(rep uint32[m] as global ids, n_new_reps) of one batch."""
        b = np.ascontiguousarray(batch, np.uint32).reshape(-1, self.s)
        m, base, kept = len(b), self.n, len(self.rep_ids)
        joint = np.concatenate([b, self.rep_rows])
        old = _block(joint, 0, m, m, m + kept) if m and kept else np.zeros((m, kept), np.int64)  # batch row = receiver
        inner = _block(b, 0, m, 0, m) if m else np.zeros((0, 0), np.int64)  # lower row = receiver
        ids = np.asarray(self.rep_ids, np.int64)
        rep, new = np.zeros(m, np.int64), []
        for i in range(m):
            cand_id = np.r_[ids[old[i] >= self.min_same], [base + r for r in new if inner[r, i] >= self.min_same]].astype(np.int64)
            cand_same = np.r_[old[i][old[i] >= self.min_same], [inner[r, i] for r in new if inner[r, i] >= self.min_same]].astype(np.int64)
            if len(cand_id) == 0:
                new.append(i)
                rep[i] = base + i
            elif self.nearest:  # the largest count, then the smallest id
                rep[i] = cand_id[np.lexsort((cand_id, -cand_same))[0]]
            else:
                rep[i] = cand_id.min()
        self.rep_ids += [base + r for r in new]
        self.rep_rows = np.concatenate([self.rep_rows, b[new]])
        self.n += m
        return rep.astype(np.uint32), len(new)


def dereplicate_in_batches(sketches, cuts, min_same: int, nearest: bool = False):
    """(rep uint32[n], n_reps) of the [n, s] sketches added as the batches between the sorted cut points."""
    sk = np.ascontiguousarray(sketches, np.uint32)
    g = GrowingDereplication(sk.shape[1], min_same, nearest)
    edges = [0, *cuts, len(sk)]
    parts = [g.add(sk[a:b]) for a, b in zip(edges[:-1], edges[1:])]
    return np.concatenate([p[0] for p in parts]).astype(np.uint32), sum(p[1] for p in parts)
