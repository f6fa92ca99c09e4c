"""Greedy representatives of a sketch set on the CPU: the checker of pg_mash_dereplicate.

The reference has no dereplication; the only reference arithmetic here is (*Mash).Similarity / Distance, through
the oracle's po_mash_similarity_block (row = receiver, scanned by cluster_oracle.links_of) and OracleMash.Distance.
Sketches r < i are linked iff row r, column i counts at least min_same.  In index order, i is a representative iff
no representative r < i is linked to i; any other i is assigned the smallest linked representative, or with
nearest=True the linked representative with the largest count, ties to the smaller index.  A plain serial loop over
the links, sharing nothing with the device's walk / mark split.
TEST INFRASTRUCTURE ONLY (tests/, __graft_entry__.smoke() and tools/bench_derep.py)."""
from __future__ import annotations

import numpy as np

from cluster_oracle import links_of


def _greedy(n: int, li, lj, ls, nearest: bool):
    """(rep uint32[n], n_reps) over the links li < lj with counts ls (every listed pair is linked)."""
    order = np.lexsort((lj, li))
    li, lj, ls = (np.asarray(a, np.int64)[order] for a in (li, lj, ls))
    start = np.searchsorted(li, np.arange(n + 1))
    rep = np.full(n, -1, np.int64)
    best = np.zeros(n, np.int64)
    for r in np.nonzero(np.diff(start))[0]:  # a sketch without later links only ever represents itself
        if rep[r] >= 0:
            continue
        rep[r] = r
        cj, cs = lj[start[r]: start[r + 1]], ls[start[r]: start[r + 1]]
        take = rep[cj] < 0
        if nearest:
            take |= cs > best[cj]  # strictly larger: an equal count keeps the earlier, smaller representative
        rep[cj[take]] = r
        best[cj[take]] = cs[take]
    alone = rep < 0
    rep[alone] = np.nonzero(alone)[0]
    return rep.astype(np.uint32), int((rep == np.arange(n)).sum())


def dereplicate(sketches, min_same: int, nearest: bool = False, nthreads=None):
    """(rep uint32[n], n_reps) of the [n, s] sketches at same >= min_same."""
    return _greedy(len(sketches), *links_of(sketches, min_same, nthreads), nearest)


def dereplicate_pairs(pair_i, pair_j, pair_same, n: int, min_same: int, nearest: bool = False):
    """(rep uint32[n], n_reps) from (i, j, same) triples, of which those with same >= min_same and i != j are the
    links, in either direction: the host half of dereplicating through a sparse pair list."""
    pi, pj, ps = (np.asarray(a, np.int64) for a in (pair_i, pair_j, pair_same))
    keep = (ps >= min_same) & (pi != pj)
    lo, hi, ps = np.minimum(pi, pj)[keep], np.maximum(pi, pj)[keep], ps[keep]
    _, first = np.unique(lo * max(n, 1) + hi, return_index=True)  # a pair listed both ways counts once
    return _greedy(n, lo[first], hi[first], ps[first], nearest)


def dereplicate_literal(mashes, max_distance: float, nearest: bool = False):
    """(rep uint32[n], n_reps) by a caller's loop over OracleMash.Distance, the lower index as the receiver:

        for i := range sketches {
            for _, r := range reps { if sketches[r].Distance(sketches[i]) <= maxDistance { rep[i] = r; continue outer } }
            reps = append(reps, i); rep[i] = i
        }

    with nearest=True the loop does not stop at the first representative within the cut but keeps the one at the
    smallest Distance, the earlier one on a tie.  Quadratic in the set: for small sets."""
    reps, rep = [], []
    for i, m in enumerate(mashes):
        pick, pick_d = -1, None
        for r in reps:
            d = mashes[r].Distance(m)
            if d <= max_distance and (pick < 0 or d < pick_d):
                pick, pick_d = r, d
                if not nearest:
                    break
        if pick < 0:
            reps.append(i)
            pick = i
        rep.append(pick)
    return np.array(rep, np.uint32), len(reps)
