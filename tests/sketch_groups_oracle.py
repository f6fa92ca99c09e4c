"""Plain restatement of the grouped sketch (pg_mash_sketch_groups), for checking its device path.  TEST
INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and tools/bench_sketch_groups.py.

The window hashes of each group come from screen_oracle.pool_hashes (the C oracle's closed-form Sketch: windows
0 .. L - k - 1 of every record, murmur3 over the raw bytes).  Then np.unique counts them, the values seen at least
min_copies times are kept, and the row is the first s of them.  Nothing here follows the device design: no hash
ranges, no tables, no passes."""
from __future__ import annotations

import numpy as np

import screen_oracle


def sketch_groups(bases, offsets, group_offsets, k: int, s: int, min_copies: int = 1, nthreads: int = 1):
    """(rows [G, s] uint32, count [G] uint32): row g = the smallest s distinct window hashes of records
    [group_offsets[g], group_offsets[g+1]) that occur at least min_copies times, ascending, then zeros."""
    bases = np.ascontiguousarray(bases, np.uint8)
    offsets = np.ascontiguousarray(offsets, np.uint64)
    goff = np.asarray(group_offsets, np.int64)
    G = len(goff) - 1
    rows, count = np.zeros((G, s), np.uint32), np.zeros(G, np.uint32)
    for g in range(G):
        v, c = np.unique(screen_oracle.pool_hashes(bases, offsets[goff[g]:goff[g + 1] + 1], k, nthreads), return_counts=True)
        v = v[c >= min_copies][:s]
        rows[g, :len(v)] = v
        count[g] = len(v)
    return rows, count


def flatten_groups(groups):
    """A list of lists of uint8 arrays / bytes -> (bases, offsets, group_offsets)."""
    recs = [np.frombuffer(bytes(r), np.uint8) if isinstance(r, (bytes, bytearray)) else np.asarray(r, np.uint8) for g in groups for r in g]
    offsets = np.zeros(len(recs) + 1, np.uint64)
    offsets[1:] = np.cumsum([len(r) for r in recs], dtype=np.uint64)
    goff = np.zeros(len(groups) + 1, np.uint64)
    goff[1:] = np.cumsum([len(g) for g in groups], dtype=np.uint64)
    bases = np.concatenate(recs) if recs else np.zeros(0, np.uint8)
    return np.ascontiguousarray(bases, np.uint8), offsets, goff
