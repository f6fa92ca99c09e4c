"""Plain restatement of the grouped sketch grown in place (pg_mash_sketcher), for checking its device path.  TEST
INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and tools/bench_sketcher.py.

The rule, word for word as include/poly_b200.h states it.  Per group g the sketcher keeps a cap C_g, which starts at
2^32 and never grows, and a state: every value v < C_g with c_g(v) >= 1, and beside each one min(c_g(v), m).  The
invariant is that every count below C_g is exact.  An add of records to group g does the following:
  1. Let V = the distinct values below the old C_g, with counts over the old state plus this batch's windows.
     Let Q = {v in V : c >= m}.
  2. t_s = (s-th smallest value of Q) + 1, or 2^32 if |Q| < s.
  3. t_B = the (B+1)-th smallest value of V, or 2^32 if |V| <= B.
  4. Set C_g = min(C_g, t_s, t_B) and keep V below it.
Batch windows at or above the old C_g are discarded.  Groups that get no records in an add are unchanged.
Row g holds the values of Q below C_g, ascending: count[g] = min(|Q below C_g|, s) of them, then zeros.
complete[g] = (count[g] == s) or (C_g == 2^32); held[g] = the number of values in the state.

The window hashes come from screen_oracle.pool_hashes (the C oracle's closed-form Sketch).  Each group is a dict of
values and saturated counts (two sorted arrays), a cap and the budget: no ranges, tables or passes."""
from __future__ import annotations

import numpy as np

import screen_oracle

RANGE = 1 << 32


class Sketcher:
    def __init__(self, n_groups: int, k: int, s: int, min_copies: int = 1, max_values: int | None = None):
        self.G, self.k, self.s, self.m = int(n_groups), int(k), int(s), int(min_copies)
        self.B = 64 * self.s if max_values is None else int(max_values)
        self.val = [np.zeros(0, np.int64) for _ in range(self.G)]
        self.cnt = [np.zeros(0, np.int64) for _ in range(self.G)]
        self.cap = [RANGE] * self.G

    def add(self, bases, offsets, group_offsets, first_group: int = 0, nthreads: int = 1) -> None:
        bases = np.ascontiguousarray(bases, np.uint8)
        offsets = np.ascontiguousarray(offsets, np.uint64)
        goff = np.asarray(group_offsets, np.int64)
        for i in range(len(goff) - 1):
            if goff[i + 1] > goff[i]:
                h = screen_oracle.pool_hashes(bases, offsets[goff[i]:goff[i + 1] + 1], self.k, nthreads)
                self.add_hashes(first_group + i, np.asarray(h, np.int64))

    def add_hashes(self, g: int, h: np.ndarray) -> None:
        C = self.cap[g]
        bv, bc = np.unique(h[h < C], return_counts=True)
        allv = np.concatenate([self.val[g], bv])
        allc = np.concatenate([self.cnt[g], bc])
        V, inv = np.unique(allv, return_inverse=True)  # step 1
        c = np.zeros(len(V), np.int64)
        np.add.at(c, inv, allc)
        Q = V[c >= self.m]
        t_s = int(Q[self.s - 1]) + 1 if len(Q) >= self.s else RANGE  # step 2
        t_B = int(V[self.B]) if len(V) > self.B else RANGE  # step 3
        C = min(C, t_s, t_B)  # step 4
        keep = V < C
        self.cap[g] = C
        self.val[g], self.cnt[g] = V[keep], np.minimum(c[keep], self.m)

    def rows(self):
        """(rows [G, s] uint32, count [G] uint32, complete [G] bool, held [G] uint64)."""
        rows = np.zeros((self.G, self.s), np.uint32)
        count = np.zeros(self.G, np.uint32)
        complete = np.zeros(self.G, bool)
        held = np.zeros(self.G, np.uint64)
        for g in range(self.G):
            q = self.val[g][self.cnt[g] >= self.m][: self.s]
            rows[g, : len(q)] = q
            count[g] = len(q)
            complete[g] = len(q) == self.s or self.cap[g] == RANGE
            held[g] = len(self.val[g])
        return rows, count, complete, held
