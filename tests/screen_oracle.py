"""Plain restatement of Mash Screen (Ondov et al. 2019) over a reference sketch set, for checking the screen's
device path.  TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and tools/bench_screen.py.

The window hashes come from the C oracle's closed-form Sketch (po_mash_sketch_closed), which writes every window
hash positionally when a sketch has more slots than the read has windows (mash.go:73-84): the windows 0 .. L - k - 1
of each read, murmur3 over their raw bytes.  The counting is NumPy: the pool's hash counts, then for each reference
its own value counts matched against them.  Nothing here follows the device design (no keys, no directory)."""
from __future__ import annotations

import numpy as np

import oracle_ffi


def pool_hashes(bases: np.ndarray, offsets: np.ndarray, k: int, nthreads: int = 1) -> np.ndarray:
    """Every window hash of every read [offsets[i], offsets[i+1]) of bases, in no particular order."""
    bases = np.ascontiguousarray(bases, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    lens = (offsets[1:] - offsets[:-1]).astype(np.int64)
    out = []
    for L in np.unique(lens):  # one batch per read length, each sketch one slot wider than its windows
        nk = int(L) - k
        if nk <= 0:
            continue
        idx = np.nonzero(lens == L)[0]
        starts = offsets[idx]
        grp = (starts[:, None] + np.arange(L, dtype=np.uint64)).reshape(-1)
        rc, sk = oracle_ffi.sketch_batch(bases[grp], np.arange(len(idx) + 1, dtype=np.uint64) * np.uint64(L), k, nk + 1, variant=1,
                                         nthreads=nthreads)
        assert rc == oracle_ffi.PO_OK, rc
        out.append(sk[:, :nk].reshape(-1))
    return np.concatenate(out) if out else np.zeros(0, np.uint32)


def mash_screen(sketches: np.ndarray, reads, k: int, nthreads: int = 1):
    """(shared uint32 [n], containment float64 [n], multiplicity uint64 [n]) of the pool `reads` (a list of str /
    bytes or a (bases, offsets) tuple of arrays) against the [n, s] reference words: shared = sum over v of
    min(c_r(v), c_pool(v)), containment = shared / s, multiplicity = the lower median of c_pool(v) over the shared
    hashes, each counted min(c_r(v), c_pool(v)) times (0 when nothing is shared)."""
    if k < 0:
        raise ValueError("k < 0")
    sk = np.ascontiguousarray(sketches, dtype=np.uint32)
    n, s = sk.shape
    bases, off = oracle_ffi.ragged(reads)
    pv, pc = np.unique(pool_hashes(bases, off, k, nthreads), return_counts=True)
    shared, cont, mult = np.zeros(n, np.uint32), np.zeros(n, np.float64), np.zeros(n, np.uint64)
    for r in range(n):
        v, c_r = np.unique(sk[r], return_counts=True)
        if len(pv):
            at = np.minimum(np.searchsorted(pv, v), len(pv) - 1)
            c_pool = np.where(pv[at] == v, pc[at], 0)
        else:
            c_pool = np.zeros(len(v), np.int64)
        take = np.minimum(c_r, c_pool)
        ms = np.sort(np.repeat(c_pool, take))
        shared[r] = len(ms)
        cont[r] = np.float64(len(ms)) / np.float64(s)
        mult[r] = ms[(len(ms) - 1) // 2] if len(ms) else 0
    return shared, cont, mult
