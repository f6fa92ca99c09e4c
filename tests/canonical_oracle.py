"""Plain restatement of canonical k-mer windows (PG_KMER_CANONICAL), for checking the canonical mode of the grouped
sketch, the sketcher and the screen.  TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
tools/bench_canonical.py.

The definition, as include/poly_b200.h states it: a record of length L has the windows 0 .. L - k (none when L < k);
for a window w, rc(w)[i] = complement(w[k - 1 - i]) with the oracle's complement table (po_reverse_complement:
upper- and lower-case IUPAC letters, every other byte to 0); canon(w) = w if w <= rc(w) in unsigned byte order, else
rc(w); the window hashes murmur3_32(canon(w)), seed 0.  This is NumPy over whole windows (a vectorised MurmurHash3
checked against oracle_ffi.murmur3_32 in test_oracle_canonical.py): no rings, no streams, nothing of the device walk.

The counting is not restated: sketch_groups, Sketcher, mash_screen and mash_screen_winners below run the forward
oracles (sketch_groups_oracle, sketcher_oracle, screen_oracle, screen_winners_oracle), which take every window hash
from screen_oracle.pool_hashes, with that one function swapped for pool_hashes here while they run."""
from __future__ import annotations

import contextlib

import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

import oracle_ffi
import screen_oracle
import screen_winners_oracle
import sketch_groups_oracle
import sketcher_oracle

_C1, _C2, _N5 = np.uint32(0xCC9E2D51), np.uint32(0x1B873593), np.uint32(0xE6546B64)
_CHUNK = 1 << 20  # windows hashed at once


def complement_table() -> np.ndarray:
    """complement() of every byte value, read from the oracle's reverse complement of bytes 0 .. 255."""
    return np.frombuffer(oracle_ffi.reverse_complement(bytes(range(256)))[::-1], np.uint8).copy()


_COMP = None


def _comp() -> np.ndarray:
    global _COMP
    if _COMP is None:
        _COMP = complement_table()
    return _COMP


def _rotl(x, r):
    return (x << np.uint32(r)) | (x >> np.uint32(32 - r))


def murmur3_rows(m: np.ndarray) -> np.ndarray:
    """MurmurHash3_x86_32 (seed 0) of every row of the [N, k] uint8 matrix m."""
    m = np.ascontiguousarray(m, np.uint8)
    n, k = m.shape
    h = np.zeros(n, np.uint32)
    nb = k // 4
    words = m[:, :4 * nb].copy().view("<u4") if nb else None
    for b in range(nb):
        kq = _rotl(words[:, b] * _C1, 15) * _C2
        h = _rotl(h ^ kq, 13) * np.uint32(5) + _N5
    if k & 3:
        t = np.zeros(n, np.uint32)
        for j in range(k & 3):
            t |= m[:, 4 * nb + j].astype(np.uint32) << np.uint32(8 * j)
        h ^= _rotl(t * _C1, 15) * _C2
    h ^= np.uint32(k)
    h ^= h >> np.uint32(16)
    h *= np.uint32(0x85EBCA6B)
    h ^= h >> np.uint32(13)
    h *= np.uint32(0xC2B2AE35)
    h ^= h >> np.uint32(16)
    return h


def canonical_rows(w: np.ndarray) -> np.ndarray:
    """canon(w) of every row of the [N, k] uint8 matrix of windows."""
    rc = _comp()[w[:, ::-1]]
    diff = w != rc
    first = np.argmax(diff, axis=1)
    at = np.arange(len(w))
    take_rc = diff[at, first] & (rc[at, first] < w[at, first])
    return np.where(take_rc[:, None], rc, w)


def window_hashes(bases, offsets, k: int) -> np.ndarray:
    """The canonical hash of every window of every record, positionally: record i's L_i - k + 1 windows in order,
    records in order."""
    if k < 1:
        raise ValueError("canonical k-mers need k >= 1")
    bases = np.ascontiguousarray(bases, np.uint8)
    offsets = np.ascontiguousarray(offsets, np.uint64).astype(np.int64)
    lens = offsets[1:] - offsets[:-1]
    nw = np.maximum(lens - k + 1, 0)
    at = np.zeros(len(lens) + 1, np.int64)
    at[1:] = np.cumsum(nw)
    out = np.zeros(int(at[-1]), np.uint32)
    for L in np.unique(lens[nw > 0]):
        L = int(L)
        idx = np.nonzero(lens == L)[0]
        per = L - k + 1
        rows_at_once = max(1, _CHUNK // per)
        for r0 in range(0, len(idx), rows_at_once):
            rid = idx[r0:r0 + rows_at_once]
            recs = bases[offsets[rid][:, None] + np.arange(L)]  # [rows, L]
            win = sliding_window_view(recs, k, axis=1)  # [rows, per, k]
            for w0 in range(0, per, _CHUNK):  # a long record in window chunks
                part = win[:, w0:w0 + _CHUNK].reshape(-1, k)
                h = murmur3_rows(canonical_rows(part)).reshape(len(rid), -1)
                for j, r in enumerate(rid):
                    out[at[r] + w0:at[r] + w0 + h.shape[1]] = h[j]
    return out


def pool_hashes(bases, offsets, k: int, nthreads: int = 1) -> np.ndarray:
    """Every canonical window hash of every record, the canonical counterpart of screen_oracle.pool_hashes."""
    return window_hashes(bases, offsets, k)


@contextlib.contextmanager
def hashing():
    """Within the block the forward oracles count canonical windows: screen_oracle.pool_hashes is this module's."""
    forward = screen_oracle.pool_hashes
    screen_oracle.pool_hashes = pool_hashes
    try:
        yield
    finally:
        screen_oracle.pool_hashes = forward


def sketch_groups(bases, offsets, group_offsets, k: int, s: int, min_copies: int = 1, nthreads: int = 1):
    with hashing():
        return sketch_groups_oracle.sketch_groups(bases, offsets, group_offsets, k, s, min_copies, nthreads)


def mash_screen(sketches, reads, k: int, nthreads: int = 1):
    with hashing():
        return screen_oracle.mash_screen(sketches, reads, k, nthreads)


def mash_screen_winners(sketches, reads, k: int, nthreads: int = 1):
    with hashing():
        return screen_winners_oracle.mash_screen_winners(sketches, reads, k, nthreads)


class Sketcher(sketcher_oracle.Sketcher):
    """sketcher_oracle.Sketcher over canonical windows."""

    def add(self, bases, offsets, group_offsets, first_group: int = 0, nthreads: int = 1) -> None:
        with hashing():
            super().add(bases, offsets, group_offsets, first_group, nthreads)
