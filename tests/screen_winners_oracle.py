"""Plain restatement of Mash Screen's winner-take-all (mash screen -w) over a reference sketch set, for checking the
screen's winners path.  TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__.smoke() and
tools/bench_screen_winners.py.

The first pass is screen_oracle.mash_screen; the reallocation is restated plainly, value by value: the references
holding each pool value, the winner by (first-pass shared, -index), then per reference the sums and the lower median
over the values it won.  No packed keys, no atomics, nothing of the device design."""
from __future__ import annotations

import numpy as np

import oracle_ffi
import screen_oracle


def mash_screen_winners(sketches: np.ndarray, reads, k: int, nthreads: int = 1):
    """Mash Screen's winner-take-all over mash_screen's first pass: each pool value goes to the contender (a
    reference holding it) with the largest first-pass shared, a tie to the smallest index; then, per reference,
    shared = sum over its won values of min(c_r(v), c_pool(v)), containment = shared / s and multiplicity = the lower
    median of c_pool(v) over its won values, each counted min(c_r(v), c_pool(v)) times (0 when it won nothing)."""
    first = screen_oracle.mash_screen(sketches, reads, k, nthreads)[0]
    sk = np.ascontiguousarray(sketches, dtype=np.uint32)
    n, s = sk.shape
    bases, off = oracle_ffi.ragged(reads)
    pv, pc = np.unique(screen_oracle.pool_hashes(bases, off, k, nthreads), return_counts=True)
    keep = np.isin(pv, sk)  # only values some reference holds can be shared
    pool = dict(zip(pv[keep].tolist(), pc[keep].tolist()))  # c_pool
    held = []  # held[r]: {value: c_r(value)}
    contenders = {}  # pool value -> the references holding it
    for r in range(n):
        v, c = np.unique(sk[r], return_counts=True)
        held.append(dict(zip(v.tolist(), c.tolist())))
        for x in v.tolist():
            if x in pool:
                contenders.setdefault(x, []).append(r)
    won = [[] for _ in range(n)]
    for x, rs in contenders.items():
        winner = max(rs, key=lambda r: (int(first[r]), -r))
        won[winner].append(x)
    shared, cont, mult = np.zeros(n, np.uint32), np.zeros(n, np.float64), np.zeros(n, np.uint64)
    for r in range(n):
        ms = sorted(c for x in won[r] for c in [pool[x]] * min(held[r][x], pool[x]))
        shared[r] = len(ms)
        cont[r] = np.float64(len(ms)) / np.float64(s)
        mult[r] = ms[(len(ms) - 1) // 2] if ms else 0
    return shared, cont, mult


def window_hashing_to(v: int, k: int, prefix: bytes = b"") -> bytes:
    """A k-byte window (k >= 4) whose murmur3 hash is v: the bytes of prefix (zero-padded, k - 4 of them at most) and
    the one full 4-byte block that murmur3's bijective block step then needs, solved backwards from v.  Lets a test
    put a given value, 0 for zero-tail words, in a pool."""
    assert k >= 4
    M = 0xFFFFFFFF
    c1, c2, n5 = 0xCC9E2D51, 0x1B873593, 0xE6546B64
    rotl = lambda x, r: ((x << r) | (x >> (32 - r))) & M
    mix = lambda w: rotl(w * c1 & M, 15) * c2 & M
    nb, tail = k // 4, k % 4
    last = 4 * (nb - 1)  # the solved block's offset
    w = (prefix + bytes(k))[:k]
    hh = 0
    for b in range(nb - 1):
        hh = (rotl(hh ^ mix(int.from_bytes(w[4 * b:4 * b + 4], "little")), 13) * 5 + n5) & M
    x = v  # undo fmix32
    x ^= x >> 16
    x = x * pow(0xC2B2AE35, -1, 1 << 32) & M
    x ^= (x >> 13) ^ (x >> 26)
    x = x * pow(0x85EBCA6B, -1, 1 << 32) & M
    x ^= x >> 16
    x ^= k  # the length
    if tail:
        x ^= mix(int.from_bytes(w[4 * nb:], "little"))
    blk = rotl((x - n5) * pow(5, -1, 1 << 32) & M, 32 - 13) ^ hh  # h = rotl(hh ^ blk, 13) * 5 + n5
    word = rotl(blk * pow(c2, -1, 1 << 32) & M, 32 - 15) * pow(c1, -1, 1 << 32) & M
    out = w[:last] + word.to_bytes(4, "little") + w[last + 4:]
    assert oracle_ffi.murmur3_32(out) == v
    return out
