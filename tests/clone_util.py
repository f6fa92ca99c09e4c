"""Seeded clone workloads for the tests and tools/bench_clone.py: a digest-screen library with planted
sites, combinatorial Golden Gate libraries (a backbone plus positions x variants with distinct
junction overhangs), and random ligation reactions over a small overhang alphabet."""
from __future__ import annotations

import random

import numpy as np

SITES = [b"GGTCTC", b"GAGACC", b"GAAGAC", b"GTCTTC", b"GCGATG", b"CATCGC", b"GCGATGCGATG", b"CATCGCATCGC"]
_ACGT = np.frombuffer(b"ACGT", np.uint8)


def scrub(seq: bytearray, sites=SITES, rng=None) -> bytearray:
    """Mutates seq until no site of `sites` occurs in it (upper case)."""
    rng = rng or np.random.default_rng(0)
    while True:
        s = bytes(seq).upper()
        hits = [s.find(x) for x in sites if s.find(x) >= 0]
        if not hits:
            return seq
        i = hits[0] + 2
        seq[i] = int(rng.choice(_ACGT[_ACGT != s[i]]))


def digest_library(n: int, seed: int, min_len: int = 20, max_len: int = 12000):
    """(parts, circular) of n parts, lengths log-uniform in [min_len, max_len], ~5% shorter than a site, mixed
    case, with planted sites of BsaI, BbsI and BtgZI (both strands, overlapping BtgZI chains, at both ends and
    across the origin of circular parts) and a few parts with a byte >= 0x80."""
    rng = np.random.default_rng(seed)
    parts, circ = [], []
    for i in range(n):
        L = int(np.exp(rng.uniform(np.log(min_len), np.log(max_len)))) if rng.random() > 0.05 else int(rng.integers(0, 6))
        s = bytearray(rng.choice(_ACGT, L).tobytes())
        for _ in range(int(rng.integers(0, 5))):
            site = SITES[int(rng.integers(len(SITES)))]
            where = rng.random()
            if len(site) > L:
                break
            p = 0 if where < 0.15 else L - len(site) if where < 0.3 else int(rng.integers(0, L - len(site) + 1))
            s[p: p + len(site)] = site
        c = bool(rng.random() < 0.4)
        if c and L > 12 and rng.random() < 0.3:  # a site across the origin
            site = SITES[int(rng.integers(len(SITES)))]
            k = int(rng.integers(1, len(site)))
            s[L - k:] = site[:k]
            s[: len(site) - k] = site[k:]
        if L and rng.random() < 0.3:  # a lower-case stretch
            a = int(rng.integers(0, L))
            b = min(L, a + int(rng.integers(1, 400)))
            s[a:b] = bytes(s[a:b]).lower()
        if L and rng.random() < 0.003:
            s[int(rng.integers(0, L))] = 0xC3
        parts.append(bytes(s))
        circ.append(c)
    return parts, circ


def overhangs(k: int, seed: int):
    """k distinct 4-mers, none palindromic and none the reverse complement of another"""
    from clone_oracle import rc

    rng = np.random.default_rng(seed)
    out = []
    while len(out) < k:
        o = rng.choice(_ACGT, 4).tobytes()
        if o == rc(o) or o in out or rc(o) in out:
            continue
        out.append(o)
    return out


def combinatorial_library(positions: int, variants: int, insert_len: int, backbone_len: int, seed: int):
    """(parts, expected clone count): a circular BsaI backbone carrying overhangs O[positions] -> O[0] and, for
    each position i, `variants` linear parts O[i] + insert + O[i+1] between BsaI sites.  Every choice of one
    variant per position closes one clone: variants ** positions distinct clones."""
    rng = np.random.default_rng(seed)
    O = overhangs(positions + 1, seed)

    def body(n):
        return scrub(bytearray(rng.choice(_ACGT, n).tobytes()), rng=rng)

    def flank():
        return bytes(body(12))

    def two_sites(make):  # exactly the two planted BsaI sites, none formed across a junction
        while True:
            p = make()
            d = p + p[:5]
            if sum(d.count(x) for x in (b"GGTCTC", b"GAGACC")) == 2:
                return p

    parts = [(two_sites(lambda: b"GGTCTCA" + O[positions] + bytes(body(backbone_len)) + O[0] + b"AGAGACC" + bytes(body(30))), True)]
    for i in range(positions):
        for _ in range(variants):
            parts.append((two_sites(lambda: flank() + b"GGTCTCA" + O[i] + bytes(body(insert_len)) + O[i + 1] + b"AGAGACC" + flank()), False))
    return parts, variants ** positions


def random_reaction(rng: random.Random):
    """Fragments over a small overhang alphabet: shared, reverse-complementary and palindromic overhangs, and
    repeated sequences, so attaches in both orientations, loops and duplicate clones all occur."""
    ohs = [b"AATT", b"GCGC", b"ACGT", b"GGAC", b"GTCC", b"TTAG", b"CTAA", b"CAGT"][: rng.randint(2, 8)]
    seqs_ = [bytes(rng.choice(b"ACGT") for _ in range(rng.randint(0, 12))) for _ in range(rng.randint(1, 4))]
    return [(rng.choice(seqs_), rng.choice(ohs), rng.choice(ohs)) for _ in range(rng.randint(1, 6))]
