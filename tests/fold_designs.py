"""Designed fold inputs for the limit tests: G/C helices in an A background.

A pairs with nothing in such an item (it holds no T, and an RNA item holds one U), so the C restatement's
cost depends on the G/C positions alone and items up to 1 024 nt stay affordable to check.  Every design
is seeded, so an item is the same string on every run."""
from __future__ import annotations

import random

COMP = {"G": "C", "C": "G"}


def rc(x: str) -> str:
    return "".join(COMP[c] for c in reversed(x))


class Designer:
    def __init__(self, seed: int, rna: bool):
        self.rnd = random.Random(seed)
        self.rna = rna

    def helix(self, k: int) -> str:
        return "".join(self.rnd.choice("GC") for _ in range(k))

    def hairpin(self, arm: int = 6, loop: int = 4) -> str:
        x = self.helix(arm)
        return x + "A" * loop + rc(x)

    def nested(self, depth: int, arm: int = 6, branches: int = 3) -> str:
        """A multiloop closed by an `arm`-bp helix around `branches` branches, the first of which is again
        such a multiloop, `depth` levels down; the others are hairpins."""
        x = self.helix(arm)
        kids = [self.nested(depth - 1, arm, branches) if depth > 1 and b == 0 else self.hairpin(arm) for b in range(branches)]
        return x + "A" + "A".join(kids) + "AA" + rc(x)

    def comb(self, k: int, arm: int = 6, close: int = 10) -> str:
        """One `close`-bp helix around k hairpins side by side."""
        x = self.helix(close)
        return x + "A" + "A".join(self.hairpin(arm) for _ in range(k)) + "A" + rc(x)

    def fit(self, core: str, n: int) -> str:
        """core centred in an A background of n nt; an RNA item gets one U in the background."""
        assert len(core) + 2 <= n, (len(core), n)
        left = (n - len(core)) // 2
        pad_l, pad_r = "A" * left, "A" * (n - len(core) - left)
        if self.rna:
            pad_l = "U" + pad_l[1:]
        return pad_l + core + pad_r

    def edge(self, core: str, n: int, arm: int = 8) -> str:
        """An `arm`-bp helix whose outer pair is (0, n - 1) around core."""
        x = self.helix(arm)
        return x + self.fit(core, n - 2 * arm) + rc(x)


LENGTHS = (200, 511, 512, 700, 1000, 1023, 1024)


def long_items(rna: bool) -> dict:
    """The structured long items of one kind, by name."""
    d = Designer(1000 + rna, rna)
    return {
        "comb_200": d.fit(d.comb(8), 200),
        "nested5_511": d.fit(d.nested(5), 511),
        "edge_512": d.edge(d.nested(4), 512),
        "comb_700": d.fit(d.comb(12), 700),
        "nested6_1000": d.fit(d.nested(6), 1000),
        "edge_1023": d.edge(d.comb(10), 1023),
        "edge_1024": d.edge(d.nested(4), 1024),
    }


def branch_heavy() -> str:
    """Seven nested 3-way multiloops in 367 nt of DNA (264 G/C): of the designs tried, the one whose MFE
    structure leaves the most branches pending in the traceback (10).  No design tried gave an MFE
    multiloop of more than 3 branches (a multibranch takes its branches from two W cells, and a branch that
    is itself a multibranch is replaced by its own branches), so the depth comes from nesting, not width."""
    d = Designer(2, False)
    core = d.nested(7)
    return d.fit(core, len(core) + 4)


def gc(s: str) -> int:
    return sum(c in "GCgc" for c in s)
