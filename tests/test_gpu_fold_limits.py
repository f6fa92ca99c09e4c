"""GPU tier for fold at its limits: structure-rich items up to 1 024 nt, temperatures at and past the ends
of float64, exact ties between candidate structures, and batches that mix every length class.  Each item is
checked against the C restatement (oracle/fold_oracle.c) as in test_gpu_fold.check: status, MFE float64
bits and dot-bracket bytes.  Where the restatement's MFE is NaN only NaN is required: Go does not specify a
NaN's sign or payload."""
import math
import os
import random

import numpy as np
import pytest

import fold_designs as fd
import fold_oracle as fo
from poly_b200 import fold

pytestmark = pytest.mark.gpu

_ORACLE = {}  # (item, temp bits) -> (status, mfe, dot-bracket): the long items are folded once per session


def oracle(raw, temp):
    key = lambda r: (r, np.float64(temp).tobytes())
    todo = [r for r in dict.fromkeys(raw) if key(r) not in _ORACLE]
    if todo:
        mfe, db, st = fo.fold_batch(todo, temp, threads=os.cpu_count() or 1)
        for r, m, d, s in zip(todo, mfe, db, st):
            _ORACLE[key(r)] = (int(s), float(m), d)
    return [_ORACLE[key(r)] for r in raw]


def run(raw, temp):
    off = np.zeros(len(raw) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    flat = np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8)
    mfe, db, dbl, st = fold.zuker_arrays(flat, off, temp)
    return [(int(st[i]), float(mfe[i]), db[int(off[i]): int(off[i]) + int(dbl[i])].tobytes()) for i in range(len(raw))]


def same(got, want, item):
    assert got[0] == want[0], (item, got[0], want[0])
    if got[0] == fold.ITEM_OK:
        if math.isnan(want[1]):
            assert math.isnan(got[1]), (item, got[1])
        else:
            assert np.float64(got[1]).tobytes() == np.float64(want[1]).tobytes(), (item, got[1], want[1])
        assert got[2] == want[2], (item, got[2], want[2])


def check(seqs, temp=37.0):
    # the restatement has no length limit: an item past MAX_LEN is the library's PG_ITEM_UNSUPPORTED
    raw = [s.encode("latin-1") if isinstance(s, str) else bytes(s) for s in seqs]
    got = run(raw, temp)
    want = dict(zip((r for r in raw if len(r) <= fold.MAX_LEN), oracle([r for r in raw if len(r) <= fold.MAX_LEN], temp)))
    for r, g in zip(raw, got):
        same(g, want.get(r, (fold.ITEM_UNSUPPORTED, 0.0, b"")), r[:40])
    return got


def mixed_case(s: str, seed: int) -> str:
    rnd = random.Random(seed)
    return "".join(c.lower() if rnd.random() < 0.5 else c for c in s)


@pytest.mark.parametrize("rna", [False, True], ids=["dna", "rna"])
def test_structured_long_items(rna):
    items = fd.long_items(rna)
    assert sorted(len(s) for s in items.values()) == sorted(fd.LENGTHS)
    assert max(fd.gc(s) for s in items.values()) <= 250  # keeps the restatement near a minute
    seqs = list(items.values()) + [mixed_case(items["edge_1024"], rna)]
    got = check(seqs)
    assert all(g[0] == fold.ITEM_OK for g in got)
    for name, (st, e, db) in zip(list(items) + ["edge_1024 mixed case"], got):
        n = len(items[name.split()[0]])
        if name.startswith("edge"):  # the outer pair (0, n - 1) puts the descriptors' position fields at the top
            assert db[:1] == b"(" and len(db) == n and db[-1:] == b")", name
    assert got[-1][1:] == got[len(items) - 1][1:]  # upper-casing comes first


def test_random_200_to_300_nt():
    rnd = random.Random(250)
    seqs = ["".join(rnd.choice("ACGU" if k % 2 else "ACGT") for _ in range(rnd.randint(200, 300))) for k in range(8)]
    got = check(seqs)
    assert all(g[0] == fold.ITEM_OK for g in got)


def test_branch_heavy_item():
    # the design with the deepest traceback stack (test_oracle_fold checks it against the kernel's capacities):
    # an overfull arena slot or stack would make it PG_ITEM_FOLD_INTERNAL
    got = check([fd.branch_heavy()])
    assert got[0][0] == fold.ITEM_OK


TEMPS = [-273.15, -500.0, 1e6, 1e305, -1e305, 1e308, -1e308, math.inf, -math.inf, math.nan, 5e-324]


def trimmed_items():
    from test_gpu_fold import PINS

    out = list(PINS)
    for rna in (False, True):
        for s in fd.long_items(rna).values():
            mid = (len(s) - 150) // 2
            out.append(s[mid: mid + 150])
    return out


@pytest.mark.parametrize("temp", TEMPS, ids=repr)
def test_extreme_temperatures(temp):
    # deltaG = H - T * (S / 1000) with T = temp + 273.15: 0 K, past both ends of float64, inf * 0 = NaN for
    # every key the tables lack, and a temperature that rounds to 0 degrees C
    check(trimmed_items(), temp)


def tie_items():
    out = []
    for rna in (False, True):
        d = fd.Designer(77 + rna, rna)
        h = d.hairpin(5)
        x = d.helix(6)
        for k in (2, 3, 5):
            out.append(d.fit(("AA" + h) * k, 12 + 14 * k))                          # tandem copies of one hairpin
        out.append(d.fit(x + "AAAA" + x + "AAAA" + fd.rc(x), 40))                # two copies of x, one partner
        out.append(d.fit(x + "AAAA" + fd.rc(x) + "AAAA" + x, 40))                # one x, two partners
        out.append(d.fit(x + "AAAAA" + x + "AAAAA" + fd.rc(x) + "AAAAA" + fd.rc(x), 60))
    for k in (1, 2, 3, 4, 6):
        out.append("GCGCAAAAGCGC" * k)                                           # palindromes
        out.append("GGAUCCAAAGGAUCC" * k)
        out.append("ACGTACGT" * (2 * k))
    for k in (2, 3):
        out += ["GGGGAAACCCC" * k, "GGGGAAACCCC" * k + "A", "A" + "GGGGAAACCCC" * k]
    # items on which a V cell's interior-loop scan meets an exact tie at 37 C, so that taking the last
    # instead of the first candidate changes the MFE or the structure
    out += ["CCAGCGGGGCCGCAGAGGGCCGCGGGAACGG", "GCCACGCGGCAGGGCGCG", "GGGAAGCCCCCGCGGGGACGGCGGACCCGGGCA",
            "CCAGCCCGGCGCAAGCCCGCCGGACCCCAGGCGGGCC", "GGCCGGGAGGCGCGCCGGCGGAAGCGCGGAGCCGCCGCCC",
            "CACAGCCCGGCGGCCGCCAGCCGCGAGCCACCAAAGCG", "CCCGGCCAGCACGCGG", "CAAGGCCGGCGACCGGGGAAGGGCGGCAGGA"]
    return out


@pytest.mark.parametrize("temp", [37.0, -273.15], ids=["37C", "0K"])
def test_exact_ties(temp):
    # ties are decided by the first strict improvement in the reference's loop order; at 0 K every deltaG is H
    check(tie_items(), temp)


def fold_scratch_bytes(n):
    # fold.cu's fold_scratch_bytes: codes, V/W energies and descriptors, branch counts, the branch arena
    a8 = lambda x: (x + 7) & ~7
    arena = sum((n - d) * ((d + 1) // 5) for d in range(n))
    return a8(a8(n) + 32 * n * n + a8(2 * n * n) + 4 * arena) if 2 <= n <= fold.MAX_LEN else 0


def test_mixed_length_groups(monkeypatch):
    dna, rna = fd.long_items(False), fd.long_items(True)
    rnd = random.Random(1025)
    short = {n: "".join(rnd.choice("ACGT") for _ in range(n)) for n in (1, 2, 3, 4, 5, 150)}
    seqs = ["", short[1], "ACGN", short[2], short[3], "ACG\xe9", short[4], short[5], short[150], dna["edge_1023"], "XYZ",
            rna["edge_1024"], short[2], "", "ACGT" * 256 + "A", short[4], "acgu" * 3]
    assert sorted({len(s) for s in seqs}) == [0, 1, 2, 3, 4, 5, 12, 150, 1023, 1024, 1025]
    whole = check(seqs)
    # a budget that holds the 1 024-nt item and the tiny items after it, but not the 1 023-nt item too
    budget = fold_scratch_bytes(1024) + 2 * 1024 + 64 + 4096
    assert budget < fold_scratch_bytes(1023) + fold_scratch_bytes(1024)
    monkeypatch.setenv("PG_GROUP_BYTES", str(budget))
    grouped = check(seqs)
    for s, a, b in zip(seqs, whole, grouped):
        same(b, a, s[:40])
