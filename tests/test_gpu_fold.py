"""GPU tier for fold: pg_fold_zuker_batch against the C restatement (oracle/fold_oracle.c), bit for bit:
MFE float64 bits, dot-bracket bytes and status on every item."""
import os
import random
import subprocess

import numpy as np
import pytest

import fold_oracle as fo
from poly_b200 import _lib, fold

pytestmark = pytest.mark.gpu


def revcomp(s: str, rna: bool) -> str:
    m = {"A": "U" if rna else "T", "C": "G", "G": "C", "T": "A", "U": "A"}
    return "".join(m[c] for c in reversed(s))


def run(seqs, temp):
    raw = [s.encode("latin-1") if isinstance(s, str) else bytes(s) for s in seqs]
    off = np.zeros(len(raw) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    flat = np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8)
    mfe, db, dbl, st = fold.zuker_arrays(flat, off, temp)
    return raw, off, mfe, db, dbl, st


def check(seqs, temp=37.0):
    raw, off, mfe, db, dbl, st = run(seqs, temp)
    w_mfe, w_db, w_st = fo.fold_batch(raw, temp, threads=min(16, os.cpu_count() or 1))
    for i, r in enumerate(raw):
        assert int(st[i]) == int(w_st[i]), (r, int(st[i]), int(w_st[i]))
        if st[i] == fold.ITEM_OK:
            got = db[int(off[i]): int(off[i]) + int(dbl[i])].tobytes()
            assert np.float64(mfe[i]).tobytes() == np.float64(w_mfe[i]).tobytes(), (r, mfe[i], w_mfe[i])
            assert got == w_db[i], (r, got, w_db[i])


PINS = ["GGGAGGTCGTTACATCTGGGTAACACCGGTACTGATCCGGTGACCTCCC",
        "GGGAGGTCGCTCCAGCTGGGAGGAGCGTTGGGGGTATATACCCCCAACACCGGTACTGATCCGGTGACCTCCC", "CGCAGGGAUACCCGCG",
        "TAGCTCAGCTGGGAGAGCGCCTGCTTTGCACGCAGGAGGT", "GGGGGCATAGCTCAGCTGGGAGAGCGCCTGCTTTGCACGCAGGAGGTCTGCGGTTCGATCCCGCGCGCTCCCACCA",
        "TGAGACGGAAGGGGATGATTGTCCCCTTCCGTCTCA", "ACCCCCTCCTTCCTTGGATCAAGGGGCTCAA", "ACCCCCUCCUUCCUUGGAUCAAGGGGCUCAA",
        "AAGGGGUUGGUCGCCUCGACUAAGCGGCUUGGAAUUCC", "UUGGAGUACACAACCUGUACACUCUUUC", "AGGGAAAAUCCC", "GCUUACGAGCAAGUUAAGCAAC",
        "UGGGAGGUCGUCUAACGGUAGGACGGCGGACUCUGGAUCCGCUGGUGGAGGUUCGAGUCCUCCCCUCCCAGCCA",
        "GGGCGAUGAGGCCCGCCCAAACUGCCCUGAAAAGGGCUGAUGGCCUCUACUG",
        "GGGGGCAUAGCUCAGCUGGGAGAGCGCCUGCUUUGCACGCAGGAGGUCUGCGGUUCGAUCCCGCGCGCUCCCACCA", "ATGGATTTAGATAGAT", "GCUCAGCUGGGAGAGC",
        "CCUGCUUUGCACGCAGG", "GCGGUUCGAUCCCGC", "ACCCCCATCCTTCCTTGAGTCAAGGGGCTCAA", "ACCCGCAAGCCCTCCTTCCTTGGATCAAGGGGCTCAA", "CUUUGCACG",
        "ATGGATTTAGATAGATADFQ#(RSDOFIA)", "XYZ"]


def test_reference_pins():
    check(PINS)
    res, err = fold.Zuker("ACCCCCUCCUUCCUUGGAUCAAGGGGCUCAA", 37.0)
    assert err is None and res.DotBracket() == ".((((.(((......)))....))))"
    res, err = fold.Zuker("ATGGATTTAGATAGATADFQ#(RSDOFIA)", 4000.0)
    assert str(err) == "error creating folding context: the sequence ATGGATTTAGATAGATADFQ#(RSDOFIA) is not RNA or DNA"


def families(n):
    rnd = random.Random(n)
    yield "A" * n
    yield "".join(rnd.choice("AC") for _ in range(n))                    # no pair at all
    yield ("AT" * n)[:n]                                                  # pairs everywhere
    yield "".join(rnd.choice("ACG") for _ in range(n))                   # A/C/G only is DNA
    yield "".join(rnd.choice("acgt") for _ in range(n))                  # lower case
    yield "".join(rnd.choice("ACGU") for _ in range(n))
    yield ("ACGN" * n)[:n]
    yield ("ACGTU" * n)[:n]
    yield "".join(rnd.choice("ACGT") for _ in range(max(n - 1, 0))) + ("\xe9" if n else "")
    yield "".join(rnd.choice("ATATGC") for _ in range(n))                # isolated pairs


def test_every_length_0_to_40():
    check([s for n in range(41) for s in families(n)])


@pytest.mark.parametrize("temp", [0.0, 37.0, 60.0, 95.0])
def test_random_dna_rna(temp):
    rnd = random.Random(int(temp))
    seqs = []
    for _ in range(48):
        n = rnd.randint(5, 150)
        seqs.append("".join(rnd.choice("ACGT" if rnd.random() < 0.5 else "ACGU") for _ in range(n)))
    check(seqs, temp)


def hairpins(rna):
    rnd = random.Random(7 + rna)
    al = "ACGU" if rna else "ACGT"
    rs = lambda k: "".join(rnd.choice(al) for _ in range(k))
    out = []
    for _ in range(12):
        x, y, z = rs(rnd.randint(4, 9)), rs(rnd.randint(4, 9)), rs(rnd.randint(4, 9))
        loop = lambda: rs(rnd.randint(3, 8))
        out.append(x + loop() + revcomp(x, rna))                                                   # one hairpin
        out.append(rs(2) + x + loop() + revcomp(x, rna) + rs(3) + y + loop() + revcomp(y, rna) + rs(2))  # tandem
        out.append(z + rs(2) + x + loop() + revcomp(x, rna) + rs(2) + y + loop() + revcomp(y, rna) + rs(1) + revcomp(z, rna))  # nested
    return out


def test_hairpin_constructions():
    check(hairpins(False) + hairpins(True))


def test_long_and_over_cap():
    rnd = random.Random(400)
    x = "".join(rnd.choice("ACGT") for _ in range(60))
    long = "".join(rnd.choice("ACGT") for _ in range(130)) + x + "GAAA" + revcomp(x, False) + "".join(rnd.choice("ACGT") for _ in range(146))
    assert len(long) == 400
    check([long])
    over = "ACGT" * 257  # 1028 nt
    raw, off, mfe, db, dbl, st = run([over, "GGGGAAAACCCC"], 37.0)
    assert list(st) == [fold.ITEM_UNSUPPORTED, fold.ITEM_OK]
    res = fold.ZukerBatch([over], 37.0)[0]
    assert res[0] is None and isinstance(res[1], fold.UnsupportedError)


def test_1024_nt():
    # the longest supported items; A-rich so that only a few G-C pairs close, which keeps the restatement fast
    rnd = random.Random(1024)
    items = []
    for rna in (False, True):
        x, y = "".join(rnd.choice("GC") for _ in range(8)), "".join(rnd.choice("GC") for _ in range(6))
        body = "A" * 200 + x + "AAAA" + revcomp(x, rna) + "A" * 300 + y + "AAAAA" + revcomp(y, rna) + "A" * 300
        items.append(body + "A" * (1024 - len(body)))
    items.append("A" * 1024)
    assert all(len(s) == 1024 for s in items)
    check(items)


def test_error_items_leave_dots():
    seqs = ["ACGN", "", "ACGT\xe9", "ACGT" * 257]
    raw, off, mfe, db, dbl, st = run(seqs, 37.0)
    assert list(dbl) == [0, 0, 0, 0] and db[: int(off[-1])].tobytes() == b"." * int(off[-1])


def test_cpp_mirror_fold_tests(tmp_path):
    rnd = random.Random(5)
    rows = []
    for temp in (37.0, 60.0):
        seqs = PINS + hairpins(False)[:6] + hairpins(True)[:6] + ["AC", "ACGT", "A" * 10, "acgtacgtaacgt", "ACGN"]
        seqs += ["".join(rnd.choice("ACGU") for _ in range(rnd.randint(5, 90))) for _ in range(10)]
        mfe, dbs, st = fo.fold_batch([s.encode() for s in seqs], temp)
        rows += [f"{s}\t{temp!r}\t{int(c)}\t{float(m).hex()}\t{d.decode()}\n" for s, m, d, c in zip(seqs, mfe, dbs, st)]
    tsv = tmp_path / "fold_expected.tsv"
    tsv.write_text("".join(rows))
    exe = tmp_path / "fold_tests"
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-o", str(exe), os.path.join(root, "hostcpp", "fold_tests.cpp"),
                           "-L" + os.path.join(root, "poly_b200", "lib"), "-lpolyb200", "-Wl,-rpath," + os.path.join(root, "poly_b200", "lib")])
    out = subprocess.run([str(exe), str(tsv)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "fold_tests: all passed" in out.stdout


def test_mixed_batch_with_errors():
    seqs = ["GGGAGGTCGTTACATCTGGGTAACACCGGTACTGATCCGGTGACCTCCC", "", "ACGN", "A", "acgu" * 5, "ACGT\xe9ACGT", "AC", "GCGCAAAAGCGC" * 3]
    check(seqs)
    out = fold.ZukerBatch(seqs, 37.0)
    assert isinstance(out[1][1], _lib.GoPanic) and isinstance(out[3][1], _lib.GoPanic)
    assert "is not RNA or DNA" in str(out[2][1]) and out[2][0].MinimumFreeEnergy() == float("inf")
    assert out[0][1] is None and out[0][0].DotBracket() == "((((((((.((((......))))..((((.......)))).))))))))"
    with pytest.raises(_lib.GoPanic):
        fold.Zuker("", 37.0)


def test_n0_and_decreasing_offsets():
    L = _lib.lib()
    z = np.zeros(4, dtype=np.uint8)
    off = np.zeros(1, dtype=np.uint64)
    mfe, dbl, st = np.zeros(1), np.zeros(1, dtype=np.uint64), np.zeros(1, dtype=np.int32)
    assert L.pg_fold_zuker_batch(z.ctypes.data, off.ctypes.data, 0, 37.0, mfe.ctypes.data, z.ctypes.data, dbl.ctypes.data, st.ctypes.data) == _lib.PG_OK
    bad = np.array([0, 3, 2], dtype=np.uint64)
    mfe2, dbl2, st2 = np.zeros(2), np.zeros(2, dtype=np.uint64), np.zeros(2, dtype=np.int32)
    assert L.pg_fold_zuker_batch(z.ctypes.data, bad.ctypes.data, 2, 37.0, mfe2.ctypes.data, z.ctypes.data, dbl2.ctypes.data,
                                 st2.ctypes.data) == _lib.PG_ERR_ARG


def test_several_groups(monkeypatch):
    rnd = random.Random(11)
    seqs = ["".join(rnd.choice("ACGT") for _ in range(rnd.randint(20, 60))) for _ in range(64)] + ["", "ACGN"]
    rnd.shuffle(seqs)
    monkeypatch.setenv("PG_GROUP_BYTES", str(300_000))  # a few items per group
    check(seqs)
