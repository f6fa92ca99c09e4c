"""The grouped sketch grown in place on the GPU (pg_mash_sketcher): after every add, rows, counts, complete and held
byte for byte against the restatement in tests/sketcher_oracle.py, and complete rows against mash.sketch_groups of
every record added so far (every row a prefix of it).  Random splits for walk and generic k, every walk k, small
budgets, a 30x read set, degenerate groups, a table overflow, rows between adds, the _dev forms, the argument rules of
a live sketcher, a FASTQ file in record-aligned chunks, and the C++ mirror."""
import ctypes as C
import gzip
import os
import subprocess
import tempfile

import numpy as np
import pytest

import sketch_groups_oracle
import sketcher_oracle
from poly_b200 import _lib, fastq, mash

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
THREADS = len(os.sched_getaffinity(0))
ACGT = np.frombuffer(b"ACGT", np.uint8)
WALK_KS = [11, 13, 15, 16, 17, 19, 21, 23, 24, 25, 27, 29, 31, 32]


def rand_seq(rng, n):
    return ACGT[rng.integers(0, 4, n)]


def random_groups(rng, k, n_groups=6, max_recs=30, max_len=3000):
    """Groups of records cut from a per-group source, so values recur; an empty group and one of records no longer
    than k."""
    groups = []
    for _ in range(n_groups):
        src = rand_seq(rng, int(rng.integers(1000, 8000)))
        recs = []
        for _ in range(int(rng.integers(1, max_recs + 1))):
            L = int(min(rng.integers(0, max_len + 1), len(src)))
            a = int(rng.integers(0, len(src) - L + 1))
            recs.append(src[a:a + L].copy())
        groups.append(recs)
    groups.insert(1, [])
    groups.insert(3, [rand_seq(rng, k), rand_seq(rng, max(k - 1, 0))])
    return groups


def random_adds(rng, groups, max_recs=12):
    """Every group's records in order, as adds (first group, [records per group]) that may begin or end inside a
    group, with empty adds and one-record adds among them."""
    flat = [(g, r) for g, recs in enumerate(groups) for r in recs]
    adds, i = [], 0
    while i < len(flat):
        n = int(rng.choice([0, 1, int(rng.integers(2, max_recs + 1))]))
        part = flat[i:i + n]
        i += n
        if not part:
            adds.append((int(rng.integers(0, len(groups))), [[]]))
            continue
        per = [[] for _ in range(part[-1][0] - part[0][0] + 1)]
        for g, r in part:
            per[g - part[0][0]].append(r)
        adds.append((part[0][0], per))
    return adds


class Pair:
    """A device sketcher and the restatement fed the same adds, and the records each group has received."""

    def __init__(self, G, k, s, m=1, B=None):
        self.dev = mash.Sketcher(G, k, s, m, B)
        self.ref = sketcher_oracle.Sketcher(G, k, s, m, self.dev.max_values)
        self.done = [[] for _ in range(G)]
        self.k, self.s, self.m = k, s, m

    def add(self, first, per):
        bases, off, goff = sketch_groups_oracle.flatten_groups(per)
        self.dev.add(bases, off, goff, first)
        self.ref.add(bases, off, goff, first, THREADS)
        for i, recs in enumerate(per):
            self.done[first + i] += recs

    def check(self, one_shot=True):
        got = self.dev.rows()
        want = self.ref.rows()
        for a, b in zip(got, want):
            assert a.tobytes() == b.tobytes()
        if one_shot:
            bases, off, goff = sketch_groups_oracle.flatten_groups(self.done)
            rows, count = mash.sketch_groups(bases, off, goff, self.k, self.s, self.m)
            for g in range(len(self.done)):
                c = int(got[1][g])
                assert c <= count[g] and got[0][g, :c].tobytes() == rows[g, :c].tobytes()
                if got[2][g]:
                    assert c == count[g] and got[0][g].tobytes() == rows[g].tobytes()
        return got


@pytest.mark.parametrize("k", [0, 11, 16, 21, 31, 33])
@pytest.mark.parametrize("s", [1, 2, 100, 1000])
def test_random_splits(gpu, k, s):
    rng = np.random.default_rng(1000 * k + s)
    groups = random_groups(rng, k)
    for m in (1, 2, 3):
        p = Pair(len(groups), k, s, m)
        for first, per in random_adds(rng, groups):
            p.add(first, per)
            rows, count, complete, held = p.check()
            if m == 1:
                assert complete.all() and (held <= s).all()
        p.dev.close()


def test_every_walk_k(gpu):
    rng = np.random.default_rng(11)
    for k in WALK_KS:
        groups = random_groups(rng, k, n_groups=3, max_recs=8, max_len=2000)
        p = Pair(len(groups), k, 50, 2)
        for first, per in random_adds(rng, groups, max_recs=6):
            p.add(first, per)
        p.check()
        p.dev.close()


def test_one_group_over_twenty_adds(gpu):
    rng = np.random.default_rng(12)
    k, s = 21, 300
    recs = random_groups(rng, k, n_groups=1, max_recs=60)[0]
    chunks = np.array_split(np.arange(len(recs)), 20)
    for m in (1, 2):
        p = Pair(3, k, s, m)
        for c in chunks:
            p.add(1, [[recs[i] for i in c]])
            p.check()
        p.dev.close()


def read_set(rng, genome, coverage=30, L=150, err=0.01):
    n = len(genome) * coverage // L
    st = rng.integers(0, len(genome) - L + 1, n)
    reads = genome[st[:, None] + np.arange(L)]
    sub = ACGT[(np.searchsorted(ACGT, reads) + rng.integers(1, 4, reads.shape)) % 4]
    return np.where(rng.random(reads.shape) < err, sub, reads)


@pytest.mark.parametrize("factor", [1, 2, 4])
def test_small_budgets(gpu, factor):
    """Read sets at 4x coverage and 3 % substitutions: most values are single error windows, so the budget binds."""
    rng = np.random.default_rng(13 + factor)
    k, s, m = 21, 100, 2
    groups = [list(read_set(rng, rand_seq(rng, 5000), coverage=4, err=0.03)) for _ in range(4)]
    p = Pair(len(groups), k, s, m, factor * s)
    for first, per in random_adds(rng, groups, max_recs=60):
        p.add(first, per)
        rows, count, complete, held = p.check()
        assert (held <= factor * s).all()
    assert not complete.all()  # the budget binds: some group ends incomplete, and still a prefix of its row
    p.dev.close()


def test_read_set_in_twenty_adds(gpu):
    rng = np.random.default_rng(14)
    k, s, m, L = 21, 1000, 2, 150
    reads = read_set(rng, rand_seq(rng, 200_000))
    p = Pair(1, k, s, m)
    for part in np.array_split(reads, 20):
        p.add(0, [list(part)])
        rows, count, complete, held = p.check(one_shot=False)
    rows, count, complete, held = p.check()
    assert complete[0] and count[0] == s and held[0] <= 64 * s
    p.dev.close()


def mm3_word(w):
    """murmur3.Sum32 of 4-byte keys (little-endian words w), seed 0."""
    M = np.uint64(0xFFFFFFFF)
    w = w.astype(np.uint64)
    rotl = lambda x, r: ((x << np.uint64(r)) | (x >> np.uint64(32 - r))) & M
    k1 = rotl((w * np.uint64(0xCC9E2D51)) & M, 15) * np.uint64(0x1B873593) & M
    h = rotl(k1, 13) * np.uint64(5) + np.uint64(0xE6546B64) & M
    h ^= np.uint64(4)
    for sh, c in ((16, 0x85EBCA6B), (13, 0xC2B2AE35)):
        h = (h ^ (h >> np.uint64(sh))) * np.uint64(c) & M
    return (h ^ (h >> np.uint64(16))).astype(np.uint32)


def test_degenerate_groups_and_overflow(gpu):
    k, s = 21, 100
    poly_a = np.full(1_000_000, ord("A"), np.uint8)
    period3 = np.tile(np.frombuffer(b"ACG", np.uint8), 5000)
    two = np.tile(np.frombuffer(b"AT", np.uint8), 5000)
    for m in (1, 3):
        p = Pair(3, k, s, m)
        p.add(0, [[poly_a[:500_000]], [period3]])
        p.add(0, [[poly_a[500_000:]], [two], [two]])
        rows, count, complete, held = p.check()
        assert list(count) == [1, 5, 2]
        p.dev.close()
    # k = 4, s = 1, m = 2: the first add's poly-A record sets a narrow first range; the second add brings 1 000
    # distinct single windows into the next range, whose table is sized from the two values seen, so it overflows
    rng = np.random.default_rng(15)
    k, s, m = 4, 1, 2
    words = rng.integers(0, 1 << 32, 1 << 22, dtype=np.uint64).astype(np.uint32)
    h = mm3_word(words)
    W = 1_000_000
    T1 = int(np.ceil((1 + 6 + 48) / W * 2.0 ** 32))
    low = np.unique(words[h < T1])[:2]
    mid = np.unique(words[(h >= T1) & (h < 65 * T1)])[:1000]
    recs = [np.frombuffer(x.tobytes() + b"C", np.uint8) for x in np.concatenate([low, mid])]
    p = Pair(2, k, s, m)
    p.add(0, [recs[:2] + [np.full(W + k, ord("A"), np.uint8)]])
    p.check()
    p.add(0, [recs[2:], [np.full(300, ord("A"), np.uint8)]])
    p.check()
    p.dev.close()


def test_rows_between_adds_change_nothing(gpu):
    rng = np.random.default_rng(16)
    k, s, m = 21, 200, 2
    groups = random_groups(rng, k)
    adds = random_adds(rng, groups)
    a, b = mash.Sketcher(len(groups), k, s, m), mash.Sketcher(len(groups), k, s, m)
    for first, per in adds:
        bases, off, goff = sketch_groups_oracle.flatten_groups(per)
        a.add(bases, off, goff, first)
        b.add(bases, off, goff, first)
        r1, r2 = a.rows(), a.rows()
        assert all(x.tobytes() == y.tobytes() for x, y in zip(r1, r2))
        a.rows(2, 3)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a.rows(), b.rows()))
    assert [m_.Sketches.tobytes() for m_ in a.sketches()] == [r.tobytes() for r in b.rows()[0]]
    a.close()
    b.close()


def test_dev_forms_and_row_stride(gpu):
    import torch

    rng = np.random.default_rng(17)
    k, s, m = 21, 150, 2
    groups = random_groups(rng, k)
    adds = random_adds(rng, groups)
    host, dev = mash.Sketcher(len(groups), k, s, m), mash.Sketcher(len(groups), k, s, m)
    d = torch.device("cuda", 0)
    for first, per in adds:
        bases, off, goff = sketch_groups_oracle.flatten_groups(per)
        host.add(bases, off, goff, first)
        dev.add(torch.from_numpy(bases).to(d), torch.from_numpy(off.view(np.int64)).to(d), torch.from_numpy(goff.view(np.int64)).to(d), first)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(host.rows(), dev.rows()))
    G, stride = len(groups), s + 37
    rows, count, complete, held = host.rows()
    d_out = torch.full((G, stride), 0x5A5A, dtype=torch.int32, device=d)
    d_n = torch.zeros(G, dtype=torch.int32, device=d)
    d_c = torch.zeros(G, dtype=torch.uint8, device=d)
    d_h = torch.zeros(G, dtype=torch.int64, device=d)
    st = torch.cuda.current_stream(d).cuda_stream
    _lib.check(_lib.lib().pg_mash_sketcher_rows_dev(dev._h, 0, G, d_out.data_ptr(), stride, d_n.data_ptr(), d_c.data_ptr(), d_h.data_ptr(), st))
    out = d_out.cpu().numpy().view(np.uint32)
    assert out[:, :s].tobytes() == rows.tobytes() and not out[:, s:].any()
    assert d_n.cpu().numpy().view(np.uint32).tobytes() == count.tobytes()
    assert d_c.cpu().numpy().astype(bool).tobytes() == complete.tobytes()
    assert d_h.cpu().numpy().view(np.uint64).tobytes() == held.tobytes()
    out = np.full((G - 1, stride), 0x5A5A, np.uint32)
    n = np.zeros(G - 1, np.uint32)
    _lib.check(_lib.lib().pg_mash_sketcher_rows(host._h, 1, G - 1, out.ctypes.data, stride, n.ctypes.data, None, None))
    assert out[:, :s].tobytes() == rows[1:].tobytes() and not out[:, s:].any() and n.tobytes() == count[1:].tobytes()
    host.close()
    dev.close()


def test_live_rules_in_order(gpu):
    L = _lib.lib()
    ARG = _lib.PG_ERR_ARG
    k, s = 21, 10
    sk = mash.Sketcher(3, k, s, 2)
    h = sk._h
    b = np.frombuffer(b"ACGTACGTACGTACGTACGTACGTACGTACGTAC", np.uint8).copy()
    off = np.array([0, 20, 34], np.uint64)
    goff = np.array([0, 1, 2], np.uint64)
    sk.add(b, off, goff, 1)
    before = sk.rows()
    for dev in (False, True):
        add = (lambda *a: L.pg_mash_sketcher_add_dev(*a, None)) if dev else L.pg_mash_sketcher_add
        assert add(h, None, None, 0, None, 7, 0) == _lib.PG_OK  # nothing to add: no rule applies
        assert add(h, None, None, 0, None, 2, 2) == ARG and "groups [2" in _lib.last_error()
        assert add(h, None, None, 0, None, 1 << 63, 1 << 63) == ARG
        assert add(h, None, None, 0, None, 1, 2) == _lib.PG_OK  # no records: a no-op
        assert add(h, b.ctypes.data, None, 2, goff.ctypes.data, 1, 2) == ARG and "null buffer" in _lib.last_error()
        assert add(h, b.ctypes.data, off.ctypes.data, 2, None, 1, 2) == ARG and "null buffer" in _lib.last_error()
        assert add(h, None, off.ctypes.data, 2, goff.ctypes.data, 1, 2) == ARG and "null buffer" in _lib.last_error()
    empty = np.array([0, 0, 0], np.uint64)  # records with no byte: bases may be null in the host add
    assert L.pg_mash_sketcher_add(h, None, empty.ctypes.data, 2, goff.ctypes.data, 0, 2) == _lib.PG_OK
    for bad in ([0, 1], [1, 2], [0, 3], [0, 2, 1]):
        g = np.array(bad, np.uint64)
        assert L.pg_mash_sketcher_add(h, b.ctypes.data, off.ctypes.data, 2, g.ctypes.data, 0, len(g) - 1) == ARG, bad
    dec = np.array([0, 30, 20], np.uint64)
    assert L.pg_mash_sketcher_add(h, b.ctypes.data, dec.ctypes.data, 2, goff.ctypes.data, 1, 2) == ARG and "decrease" in _lib.last_error()
    assert L.pg_mash_sketcher_add(h, b.ctypes.data, dec.ctypes.data, 2, np.array([0, 1], np.uint64).ctypes.data, 1, 1) == ARG
    assert "group offsets" in _lib.last_error()  # the partition is checked before the record offsets
    after = sk.rows()
    assert all(x.tobytes() == y.tobytes() for x, y in zip(before, after))
    out, n = np.zeros(3 * s, np.uint32), np.zeros(3, np.uint32)
    for dev in (False, True):
        rows = (lambda *a: L.pg_mash_sketcher_rows_dev(*a, None)) if dev else L.pg_mash_sketcher_rows
        assert rows(h, 2, 2, None, 0, None, None, None) == ARG and "rows [2" in _lib.last_error()
        assert rows(h, 0, 3, None, s - 1, None, None, None) == ARG and "row_stride" in _lib.last_error()
        assert rows(h, 0, 3, None, s, n.ctypes.data, None, None) == ARG and "null out" in _lib.last_error()
        assert rows(h, 0, 3, out.ctypes.data if not dev else 1, s, None, None, None) == ARG and "null out" in _lib.last_error()
        assert rows(h, 3, 0, None, s, None, None, None) == _lib.PG_OK
    sk.close()


def test_fastq_in_record_aligned_chunks(gpu):
    import torch

    text = gzip.open(os.path.join(ROOT, "tests", "golden", "fastq", "nanosavseq.fastq.gz")).read()
    lines = text.split(b"\n")
    n_rec = len(lines) // 4
    cuts = np.linspace(0, n_rec, 5).astype(int)
    k, s = 15, 200
    d = torch.device("cuda", 0)
    L = _lib.lib()
    for m in (1, 2):
        sk = mash.Sketcher(1, k, s, m)
        for a, b in zip(cuts[:-1], cuts[1:]):
            chunk = b"\n".join(lines[4 * a:4 * b]) + b"\n"
            d_text = torch.from_numpy(np.frombuffer(chunk, np.uint8).copy()).to(d)
            d_bases = torch.zeros(len(chunk), dtype=torch.uint8, device=d)
            d_off = torch.zeros(b - a + 2, dtype=torch.int64, device=d)
            nr, tot, ec, el = C.c_uint64(), C.c_uint64(), C.c_int32(), C.c_uint64()
            st = torch.cuda.current_stream(d).cuda_stream
            _lib.check(L.pg_fastq_ingest_dev(d_text.data_ptr(), len(chunk), d_bases.data_ptr(), len(chunk), d_off.data_ptr(), b - a + 1,
                                             C.byref(nr), C.byref(tot), C.byref(ec), C.byref(el), st))
            assert ec.value == 0 and nr.value == b - a
            goff = torch.tensor([0, nr.value], dtype=torch.int64, device=d)
            sk.add(d_bases, d_off[:nr.value + 1], goff)
        bases, off, err = fastq.ingest(text)
        assert err is None and len(off) - 1 == n_rec
        want = mash.sketch_groups(bases, off, np.array([0, n_rec], np.uint64), k, s, m)
        rows, count, complete, held = sk.rows()
        c = int(count[0])
        assert rows[0, :c].tobytes() == want[0][0, :c].tobytes()
        if m == 1:
            assert complete[0]
        if complete[0]:
            assert rows.tobytes() == want[0].tobytes() and count.tobytes() == want[1].tobytes()
        sk.close()


def test_cpp_mirror(gpu):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "sketcher_tests"])
    rng = np.random.default_rng(18)
    k, s, m = 21, 300, 2
    groups = [g for g in random_groups(rng, k) if g]
    with tempfile.TemporaryDirectory() as td:
        txt = os.path.join(td, "groups.txt")
        with open(txt, "wb") as f:  # one record per line, "g record"; records with no byte are left out
            for g, recs in enumerate(groups):
                f.write(b"".join(b"%d " % g + bytes(r) + b"\n" for r in recs if len(r)))
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "sketcher_tests"), txt, str(len(groups)), str(k), str(s), str(m)],
                             capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: sketcher tests pass"
    bases, off, goff = sketch_groups_oracle.flatten_groups([[r for r in g if len(r)] for g in groups])
    rows, count = sketch_groups_oracle.sketch_groups(bases, off, goff, k, s, m, THREADS)
    assert len(lines) == len(groups) + 1
    for g, line in enumerate(lines[:-1]):
        vals = [int(x) for x in line.split()]
        assert vals[0] == count[g] and vals[1:] == [int(v) for v in rows[g, :count[g]]]
