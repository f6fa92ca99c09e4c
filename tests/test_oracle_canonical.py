"""CPU tier of canonical k-mers (PG_KMER_CANONICAL): the canonical oracle against a plain-Python restatement of the
definition, its strand symmetry, and the argument rules of the new entry points, in their order, before any device
work."""
import ctypes as C

import numpy as np
import pytest

import canonical_oracle
import oracle_ffi
import sketch_groups_oracle
from poly_b200 import _lib, mash

ARG = _lib.PG_ERR_ARG
LETTERS = b"ABCDGHKMNRSTVWYabcdghkmnrstvwy"


def plain_hashes(rec: bytes, k: int):
    """The definition word for word: windows 0 .. L - k, canon(w) = min(w, rc(w)) in byte order, murmur3 of it."""
    out = []
    for p in range(len(rec) - k + 1):
        w = rec[p:p + k]
        rc = oracle_ffi.reverse_complement(w)
        out.append(oracle_ffi.murmur3_32(w if w <= rc else rc))
    return out


def ragged(recs):
    off = np.zeros(len(recs) + 1, np.uint64)
    off[1:] = np.cumsum([len(r) for r in recs])
    bases = np.frombuffer(b"".join(recs) + b"\0", np.uint8)
    return bases, off


def cases(rng):
    acgt = lambda n: bytes(rng.choice(list(b"ACGT"), n).tolist())
    return {
        "acgt": [acgt(n) for n in (40, 41, 63, 100)],
        "lower": [acgt(60).lower(), bytes(rng.choice(list(b"acgtACGT"), 57).tolist())],
        "iupac": [bytes(rng.choice(list(LETTERS), n).tolist()) for n in (50, 77)],
        "arbitrary": [bytes(rng.integers(0, 256, n, dtype=np.uint8).tolist()) for n in (45, 90)],  # unlisted bytes -> 0
        "palindrome": [b"ACGT" * 12, b"AATT" * 10 + b"A", b"GC" * 30],
        "poly": [b"A" * 50, b"T" * 50, b"A" * 25 + b"T" * 25],
    }


@pytest.mark.parametrize("k", [1, 2, 3, 4, 5, 11, 16, 21, 32, 33, 40])
def test_oracle_against_the_definition(k):
    rng = np.random.default_rng(k)
    for name, recs in cases(rng).items():
        recs = recs + [recs[0][:k], recs[0][:k - 1], b""]  # L = k (one window), L < k and L = 0 (none)
        bases, off = ragged(recs)
        got = canonical_oracle.window_hashes(bases, off, k)
        want = [h for r in recs for h in plain_hashes(r, k)]
        assert got.tolist() == want, (name, k)
        assert len(got) == sum(max(len(r) - k + 1, 0) for r in recs)


def test_complement_table_is_the_oracles():
    t = canonical_oracle.complement_table()
    assert bytes(t[list(b"ACGTacgtNn")]) == b"TGCAtgcaNn"
    assert int(t[ord("U")]) == 0 and int(t[0]) == 0 and int(t[0xFF]) == 0
    assert sorted(bytes(t[list(LETTERS)])) == sorted(LETTERS)  # the listed letters are closed under complement


def test_mash_choice_on_acgt():
    """On upper-case ACGT the chosen strand is Mash's: the forward k-mer when memcmp(fwd, rev) <= 0."""
    rng = np.random.default_rng(5)
    k = 21
    rec = bytes(rng.choice(list(b"ACGT"), 500).tolist())
    bases, off = ragged([rec])
    got = canonical_oracle.window_hashes(bases, off, k)
    comp = bytes.maketrans(b"ACGT", b"TGCA")
    for p in range(len(rec) - k + 1):
        fwd = rec[p:p + k]
        rev = fwd.translate(comp)[::-1]
        assert got[p] == oracle_ffi.murmur3_32(fwd if fwd <= rev else rev)


@pytest.mark.parametrize("k", [5, 21, 33])
def test_oracle_strand_symmetry(k):
    rng = np.random.default_rng(100 + k)
    recs = [bytes(rng.choice(list(LETTERS), int(n)).tolist()) for n in rng.integers(0, 300, 40)]
    flip = [oracle_ffi.reverse_complement(r) if i % 3 == 0 else r for i, r in enumerate(recs)]
    a = canonical_oracle.window_hashes(*ragged(recs), k)
    b = canonical_oracle.window_hashes(*ragged(flip), k)
    assert sorted(a.tolist()) == sorted(b.tolist())
    goff = np.array([0, 10, 10, 25, 40], np.uint64)
    for m in (1, 2):
        ra = canonical_oracle.sketch_groups(*ragged(recs), goff, k, 50, m)
        rb = canonical_oracle.sketch_groups(*ragged(flip), goff, k, 50, m)
        assert ra[0].tobytes() == rb[0].tobytes() and ra[1].tobytes() == rb[1].tobytes()


def test_counting_oracles_restore_the_forward_hashes():
    """The canonical counting runs the forward oracles with their hash function swapped only while they run."""
    rng = np.random.default_rng(9)
    rec = bytes(rng.choice(list(b"ACGT"), 300).tolist())
    bases, off = ragged([rec, oracle_ffi.reverse_complement(rec)])
    goff = np.array([0, 1, 2], np.uint64)
    fwd = sketch_groups_oracle.sketch_groups(bases, off, goff, 15, 400)
    can = canonical_oracle.sketch_groups(bases, off, goff, 15, 400)
    assert sketch_groups_oracle.sketch_groups(bases, off, goff, 15, 400)[0].tobytes() == fwd[0].tobytes()
    assert can[0][0].tobytes() == can[0][1].tobytes() and can[1][0] == can[1][1]
    assert fwd[0][0].tobytes() != fwd[0][1].tobytes()
    want = sorted(set(plain_hashes(rec, 15)))
    assert can[0][0, :can[1][0]].tolist() == want[:400]
    s = canonical_oracle.Sketcher(2, 15, 400)
    s.add(bases, off, goff)
    assert s.rows()[0].tobytes() == can[0].tobytes()


# ---- the argument rules of the new entry points ------------------------------------------------------------------
def groups(dev, k=21, s=10, m=1, flags=0, out=True):
    L = _lib.lib()
    b = np.frombuffer(b"ACGTACGTAC", np.uint8)
    off = np.array([0, 4, 10], np.uint64)
    goff = np.array([0, 2], np.uint64)
    o = np.zeros(s if s > 0 else 1, np.uint32)
    c = np.zeros(1, np.uint32)
    args = (b.ctypes.data, off.ctypes.data, 2, goff.ctypes.data, 1, k, s, m, flags, o.ctypes.data if out else None, max(s, 0), c.ctypes.data)
    if dev:
        return L.pg_mash_sketch_groups_flags_dev(*args, None)
    return L.pg_mash_sketch_groups_flags(*args)


@pytest.mark.parametrize("dev", [False, True])
def test_sketch_groups_flags_rules_in_order(dev):
    assert groups(dev, k=-1, s=0, m=0, flags=6, out=False) == ARG and "null out" in _lib.last_error()
    assert groups(dev, k=-1, s=0, m=0, flags=6) == ARG and "kmerSize" in _lib.last_error()
    assert groups(dev, k=0, s=0, m=0, flags=2) == ARG and "unknown k-mer flags 0x2" in _lib.last_error()
    assert groups(dev, k=0, s=0, m=0, flags=1 | 0x80000000) == ARG and "unknown k-mer flags 0x80000000" in _lib.last_error()
    assert groups(dev, k=0, s=0, m=0, flags=1) == ARG and "canonical k-mers of size 0" in _lib.last_error()
    assert groups(dev, k=1, s=0, m=0, flags=1) == ARG and "sketchSize" in _lib.last_error()
    assert groups(dev, k=0, s=0, m=0, flags=0) == ARG and "sketchSize" in _lib.last_error()  # k = 0 is fine forward
    assert groups(dev, k=1, m=0, flags=1) == ARG and "min_copies" in _lib.last_error()


def sketcher_create(k=21, s=10, m=1, B=100, flags=0, G=1, out=True):
    h = C.c_void_p()
    rc = _lib.lib().pg_mash_sketcher_create_flags(G, k, s, m, B, flags, C.byref(h) if out else None)
    assert not h.value
    return rc


def test_sketcher_create_flags_rules_in_order():
    assert sketcher_create(G=0, k=-1, s=0, flags=2, out=False) == ARG and "null sketcher pointer" in _lib.last_error()
    assert sketcher_create(G=0, k=-1, s=0, flags=2) == ARG and "groups" in _lib.last_error()
    assert sketcher_create(k=-1, s=0, flags=2) == ARG and "kmerSize" in _lib.last_error()
    assert sketcher_create(k=0, s=0, flags=2) == ARG and "unknown k-mer flags" in _lib.last_error()
    assert sketcher_create(k=0, s=0, flags=1) == ARG and "canonical k-mers of size 0" in _lib.last_error()
    assert sketcher_create(k=1, s=0, flags=1) == ARG and "sketchSize" in _lib.last_error()
    assert sketcher_create(k=1, m=0, flags=1) == ARG and "min_copies" in _lib.last_error()
    assert sketcher_create(k=1, B=5, flags=1) == ARG and "max_values" in _lib.last_error()


def screen_create(dev, k=21, s=4, n=2, samples=1, flags=0, sk=True, out=True):
    L = _lib.lib()
    rows = np.arange(64, dtype=np.uint32)  # only its pointer is passed where n x s exceeds it
    h = C.c_void_p()
    args = (rows.ctypes.data if sk else None, n, s, k, samples, flags)
    o = C.byref(h) if out else None
    rc = L.pg_mash_screen_create_flags_dev(*args, None, o) if dev else L.pg_mash_screen_create_flags(*args, o)
    assert not h.value
    return rc


@pytest.mark.parametrize("dev", [False, True])
def test_screen_create_flags_rules_in_order(dev):
    assert screen_create(dev, k=-1, s=0, samples=0, flags=2, sk=False, out=False) == ARG and "null screen pointer" in _lib.last_error()
    assert screen_create(dev, k=-1, s=0, samples=0, flags=2, sk=False) == ARG and "k-mer size" in _lib.last_error()
    assert screen_create(dev, k=0, s=0, samples=0, flags=4, sk=False) == ARG and "unknown k-mer flags" in _lib.last_error()
    assert screen_create(dev, k=0, s=0, samples=0, flags=1, sk=False) == ARG and "canonical k-mers of size 0" in _lib.last_error()
    assert screen_create(dev, k=1, s=0, samples=0, flags=1, sk=False) == _lib.PG_ERR_PANIC
    assert screen_create(dev, k=1, n=1 << 32, samples=0, flags=1, sk=False) == ARG and "2^32" in _lib.last_error()
    assert screen_create(dev, k=1, samples=0, flags=1, sk=False) == ARG and "0 samples" in _lib.last_error()
    assert screen_create(dev, k=1, flags=1, sk=False) == ARG and "null buffer" in _lib.last_error()


def test_python_mirror_rules():
    b, off, goff = np.zeros(4, np.uint8), np.array([0, 4], np.uint64), np.array([0, 1], np.uint64)
    with pytest.raises(_lib.PolyError) as e:
        mash.sketch_groups(b, off, goff, 0, 10, 1, canonical=True)
    assert e.value.code == ARG
    with pytest.raises(_lib.PolyError) as e:
        mash.Sketcher(1, 0, 10, canonical=True)
    assert e.value.code == ARG
    with pytest.raises(_lib.PolyError) as e:
        mash.Screen(np.zeros((1, 4), np.uint32), 0, canonical=True)
    assert e.value.code == ARG
