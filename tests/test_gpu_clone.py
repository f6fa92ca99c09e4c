"""GPU tier: clone digests and Golden Gate assemblies, bit-exact against the clone oracle (oracle/clone_oracle.c)."""
from __future__ import annotations

import ctypes as C
import json
import os
import random
import subprocess

import numpy as np
import pytest

import clone_oracle as co
import clone_util
import seqhash_oracle

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIX = json.load(open(os.path.join(ROOT, "tests", "golden", "clone", "clone_fixtures.json")))
BSAI, BSAI_RC = "GGTCTCAATGC", "ATGCAGAGACC"


@pytest.fixture(scope="module")
def clone():
    from poly_b200 import _lib, clone

    _lib.check(_lib.lib().pg_init(0))
    return clone


def frag_tuples(frags):
    return [(f.Sequence.encode("latin-1"), f.ForwardOverhang.encode("latin-1"), f.ReverseOverhang.encode("latin-1")) for f in frags]


def gg_parts(clone, pairs):
    return [clone.Part(s.decode("latin-1") if isinstance(s, bytes) else s, c) for s, c in pairs]


def test_digest_pins(clone):
    em = clone.NewEnzymeManager(clone.GetBaseRestrictionEnzymes())
    part = clone.Part("ATATATA" + BSAI_RC + BSAI + "ATGCATCGATCGACTAGCATG" + BSAI_RC + BSAI[:8], False)
    assert [f.Sequence for f in em.CutWithEnzymeByName(part, True, "BsaI")] == ["ATGCATCGATCGACTAGCATG"]
    part.Circular = True
    assert [f.Sequence for f in em.CutWithEnzymeByName(part, True, "BsaI")] == ["ATGCATCGATCGACTAGCATG", "TATA"]
    part = clone.Part("ATATATATATATATAT" + BSAI + "GCGCGCGCGCGCGCGCGCGC", False)
    assert [f.Sequence for f in em.CutWithEnzymeByName(part, False, "BsaI")] == ["GCGCGCGCGCGCGCGCGCGC", "ATATATATATATATATGGTCTCA"]
    part.Circular = True
    assert [f.Sequence for f in em.CutWithEnzymeByName(part, False, "BsaI")] == ["GCGCGCGCGCGCGCGCGCGCATATATATATATATATGGTCTCA"]
    popen = clone.Part(FIX["popen"], True)
    got = em.CutWithEnzymeByName(popen, False, "BbsI")
    assert len(got) == 2 and frag_tuples(got) == co.cut(FIX["popen"].encode(), True, False, "BbsI")[1]
    seq = "AGCTGCTGTTTAAAGCTATTACTTTGAGACC"
    f = clone.CutWithEnzyme(clone.Part(seq, False), False, em.GetEnzymeByName("BsaI"))
    assert [(x.ForwardOverhang, x.ReverseOverhang) for x in f] == [("", "ACTT"), ("ACTT", "")]
    assert f[0].Sequence + f[0].ReverseOverhang + f[1].Sequence == seq
    s, c = FIX["tests"]["TestCircularCutRegression"]["plasmid1"]
    assert len(em.CutWithEnzymeByName(clone.Part(s, c), True, "BsaI")) == 1
    with pytest.raises(clone.EnzymeNotFound, match="Enzyme EcoFake not found"):
        em.CutWithEnzymeByName(popen, True, "EcoFake")


def test_digest_panics_and_unsupported(clone):
    from poly_b200 import _lib

    bsai = clone.NewEnzymeManager(clone.GetBaseRestrictionEnzymes()).GetEnzymeByName("BsaI")
    with pytest.raises(_lib.GoPanic):
        clone.CutWithEnzyme(clone.Part("GAGACC" + "A" * 30, False), False, bsai)
    with pytest.raises(clone.UnsupportedError):
        clone.CutWithEnzyme(clone.Part("ACGTé" + "GGTCTC" + "A" * 20, False), True, bsai)
    with pytest.raises(clone.UnsupportedError):
        clone.Enzyme("EcoRI-ish", "GA.TTC", "GAATTC", 0, 4, "GAATTC")
    frags = clone.CutWithEnzyme(clone.Part("A" * 20 + "GCGATGCGATG" + "T" * 40, False), False, clone.GetBaseRestrictionEnzymes()[2])
    assert frag_tuples(frags) == co.cut(b"A" * 20 + b"GCGATGCGATG" + b"T" * 40, False, False, "BtgZI")[1] and len(frags) == 2


@pytest.mark.parametrize("directional", [True, False])
def test_digest_library(clone, directional):
    parts, circ = clone_util.digest_library(12000, seed=11 + directional)
    enzymes = clone.GetBaseRestrictionEnzymes()
    got, st = clone.CutWithEnzymeBatch([clone.Part(p.decode("latin-1"), c) for p, c in zip(parts, circ)], directional, enzymes)
    seen = set()
    for i, (p, c) in enumerate(zip(parts, circ)):
        for e, enz in enumerate(enzymes):
            rc, want = co.cut(p, c, directional, enz.Name)
            assert st[i][e] == rc, (i, e)
            assert frag_tuples(got[i][e]) == want, (i, e)
            seen.add(rc)
    # a directional cut only slices between a forward and a later reverse overhang, which stays in range
    assert seen == ({co.OK, co.UNSUPPORTED} if directional else {co.OK, co.PANIC, co.UNSUPPORTED})
    assert sum(len(f) for row in got for f in row) > 5000


def test_golden_gate_pins(clone):
    em = clone.NewEnzymeManager(clone.GetBaseRestrictionEnzymes())
    bbsi = em.GetEnzymeByName("BbsI")
    popen = clone.Part(FIX["popen"], True)
    clones, loops = clone.CircularLigate([clone.Fragment("AAAAAA", "GTTG", "CTAT"), clone.Fragment("AAAAAA", "CAAC", "ATAG")])
    assert (len(clones), len(loops)) == (1, 0)
    for test in ("TestSignalKilledGoldenGate", "TestPanicGoldenGate"):
        parts = [popen] + [clone.Part(s, c) for s, c in FIX["tests"][test].values()]
        clones, loops = clone.GoldenGate(parts, bbsi)
        _, wc, wl = co.golden_gate([(p.Sequence.encode(), p.Circular) for p in parts], "BbsI")
        assert ([c.encode() for c in clones], [l.encode() for l in loops]) == (wc, wl)
        if test == "TestSignalKilledGoldenGate":
            assert (len(clones), len(loops)) == (1, 4)
    parts = [clone.Part(s, c) for s, c in FIX["example"].values()] + [popen]
    clones, _ = clone.GoldenGate(parts, bbsi)
    assert seqhash_oracle.rotate_sequence(clones[0].encode()) == FIX["example_output"].encode()


def test_golden_gate_combinatorial_library(clone):
    parts, want = clone_util.combinatorial_library(4, 8, 300, 1200, seed=5)
    _, wc, wl = co.golden_gate(parts, "BsaI")
    assert len(wc) == want == 4096
    bsai = clone.GetBaseRestrictionEnzymes()[0]
    old = os.environ.get("PG_GROUP_BYTES")
    for budget in (None, str(3 << 20)):  # one group, then many groups across the emits
        if budget:
            os.environ["PG_GROUP_BYTES"] = budget
        try:
            (clones, loops, cd, ld), = clone.GoldenGateBatch([gg_parts(clone, parts)], bsai, digests=True)
        finally:
            if old is None:
                os.environ.pop("PG_GROUP_BYTES", None)
            else:
                os.environ["PG_GROUP_BYTES"] = old
        assert [c.encode() for c in clones] == wc and [l.encode() for l in loops] == wl
        for k in range(0, len(clones), 97):
            assert seqhash_oracle.seqhash(wc[k], "DNA", True, True)[1] == cd[k]
        for k in range(len(loops)):
            assert seqhash_oracle.seqhash(wl[k], "DNA", False, True)[1] == ld[k]


def test_golden_gate_many_small_reactions(clone):
    rng = random.Random(3)
    reactions, want = [], []
    for r in range(1200):
        parts, _ = clone_util.combinatorial_library(rng.randint(1, 3), rng.randint(1, 3), rng.randint(10, 80), rng.randint(10, 60), seed=r)
        if rng.random() < 0.2:  # shuffled, a circular variant, a reused part
            parts = [(p, c or rng.random() < 0.3) for p, c in parts] + [parts[rng.randrange(len(parts))]]
            rng.shuffle(parts)
        if r == 7:
            parts = parts + [(b"ACGT\xc3\xa9" + b"GGTCTCA" + b"ACGT" * 8, False)]  # unsupported: a byte >= 0x80
        reactions.append(parts)
        want.append(co.golden_gate(parts, "BsaI"))
    from poly_b200 import _lib

    bsai = clone.GetBaseRestrictionEnzymes()[0]
    ok = [r for r in range(len(reactions)) if want[r][0] == co.OK]
    got = clone.GoldenGateBatch([gg_parts(clone, reactions[r]) for r in ok], bsai)
    for g, r in zip(got, ok):
        assert ([c.encode() for c in g[0]], [l.encode() for l in g[1]]) == (want[r][1], want[r][2]), r
    assert sum(len(g[0]) for g in got) > 1000 and len(ok) >= 1000
    bad = [r for r in range(len(reactions)) if want[r][0] != co.OK]
    assert bad == [7]
    for r in bad:
        with pytest.raises((_lib.GoPanic, clone.UnsupportedError)):
            clone.GoldenGate(gg_parts(clone, reactions[r]), bsai)


def test_golden_gate_byte_cap(clone):
    from poly_b200 import _lib

    parts, _ = clone_util.combinatorial_library(3, 3, 100, 200, seed=9)
    seqs = [p for p, _ in parts]
    off = np.zeros(len(parts) + 1, np.uint64)
    off[1:] = np.cumsum([len(s) for s in seqs])
    data = np.frombuffer(b"".join(seqs), np.uint8)
    circ = np.array([c for _, c in parts], np.uint8)
    roff = np.array([0, len(parts)], np.uint64)
    enz, keep = clone._enzymes([clone.GetBaseRestrictionEnzymes()[0]])
    L = _lib.lib()
    nb, nc = C.c_uint64(), C.c_uint64()

    def run(bcap, ccap):
        out, coff = np.zeros(max(bcap, 1), np.uint8), np.zeros(ccap + 1, np.uint64)
        kinds, counts, st = np.zeros(max(ccap, 1), np.uint8), np.zeros(2, np.uint64), np.zeros(1, np.int32)
        launches = L.pg_launch_count()
        rc = L.pg_clone_golden_gate_batch(_lib.ptr(data), _lib.ptr(off), _lib.ptr(circ), len(parts), _lib.ptr(roff), 1, C.cast(enz, C.c_void_p),
                                          bcap, ccap, _lib.ptr(out), _lib.ptr(coff), _lib.ptr(kinds), None, _lib.ptr(counts), _lib.ptr(st),
                                          C.byref(nb), C.byref(nc))
        return rc, L.pg_launch_count() - launches, out, coff, counts

    rc, launched, *_ = run(1000, 4)
    assert rc == _lib.PG_ERR_ARG and nb.value > 1000 and nc.value > 4
    need_b, need_c = nb.value, nc.value
    rc, launched_ok, out, coff, counts = run(need_b, need_c)
    assert rc == _lib.PG_OK and (nb.value, nc.value) == (need_b, need_c) and launched_ok > launched
    _, wc, wl = co.golden_gate(parts, "BsaI")
    got = [out[coff[k]: coff[k + 1]].tobytes() for k in range(int(counts.sum()))]
    assert sorted(got) == sorted(wc + wl) and int(counts[0]) == len(wc) == 27


def test_cpp_mirror_clone_tests(tmp_path):
    lines = [("popen", "popen", True, FIX["popen"])]
    for group in ("TestSignalKilledGoldenGate", "TestPanicGoldenGate", "TestCircularCutRegression"):
        lines += [(group, name, c, s) for name, (s, c) in FIX["tests"][group].items()]
    lines += [("example", name, c, s) for name, (s, c) in FIX["example"].items()]
    lines.append(("example_output", "output", False, FIX["example_output"]))
    tsv = tmp_path / "clone_fixtures.tsv"
    tsv.write_text("".join(f"{g}\t{n}\t{int(c)}\t{s}\n" for g, n, c, s in lines))
    exe = tmp_path / "clone_tests"
    hostcpp = os.path.join(ROOT, "hostcpp")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-o", str(exe), os.path.join(hostcpp, "clone_tests.cpp"),
                           "-L" + os.path.join(ROOT, "poly_b200", "lib"), "-lpolyb200", "-Wl,-rpath," + os.path.join(ROOT, "poly_b200", "lib")])
    out = subprocess.run([str(exe), str(tsv)], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "clone_tests: all passed" in out.stdout


def test_circular_ligate_refuses_non_ascii_fragments(clone):
    from poly_b200 import _lib

    # strings.ToUpper maps U+017F to S, so the reference hashes this construct; the library does not guess
    for bad in (clone.Fragment("AAAA\u017f", "GTTG", "GTTG"), clone.Fragment("AAAAAA", "GT\u212aG", "GTTG")):
        launches = _lib.lib().pg_launch_count()
        with pytest.raises(clone.UnsupportedError):
            clone.CircularLigate([clone.Fragment("AAAAAA", "GTTG", "CTAT"), bad])
        assert _lib.lib().pg_launch_count() == launches


def test_digest_batch_limits_checked_before_launch(clone):
    from poly_b200 import _lib

    L = _lib.lib()
    enz, keep = clone._enzymes(clone.GetBaseRestrictionEnzymes())
    off = np.zeros(2, np.uint64)
    z = C.c_uint64()
    launches = L.pg_launch_count()
    # n_parts x n_enzymes past 2^64: refused before the offsets are read
    rc = L.pg_clone_digest_batch(None, _lib.ptr(off), _lib.ptr(np.zeros(1, np.uint8)), 1 << 63, C.cast(enz, C.c_void_p), 3, 1,
                                 _lib.ptr(np.zeros(1, np.uint32)), None, None, 0, _lib.ptr(off), None, 0, _lib.ptr(off), 0,
                                 C.byref(z), C.byref(z), C.byref(z))
    assert rc == _lib.PG_ERR_ARG and L.pg_launch_count() == launches


def test_digest_more_items_than_one_grid_pass(clone):
    """2.7e8 (part, enzyme) items: more than one thread per item of the capped launch grids, so the per-item
    kernels must stride.  Empty parts, with BsaI sites in the last three."""
    import torch

    from poly_b200 import _lib

    n_parts, n_enz = 9_000_000, 30
    if torch.cuda.mem_get_info()[0] < 60 << 30:
        pytest.skip("needs 60 GiB of free device memory")
    tail = [b"GGTCTCAACGTACGTACGTACGTAGAGACC", b"AAGGTCTCATTTTCCCCGGGGAAAAGAGACCAA", b"GGTCTCA" + b"C" * 20]
    data = np.frombuffer(b"".join(tail), np.uint8)
    off = np.zeros(n_parts + 1, np.uint64)
    off[-len(tail):] = np.cumsum([len(t) for t in tail])
    circ = np.zeros(n_parts, np.uint8)
    circ[-1] = 1
    enz, keep = clone._enzymes([clone.GetBaseRestrictionEnzymes()[0]] * n_enz)
    n_items = n_parts * n_enz
    assert n_items > (1 << 28)
    cnt, st = np.zeros(n_items, np.uint32), np.zeros(n_items, np.int32)
    sb, so, ob, oo = np.zeros(4096, np.uint8), np.zeros(1025, np.uint64), np.zeros(4096, np.uint8), np.zeros(2049, np.uint64)
    nf, ns, no = C.c_uint64(), C.c_uint64(), C.c_uint64()
    rc = _lib.lib().pg_clone_digest_batch(_lib.ptr(data), _lib.ptr(off), _lib.ptr(circ), n_parts, C.cast(enz, C.c_void_p), n_enz, 1,
                                          _lib.ptr(cnt), _lib.ptr(st), _lib.ptr(sb), 4096, _lib.ptr(so), _lib.ptr(ob), 4096, _lib.ptr(oo), 1024,
                                          C.byref(nf), C.byref(ns), C.byref(no))
    _lib.check(rc)
    want = []
    for t, c in zip(tail, circ[-len(tail):]):
        rc_, frags = co.cut(t, bool(c), True, "BsaI")
        assert rc_ == co.OK
        want.append(frags)
    assert not cnt[: -len(tail) * n_enz].any() and not st.any()
    got_cnt = cnt[-len(tail) * n_enz:].reshape(len(tail), n_enz)
    assert (got_cnt == np.array([len(w) for w in want])[:, None]).all()
    expect = [f for w in want for _ in range(n_enz) for f in w]
    assert nf.value == len(expect) > 0
    got = [(sb[so[f]: so[f + 1]].tobytes(), ob[oo[2 * f]: oo[2 * f + 1]].tobytes(), ob[oo[2 * f + 1]: oo[2 * f + 2]].tobytes())
           for f in range(nf.value)]
    assert got == expect
