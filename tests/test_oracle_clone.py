"""CPU tier: the clone oracle (oracle/clone_oracle.c) against the reference's own pins (clone/clone_test.go,
clone/example_test.go), and the deferred-hash ligation design against the oracle's eager hashing."""
from __future__ import annotations

import json
import os
import random

import pytest

import clone_oracle as co
import seqhash_oracle

FIX = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "clone", "clone_fixtures.json")))
BSAI, BSAI_RC = b"GGTCTCAATGC", b"ATGCAGAGACC"


def parts_of(test):
    return [(FIX["popen"].encode(), True)] + [(s.encode(), c) for s, c in FIX["tests"][test].values()]


def seqs(frags):
    return [f[0] for f in frags]


def test_cut_with_enzyme_pins():
    part = b"ATATATA" + BSAI_RC + BSAI + b"ATGCATCGATCGACTAGCATG" + BSAI_RC + BSAI[:8]
    assert seqs(co.cut(part, False, True, "BsaI")[1]) == [b"ATGCATCGATCGACTAGCATG"]                # test(1)
    assert seqs(co.cut(part, True, True, "BsaI")[1]) == [b"ATGCATCGATCGACTAGCATG", b"TATA"]         # test(2)
    part = b"ATATATATATATATAT" + BSAI + b"GCGCGCGCGCGCGCGCGCGC"
    assert seqs(co.cut(part, False, False, "BsaI")[1]) == [b"GCGCGCGCGCGCGCGCGCGC", b"ATATATATATATATATGGTCTCA"]  # test(3)
    assert seqs(co.cut(part, True, False, "BsaI")[1]) == [b"GCGCGCGCGCGCGCGCGCGCATATATATATATATATGGTCTCA"]     # test(4)
    rc, frags = co.cut(FIX["popen"].encode(), True, False, "BbsI")                                     # test(5)
    assert rc == co.OK and len(frags) == 2


def test_cut_with_enzyme_regression():
    seq = b"AGCTGCTGTTTAAAGCTATTACTTTGAGACC"
    rc, f = co.cut(seq, False, False, "BsaI")
    assert rc == co.OK and len(f) == 2
    assert (f[0][1], f[0][2], f[1][1], f[1][2]) == (b"", b"ACTT", b"ACTT", b"")
    assert f[0][0] + f[0][2] + f[1][0] == seq


def test_circular_ligate_pin():
    clones, loops = co.circular_ligate([(b"AAAAAA", b"GTTG", b"CTAT"), (b"AAAAAA", b"CAAC", b"ATAG")])
    assert (len(clones), len(loops)) == (1, 0)


def test_signal_killed_golden_gate_pin():
    rc, clones, loops = co.golden_gate(parts_of("TestSignalKilledGoldenGate"), "BbsI")
    assert (rc, len(clones), len(loops)) == (co.OK, 1, 4)


def test_panic_golden_gate_pin_runs():
    rc, _, _ = co.golden_gate(parts_of("TestPanicGoldenGate"), "BbsI")
    assert rc == co.OK


def test_circular_cut_regression_pin():
    seq, circ = FIX["tests"]["TestCircularCutRegression"]["plasmid1"]
    rc, frags = co.cut(seq.encode(), circ, True, "BsaI")
    assert rc == co.OK and len(frags) == 1


def test_example_golden_gate_pin():
    parts = [(s.encode(), c) for s, c in FIX["example"].values()] + [(FIX["popen"].encode(), True)]
    rc, clones, _ = co.golden_gate(parts, "BbsI")
    assert rc == co.OK
    assert seqhash_oracle.rotate_sequence(clones[0]) == FIX["example_output"].encode()


def test_btgzi_chain_is_one_match():
    # GCGATGCGATG: the second GCGATG starts inside the first, so FindAllStringIndex returns one match
    part = b"A" * 20 + b"GCGATGCGATG" + b"T" * 40
    rc, frags = co.cut(part, False, False, "BtgZI")
    assert rc == co.OK and len(frags) == 2  # a single forward cut on a linear part
    assert frags[0][1] == part[6 + 20 + 10: 6 + 20 + 14]


def test_reference_panics_are_reported():
    # a lone BsaI reverse site at position 0: overhang position 0 - 1 = -1, sequence[-1:] panics (clone.go:201)
    rc, frags = co.cut(b"GAGACC" + b"A" * 30, False, False, "BsaI")
    assert (rc, frags) == (co.PANIC, [])
    # TestPanicGoldenGate's pair of intercepting BbsI sites (GAAGACATAATGGTCTTC): the overhangs sit at 12
    # (forward) and 14 (reverse), so the only piece is sequence[12:14] = "AT", which the len > 8 filter drops
    # before the overhang slices that once panicked ([4:-2]).  Both ways the reference returns no fragment.
    for directional in (False, True):
        assert co.cut(b"AAAAGAAGACATAATGGTCTTCAAAA", False, directional, "BbsI") == (co.OK, [])
    assert co.cut(b"ACGT\xc3\xa9GGTCTCAAAAAAAAAAA", False, True, "BsaI")[0] == co.UNSUPPORTED


def test_enzyme_not_found_text():
    from poly_b200 import clone

    with pytest.raises(clone.EnzymeNotFound) as e:
        clone.NewEnzymeManager(clone.GetBaseRestrictionEnzymes()).GetEnzymeByName("EcoRFake")
    assert str(e.value) == "Enzyme EcoRFake not found"


def _deferred_equals_eager(frags):
    assert co.ligate_deferred(frags) == co.circular_ligate(frags)


@pytest.mark.parametrize("test", ["TestSignalKilledGoldenGate", "TestPanicGoldenGate"])
def test_deferred_hash_matches_eager_on_fixtures(test):
    frags = []
    for seq, circ in parts_of(test):
        frags += co.cut(seq, circ, True, "BbsI")[1]
    _deferred_equals_eager(frags)
    _deferred_equals_eager([(b"AAAAAA", b"GTTG", b"CTAT"), (b"AAAAAA", b"CAAC", b"ATAG")])


def random_reaction(rng: random.Random):
    """Fragments over a small overhang alphabet: shared, reverse-complementary and palindromic overhangs, and
    repeated sequences, so attaches in both orientations, loops and duplicate clones all occur."""
    ohs = [b"AATT", b"GCGC", b"ACGT", b"GGAC", b"GTCC", b"TTAG", b"CTAA", b"CAGT"][: rng.randint(2, 8)]
    seqs_ = [bytes(rng.choice(b"ACGT") for _ in range(rng.randint(0, 12))) for _ in range(rng.randint(1, 4))]
    return [(rng.choice(seqs_), rng.choice(ohs), rng.choice(ohs)) for _ in range(rng.randint(1, 6))]


def test_deferred_hash_matches_eager_on_random_reactions():
    rng = random.Random(20261016)
    n_clones = n_loops = dropped = 0
    for _ in range(400):
        frags = random_reaction(rng)
        _deferred_equals_eager(frags)
        c, l = co.circular_ligate(frags)
        n_clones += len(c)
        n_loops += len(l)
        dropped += sum(1 for e in co.emits(frags) if not e[1])
    assert n_clones > 100 and n_loops > 50 and dropped > 10  # every path of the enumeration was taken
