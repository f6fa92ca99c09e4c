"""CPU tier of the clone limit tests: the C oracle (oracle/clone_oracle.c) against an independent Python
restatement of CutWithEnzyme on caller-defined enzymes and the part families of clone_limits_cases (the
oracle's palindromic, negative-skip, tie and extreme-skip paths had been checked against nothing), the
generators' own claims, the deferred-hash ligation on the new reaction families, and the mirrors' refusal
of Skip / OverheadLength values that do not fit pg_clone_enzyme's int32."""
from __future__ import annotations

import pytest

import clone_limits_cases as cl
import clone_oracle as co

BSAI = co.BASE_ENZYMES["BsaI"]


def agree(parts, circ, enzymes, directionals=(False, True)):
    """Asserts restatement == oracle on every item; returns the traces of the restatement."""
    traces = []
    for i, (p, c) in enumerate(zip(parts, circ)):
        for e in enzymes:
            for d in directionals:
                t = {}
                want = co.cut(p, c, d, e)
                got = cl.cut(p, c, d, e, t)
                assert got == want, (i, p[:80], c, d, e)
                t.update(status=got[0], n=len(got[1]), directional=d, circular=c, enzyme=e)
                traces.append(t)
    return traces


def test_panel_library_matches_oracle():
    parts, circ, _ = cl.panel_library(600, seed=1)
    traces = agree(parts, circ, list(cl.PANEL.values()))
    pal = [t for t in traces if t["palindromic"] and t["n"]]
    assert len(pal) > 100 and {t["status"] for t in traces} == {cl.OK, cl.PANIC, cl.UNSUPPORTED}
    assert {t["branch"] for t in traces} >= {"single_forward", "single_reverse", "circular_one", "pairwise_all", "pairwise_directional"}


def test_panel_library_plants_sit_where_meant():
    parts, circ, plants = cl.panel_library(600, seed=1)
    n = 0
    for p, c, here in zip(parts, circ, plants):
        for pos, site in here:
            assert ((p + p).upper() if c or pos + len(site) > len(p) else p.upper())[pos: pos + len(site)] == site
            n += 1
    assert n > 1000 and any(pos + len(site) > len(p) for p, here in zip(parts, plants) for pos, site in here)


@pytest.mark.parametrize("fl,rl", cl.SWEEP_PAIRS)
def test_site_length_sweep_matches_oracle(fl, rl):
    enzyme, parts, circ, _ = cl.sweep_parts(fl, rl, seed=fl * 100 + rl)
    traces = agree(parts, circ, [enzyme])
    assert sum(t["n"] for t in traces) > 100


@pytest.mark.parametrize("fl,rl", cl.SWEEP_PAIRS)
def test_site_length_sweep_generator(fl, rl):
    enzyme, parts, circ, starts = cl.sweep_parts(fl, rl, seed=fl * 100 + rl)
    fsite, rsite = enzyme[0], enzyme[1]
    assert (len(fsite), len(rsite)) == (fl, rl) and not cl.is_palindromic(enzyme[4])
    for p, c, (f, r) in zip(parts, circ, starts):
        assert set(cl.occurrences(p, c, fsite)) == f and set(cl.occurrences(p, c, rsite)) == r, (p, c)
    fwd = [s for (f, _), c in zip(starts, circ) for s in f]
    rev = [s for (_, r), c in zip(starts, circ) for s in r]
    for got in (fwd, rev):
        assert {s % 64 for s in got} == set(range(64)) and {s % 32 for s in got} == set(range(32))
    # a match that ends at the end of a linear part; one a byte short; each split across the origin
    ends = [(p, f, r) for p, c, (f, r) in zip(parts, circ, starts) if not c and (len(p) - fl in f or len(p) - rl in r) and len(p) > 40]
    assert len(ends) >= 2
    for site in (fsite, rsite):
        splits = {len(p) - s for p, c, st in zip(parts, circ, starts) if c for s in st[site is rsite] if s < len(p) < s + len(site)}
        assert splits == set(range(1, len(site)))


def test_self_overlapping_sites_match_oracle():
    n_frag = 0
    for site, enzymes, parts, circ in cl.periodic_parts(seed=3):
        runs = {len(p) for p in parts}
        assert len(runs) > 1
        traces = agree(parts, circ, enzymes)
        n_frag += sum(t["n"] for t in traces)
    assert n_frag > 1000


def test_ties_match_oracle():
    ties = 0
    for enzyme, parts, circ in cl.tie_parts(seed=4):
        traces = agree(parts, circ, [enzyme])
        ties += sum(t["ties"] for t in traces)
        # the forward overhang of a tied pair sorts first, so the only forward -> reverse pieces are the empty
        # ones inside each pair: a directional cut keeps nothing.  Reverse-first would keep site-to-site pieces.
        assert all(t["n"] == 0 and t["status"] == cl.OK for t in traces if t["directional"])
        assert any(t["n"] for t in traces if not t["directional"])
    assert ties > 50


def test_skip_and_overhang_extremes_match_oracle():
    parts, circ = cl.skip_ohl_parts(seed=5)
    traces = agree(parts, circ, cl.skip_ohl_enzymes())
    statuses = {t["status"] for t in traces}
    branches = {(t["branch"], t["status"]) for t in traces}
    assert statuses == {cl.OK, cl.PANIC}
    for b in ("single_forward", "single_reverse", "circular_one", "pairwise_all", "pairwise_directional"):
        assert (b, cl.OK) in branches and (b, cl.PANIC) in branches, b
    assert any(t["short"] for t in traces) and sum(t["n"] for t in traces) > 500


def test_recognition_site_corners_match_oracle():
    parts, circ, _ = cl.panel_library(150, seed=6)
    enzymes = cl.recognition_enzymes()
    traces = agree(parts, circ, enzymes)
    pal = {e[4]: cl.is_palindromic(e[4]) for e in enzymes}
    assert pal == {b"": True, b"GASTC": True, b"GAWTC": True, b"GANTC": True, b"GAATC": False, b"gaattc": True, b"GGTCTC": False,
                   b"GAUTC": False, b"UA": False, b"ZZ": False, b"GAATTC": True}
    # a lower-case forward site never matches the upper-cased part
    assert all(not t["overhangs"] or not any(o[1] for o in t["overhangs"]) for t in traces if t["enzyme"][0] == b"gaattc")


def test_many_matches_match_oracle():
    parts, circ, enzyme = cl.many_matches_parts(seed=7, L=20000)
    traces = agree(parts, circ, [enzyme], directionals=(False,))
    assert len(traces[0]["overhangs"]) > 30000 and traces[1]["n"] > 1000


def test_palindromic_reverse_overhang_quirk():
    # With a palindromic enzyme only forward overhang positions exist, so a fragment's ReverseOverhang is the
    # OH bytes before the next cut -- here TTTG, not the enzyme's AATT.  It looks wrong; it is the reference.
    part = b"CCCCTTTTGAATTCAAAACCCCGGGGTTTTGAATTCAAAACCCC"
    want = (b"CAAAACCCCGGGGT", b"AATT", b"TTTG")
    for d in (False, True):
        assert co.cut(part, False, d, cl.PANEL["EcoRI"]) == (co.OK, [want])
        assert cl.cut(part, False, d, cl.PANEL["EcoRI"]) == (co.OK, [want])


def test_oracle_takes_skips_past_int32():
    """The C oracle takes int64 skips: with Skip = 2^32 + 1, BsaI's sites cut nowhere on a linear part and
    panic on a circular one, where an int32 that wrapped to 1 would cut like BsaI."""
    part = b"A" * 20 + b"GGTCTC" + b"A" * 30
    wide = BSAI[:2] + (2**32 + 1,) + BSAI[3:]
    assert co.cut(part, False, False, wide) == cl.cut(part, False, False, wide) == (co.OK, [])
    assert co.cut(part, True, False, wide)[0] == cl.cut(part, True, False, wide)[0] == co.PANIC
    assert len(co.cut(part, False, False, BSAI)[1]) == 2


def test_mirror_refuses_skip_and_overhang_outside_int32():
    from poly_b200 import clone

    for skip, ohl in ((1 << 31, 4), (-(1 << 31) - 1, 4), ((1 << 32) + 1, 4), (1, 1 << 31), (1, -(1 << 31) - 1), (1, 1 << 40)):
        with pytest.raises(clone.UnsupportedError, match="int32"):
            clone.Enzyme("Wide", "GGTCTC", "GAGACC", skip, ohl, "GGTCTC")
    for v in ((1 << 31) - 1, -(1 << 31), -((1 << 31) - 1), 0):
        e = clone.Enzyme("Edge", "GGTCTC", "GAGACC", v, v, "GGTCTC")
        arr, _ = clone._enzymes([e])
        assert (arr[0].skip, arr[0].overhang_length) == (v, v)


def test_ligation_reactions_deferred_matches_eager():
    reactions = cl.ligation_reactions(1500, seed=8)
    total = dict.fromkeys(("forward", "reverse", "palindrome_guard", "clones", "loops", "dropped", "empty_key"), 0)
    for frags in reactions:
        assert co.ligate_deferred(frags) == co.circular_ligate(frags)
        for k, v in cl.ligation_paths(frags).items():
            total[k] += v
    assert all(v > 20 for v in total.values()), total
    assert co.circular_ligate(reactions[-1]) == ([b"AATTAXXA"], [])


def test_golden_gate_libraries_for_other_enzymes():
    parts, want = cl.type_iis_library(cl.PANEL["SapI"], 3, 3, 60, 200, seed=9)
    rc, clones, _ = co.golden_gate(parts, cl.PANEL["SapI"])
    assert rc == co.OK and len(clones) == want == 27
    clones = loops = 0
    for seed in range(40):
        rc, c, l = co.golden_gate(cl.palindromic_library(cl.PANEL["EcoRI"], 4, 40, seed), cl.PANEL["EcoRI"])
        assert rc == co.OK
        clones += len(c)
        loops += len(l)
    assert clones > 20 and loops > 5
