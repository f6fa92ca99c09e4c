"""GPU tier of the clone limit tests: digests and ligations with caller-defined enzymes, bit-exact against the
clone oracle (oracle/clone_oracle.c) -- status, fragment count and the bytes of every fragment; constructs in
order.  The enzymes and part families (clone_limits_cases) reach the kernel paths the built-in Type IIS
enzymes never do: palindromic sites (no reverse walk, every overhang pair fragmented), sites of 1..32 bytes
matching at every offset of the walk's 32-position steps, self-overlapping sites whose greedy matches carry
across steps, forward/reverse ties, extreme skips and overhang lengths, and ligations with reverse attaches,
palindrome guards, loops and failed hashes.  The file runs in about 15 s of wall time on an H100 80GB HBM3
at a 700 W power limit."""
from __future__ import annotations

import ctypes as C

import numpy as np
import pytest

import clone_limits_cases as cl
import clone_oracle as co
import seqhash_oracle

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def clone():
    from poly_b200 import _lib, clone

    _lib.check(_lib.lib().pg_init(0))
    return clone


def enzyme(clone, e, name="custom"):
    return clone.Enzyme(name, e[0].decode("latin-1"), e[1].decode("latin-1"), e[2], e[3], e[4].decode("latin-1"))


def frag_tuples(frags):
    return [(f.Sequence.encode("latin-1"), f.ForwardOverhang.encode("latin-1"), f.ReverseOverhang.encode("latin-1")) for f in frags]


def digest_matches_oracle(clone, parts, circ, enzymes, directional):
    """One CutWithEnzymeBatch of every part x enzyme, checked item by item; returns [(status, n_frags)]."""
    got, st = clone.CutWithEnzymeBatch([clone.Part(p.decode("latin-1"), c) for p, c in zip(parts, circ)], directional,
                                       [enzyme(clone, e) for e in enzymes])
    out = []
    for i, (p, c) in enumerate(zip(parts, circ)):
        for k, e in enumerate(enzymes):
            rc, want = co.cut(p, c, directional, e)
            assert st[i][k] == rc and frag_tuples(got[i][k]) == want, (i, p[:80], c, directional, e)
            out.append((rc, len(want)))
    return out


def raw_digest(clone, parts, circ, enzymes, directional, caps=None):
    """pg_clone_digest_batch called directly: (rc, frag_count, status, fragments, totals, launches)."""
    from poly_b200 import _lib

    L = _lib.lib()
    data = np.frombuffer(b"".join(parts) or b"\0", np.uint8)
    off = np.zeros(len(parts) + 1, np.uint64)
    np.cumsum([len(p) for p in parts], out=off[1:])
    cv = np.array(circ, np.uint8)
    enz, keep = clone._enzymes([enzyme(clone, e) for e in enzymes])
    n = len(parts) * len(enzymes)
    cnt, st = np.zeros(n, np.uint32), np.zeros(n, np.int32)
    nf, ns, no = C.c_uint64(), C.c_uint64(), C.c_uint64()

    def call(fcap, scap, ocap):
        sb, so = np.zeros(max(scap, 1), np.uint8), np.zeros(fcap + 1, np.uint64)
        ob, oo = np.zeros(max(ocap, 1), np.uint8), np.zeros(2 * fcap + 1, np.uint64)
        before = L.pg_launch_count()
        rc = L.pg_clone_digest_batch(_lib.ptr(data), _lib.ptr(off), _lib.ptr(cv), len(parts), C.cast(enz, C.c_void_p), len(enzymes),
                                     int(directional), _lib.ptr(cnt), _lib.ptr(st), _lib.ptr(sb), scap, _lib.ptr(so), _lib.ptr(ob), ocap,
                                     _lib.ptr(oo), fcap, C.byref(nf), C.byref(ns), C.byref(no))
        return rc, L.pg_launch_count() - before, (sb, so, ob, oo)

    rc, launched, bufs = call(*(caps or (0, 0, 0)))
    if caps is None and rc == _lib.PG_ERR_ARG:
        rc, launched, bufs = call(nf.value, ns.value, no.value)
    sb, so, ob, oo = bufs
    frags = []
    if rc in (_lib.PG_OK, _lib.PG_ERR_PANIC, _lib.PG_ERR_UNSUPPORTED):  # written; per-item codes say why an item has none
        frags = [(sb[so[f]: so[f + 1]].tobytes(), ob[oo[2 * f]: oo[2 * f + 1]].tobytes(), ob[oo[2 * f + 1]: oo[2 * f + 2]].tobytes())
                 for f in range(nf.value)]
    del keep
    return rc, cnt.copy(), st.copy(), frags, (nf.value, ns.value, no.value), launched


@pytest.mark.parametrize("directional", [False, True])
def test_panel_library(clone, directional):
    """Every panel enzyme in one call, so items of different enzymes share each launch."""
    parts, circ, _ = cl.panel_library(3000, seed=21 + directional)
    res = digest_matches_oracle(clone, parts, circ, list(cl.PANEL.values()), directional)
    ne = len(cl.PANEL)
    pal = [i for i, e in enumerate(cl.PANEL.values()) if cl.is_palindromic(e[4])]
    assert sum(1 for j, (rc, n) in enumerate(res) if j % ne in pal and rc == co.OK and n) > 300  # palindromic items with fragments
    # a directional cut only slices forward -> reverse pieces, which stay in range for these enzymes
    assert {rc for rc, _ in res} == ({co.OK, co.UNSUPPORTED} if directional else {co.OK, co.PANIC, co.UNSUPPORTED})
    # a byte >= 0x80 makes the part unsupported for every enzyme
    for i, p in enumerate(parts):
        if any(b >= 0x80 for b in p):
            assert [rc for rc, _ in res[i * ne: (i + 1) * ne]] == [co.UNSUPPORTED] * ne


def test_palindromic_reverse_overhang_quirk(clone):
    # With a palindromic enzyme only forward overhang positions exist, so a fragment's ReverseOverhang is the
    # OH bytes before the next cut (TTTG), not the enzyme's overhang (AATT).  It looks wrong; it is the
    # reference's answer, and the library reproduces it.
    part = "CCCCTTTTGAATTCAAAACCCCGGGGTTTTGAATTCAAAACCCC"
    for d in (False, True):
        got = clone.CutWithEnzyme(clone.Part(part, False), d, enzyme(clone, cl.PANEL["EcoRI"], "EcoRI"))
        assert frag_tuples(got) == [(b"CAAAACCCCGGGGT", b"AATT", b"TTTG")]


@pytest.mark.parametrize("fl,rl", cl.SWEEP_PAIRS)
def test_site_length_sweep(clone, fl, rl):
    e, parts, circ, starts = cl.sweep_parts(fl, rl, seed=fl * 100 + rl)
    for got in ([s for f, _ in starts for s in f], [s for _, r in starts for s in r]):  # the coverage the sweep claims
        assert {s % 64 for s in got} == set(range(64))
    n = 0
    for d in (False, True):
        n += sum(k for _, k in digest_matches_oracle(clone, parts, circ, [e], d))
    assert n > 100


def test_site_of_33_bytes_is_refused_before_launch(clone):
    from poly_b200 import _lib

    L = _lib.lib()
    site = b"ACGTTGCAAC" * 3 + b"GTA"
    part = np.frombuffer(b"T" * 10 + site + b"T" * 10, np.uint8)
    off = np.array([0, part.size], np.uint64)
    z = C.c_uint64()
    for f, r in ((site, b"GAGACC"), (b"GGTCTC", site)):
        enz = (clone._Enzyme * 1)(clone._Enzyme(f, len(f), r, len(r), b"GGTCTC", 6, 1, 4))
        before = L.pg_launch_count()
        rc = L.pg_clone_digest_batch(_lib.ptr(part), _lib.ptr(off), _lib.ptr(np.zeros(1, np.uint8)), 1, C.cast(enz, C.c_void_p), 1, 0,
                                     _lib.ptr(np.zeros(1, np.uint32)), _lib.ptr(np.zeros(1, np.int32)), None, 0,
                                     _lib.ptr(np.zeros(1, np.uint64)), None, 0, _lib.ptr(np.zeros(1, np.uint64)), 0, C.byref(z), C.byref(z),
                                     C.byref(z))
        assert rc == _lib.PG_ERR_UNSUPPORTED and L.pg_launch_count() == before
    with pytest.raises(clone.UnsupportedError):
        clone.Enzyme("Long", site.decode(), "GAGACC", 1, 4, "GGTCTC")


def test_self_overlapping_sites(clone):
    n = 0
    for site, enzymes, parts, circ in cl.periodic_parts(seed=3):
        for d in (False, True):
            n += sum(k for _, k in digest_matches_oracle(clone, parts, circ, enzymes, d))
    assert n > 1000


def test_ties(clone):
    ties = 0
    for e, parts, circ in cl.tie_parts(seed=4):
        for p, c in zip(parts, circ):
            t = {}
            cl.cut(p, c, False, e, t)
            ties += t["ties"]
        directed = digest_matches_oracle(clone, parts, circ, [e], True)
        assert all(r == (co.OK, 0) for r in directed)  # forward first on a tie: no forward -> reverse piece
        assert any(k for _, k in digest_matches_oracle(clone, parts, circ, [e], False))
    assert ties > 50


def test_skip_and_overhang_extremes(clone):
    """Every skip x overhang length of the grid in one call: statuses include PG_ITEM_PANIC and the call
    returns PG_ERR_PANIC after writing every other item's fragments."""
    from poly_b200 import _lib

    parts, circ = cl.skip_ohl_parts(seed=5)
    enzymes = cl.skip_ohl_enzymes()
    for d in (False, True):
        res = digest_matches_oracle(clone, parts, circ, enzymes, d)
        assert {rc for rc, _ in res} == {co.OK, co.PANIC} and sum(k for _, k in res) > 100
        rc, cnt, st, frags, _, _ = raw_digest(clone, parts, circ, enzymes, d)
        assert rc == _lib.PG_ERR_PANIC
        want = [co.cut(p, c, d, e) for p, c in zip(parts, circ) for e in enzymes]
        assert st.tolist() == [w[0] for w in want] and cnt.tolist() == [len(w[1]) for w in want]
        assert frags == [f for w in want for f in w[1]]


def test_recognition_site_corners(clone):
    parts, circ, _ = cl.panel_library(400, seed=6)
    parts += [b"", b"GAATTC", b"gaattc" * 3, b"GAA\x00TTCGAATTC\x01GAATTC", bytes(range(1, 32)) + b"GAATTCAAAAAAAAAAGAATTC"]
    circ += [False, True, True, False, True]
    for d in (False, True):
        res = digest_matches_oracle(clone, parts, circ, cl.recognition_enzymes(), d)
        assert sum(k for _, k in res) > 500


def test_lengths_around_each_site_length(clone):
    """Parts of every length 0 .. m + 1 against sites of every sweep length at once."""
    enzymes, parts, circ = [], [], []
    for fl, rl in cl.SWEEP_PAIRS:
        e, p, c, _ = cl.sweep_parts(fl, rl, seed=fl * 100 + rl)
        enzymes.append(e)
        short = [(x, y) for x, y in zip(p, c) if len(x) <= max(fl, rl) + 1]
        parts += [x for x, _ in short]
        circ += [y for _, y in short]
    for d in (False, True):
        digest_matches_oracle(clone, parts, circ, enzymes, d)


def test_many_matches_in_one_item(clone):
    """A 1-byte site on circular parts of 3 Mbp: millions of match starts, and hundreds of thousands of
    fragments, in single items."""
    from poly_b200 import _lib

    parts, circ, e = cl.many_matches_parts(seed=7)
    rc, cnt, st, frags, _, _ = raw_digest(clone, parts, circ, [e], False)
    assert rc == _lib.PG_OK
    want = [co.cut(p, c, False, e) for p, c in zip(parts, circ)]
    assert st.tolist() == [w[0] for w in want] and cnt.tolist() == [len(w[1]) for w in want]
    assert frags == [f for w in want for f in w[1]]
    assert 2 * parts[0].count(b"A") > 4_000_000 and len(frags) > 200_000  # each A of the doubled part is a start


def test_digest_capacity_rule(clone):
    """Too small an output: PG_ERR_ARG with the totals, frag_count and status written, and no copy kernel;
    then the exact totals suffice."""
    from poly_b200 import _lib

    parts, circ, _ = cl.panel_library(200, seed=9)
    enzymes = list(cl.PANEL.values())
    rc, cnt, st, _, need, launched_small = raw_digest(clone, parts, circ, enzymes, True, caps=(1, 1, 1))
    assert rc == _lib.PG_ERR_ARG and need[0] > 1
    rc2, cnt2, st2, frags, need2, launched = raw_digest(clone, parts, circ, enzymes, True, caps=need)
    assert rc2 in (_lib.PG_OK, _lib.PG_ERR_UNSUPPORTED) and need2 == need and (cnt2 == cnt).all() and (st2 == st).all()
    assert launched > launched_small
    want = [co.cut(p, c, True, e) for p, c in zip(parts, circ) for e in enzymes]
    assert frags == [f for w in want for f in w[1]]


def test_skip_past_int32_is_refused(clone):
    """Skip = 2^32 + 1 once wrapped to 1 in the mirror's int32 field, so the enzyme digested like BsaI; the
    reference (and the oracle, which takes int64) cuts nothing on this linear part."""
    from poly_b200 import _lib

    part = b"A" * 20 + b"GGTCTC" + b"A" * 30
    want = co.cut(part, False, False, (b"GGTCTC", b"GAGACC", 2**32 + 1, 4, b"GGTCTC"))
    assert want == (co.OK, [])
    before = _lib.lib().pg_launch_count()
    with pytest.raises(clone.UnsupportedError):
        clone.CutWithEnzyme(clone.Part(part.decode(), False), False, clone.Enzyme("BsaI+2^32", "GGTCTC", "GAGACC", 2**32 + 1, 4, "GGTCTC"))
    assert _lib.lib().pg_launch_count() == before
    # the int32 edges are accepted and digest as the oracle does
    edges = [(b"GGTCTC", b"GAGACC", s, o, b"GGTCTC") for s in (cl.I32_MIN, cl.I32_MAX) for o in (cl.I32_MIN, cl.I32_MAX, 4)]
    digest_matches_oracle(clone, [part, part], [False, True], edges, False)


def test_circular_ligate_reactions(clone, monkeypatch):
    reactions = cl.ligation_reactions(3000, seed=8)
    total = dict.fromkeys(("forward", "reverse", "palindrome_guard", "clones", "loops", "dropped", "empty_key"), 0)
    want = []
    for frags in reactions:
        want.append(co.circular_ligate(frags))
        for k, v in cl.ligation_paths(frags).items():
            total[k] += v
    assert all(v > 20 for v in total.values()), total
    as_frags = [[clone.Fragment(*(x.decode("latin-1") for x in f)) for f in r] for r in reactions]
    got = clone.CircularLigateBatch(as_frags, digests=True)
    for r, ((c, l, cd, ld), (wc, wl)) in enumerate(zip(got, want)):
        assert ([x.encode("latin-1") for x in c], [x.encode("latin-1") for x in l]) == (wc, wl), r
        if r % 50 == 0:
            for x, dg in zip(wc, cd):
                assert seqhash_oracle.seqhash(x, "DNA", True, True)[1] in (dg, None)
            for x, dg in zip(wl, ld):
                assert seqhash_oracle.seqhash(x, "DNA", False, True)[1] in (dg, None)
    assert want[-1] == ([b"AATTAXXA"], [])
    # the same reactions with a small group budget, so the emits span many groups
    monkeypatch.setenv("PG_GROUP_BYTES", "4096")
    again = clone.CircularLigateBatch(as_frags[:600])
    assert [([x.encode("latin-1") for x in c], [x.encode("latin-1") for x in l]) for c, l in again] == want[:600]


def test_golden_gate_other_enzymes(clone):
    sapi = cl.PANEL["SapI"]
    reactions, want = [], []
    for seed in range(60):
        parts, n = cl.type_iis_library(sapi, 1 + seed % 3, 1 + seed % 4, 40 + seed, 80, seed=seed)
        reactions.append(parts)
        want.append(co.golden_gate(parts, sapi))
        assert want[-1][0] == co.OK and len(want[-1][1]) == n
    got = clone.GoldenGateBatch([[clone.Part(p.decode(), c) for p, c in r] for r in reactions], enzyme(clone, sapi, "SapI"))
    assert [([x.encode() for x in c], [x.encode() for x in l]) for c, l in got] == [(w[1], w[2]) for w in want]

    eco = cl.PANEL["EcoRI"]
    reactions = [cl.palindromic_library(eco, 4, 40, seed) for seed in range(200)]
    want = [co.golden_gate(r, eco) for r in reactions]
    assert all(w[0] == co.OK for w in want)
    got = clone.GoldenGateBatch([[clone.Part(p.decode(), c) for p, c in r] for r in reactions], enzyme(clone, eco, "EcoRI"))
    assert [([x.encode() for x in c], [x.encode() for x in l]) for c, l in got] == [(w[1], w[2]) for w in want]
    assert sum(len(w[1]) for w in want) > 100 and sum(len(w[2]) for w in want) > 20
