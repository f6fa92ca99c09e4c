"""CPU tier for synthesis/fragment: the library's fidelity table equals tests/golden/fragment/ligation_fidelity.json
entry for entry; the C restatement (tests/fragment_oracle.c) reproduces every pin of poly's fragment_test.go
and example_test.go; and an independent Python restatement of the GPU's incremental formulation (R over the
120 keys, one pass over the keyed members per candidate) gives the oracle's bits on seeded cases."""
import os
import random
import re
import struct

import pytest

import fragment_oracle as fo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = fo.pins()


def test_library_table_equals_golden():
    text = open(os.path.join(ROOT, "poly_b200", "csrc", "fragment_fidelity.inc")).read()
    head, body = text.split("k_fidelity_keys[120][5] = ")[1].split("k_fidelity_counts[120][120] = ")
    keys = re.findall(r'"([ACGT]{4})"', head)
    rows = re.findall(r"\{([0-9, ]+)\}", body)
    counts = [[int(x) for x in r.split(",")] for r in rows]
    g = fo.fidelity()
    assert keys == g["keys"] and counts == g["counts"]
    flat = [x for r in counts for x in r]
    assert len(keys) == 120 and len(flat) == 14400 and max(flat) == 789
    assert sum(1 for i in range(120) for j in range(120) if i != j and counts[i][j]) == 1609


def test_examples():
    b = P["Example_basic"]
    st, frags, eff, _, _ = fo.fragment(b["seq"], b["min"], b["max"], b["exclude"])
    assert st == fo.OK and [f.decode() for f in frags] == b["fragments"]
    b = P["ExampleFragment"]
    st, frags, eff, _, _ = fo.fragment(b["seq"], b["min"], b["max"])
    assert st == fo.OK and frags[1].decode() == b["fragment_1"] and "%f" % eff == b["efficiency_text"]
    s = list(P["ExampleNextOverhang"]["start"])
    for _ in range(3):
        c, e = fo.next_overhangs(s)
        best, pick = 0.0, ""
        for x, v in zip(c, e):
            if v > best:
                best, pick = v, x
        s.append(pick)
    assert s == P["ExampleNextOverhang"]["output"]


def test_fragment_tests():
    for name in ("TestFragment", "TestSmallFragmentSize", "TestLongFragment"):
        b = P[name]
        st, frags, _, _, _ = fo.fragment(b["seq"], b["min"], b["max"])
        assert st == fo.OK, name
    assert all(len(f) <= 94 for f in fo.fragment(P["TestLongFragment"]["seq"], 79, 94)[1])
    assert fo.fragment(P["TestUnfragmentable"]["seq"], 40, 80)[0] == fo.NO_POSITION
    a, b = P["TestFragmentSizes"]
    assert fo.fragment(a["seq"], a["min"], a["max"])[0::3] == (fo.MIN_GT_MAX, 105)
    assert fo.fragment(b["seq"], b["min"], b["max"])[0::3] == (fo.MIN_LT_12, 7)
    b = P["TestFragmentWithOverhangs"]
    assert fo.fragment(b["seq"], b["min"], b["max"], [], b["include"])[0] == fo.OK
    assert "GTCT" not in fo.next_overhangs(P["TestCheckLongRegresssion"]["set"])[0]
    e = fo.set_efficiency(P["TestRegressionTestMatching12"]["set"])
    assert 0.965 <= e <= 1 and e == P["TestRegressionTestMatching12"]["efficiency"]


def test_quirks():
    assert fo.set_efficiency(["AAAA"]) == 1.0 and fo.set_efficiency(["AAAA", "TTTT"]) == 0.5
    assert fo.set_efficiency([]) == 1.0 and fo.set_efficiency(["AAAAA", "aaaa", "NNNN"]) == 1.0
    assert fo.fragment("ACG", 12, 30)[0] == fo.PANIC
    assert fo.fragment("ACGT\xe9ACGT", 12, 30)[0] == fo.UNSUPPORTED
    st, frags, eff, _, _ = fo.fragment("acgtacgtac", 40, 30)  # shorter than max: success before any argument check
    assert st == fo.OK and frags == [b"ACGTACGTAC"] and eff == fo.set_efficiency(["ACGT", "GTAC"])
    # the end game can push min below 12 for the next step: the error carries the adjusted values
    rnd = random.Random(3)
    found = False
    for _ in range(400):
        g = "".join(rnd.choice("ACGT") for _ in range(rnd.randint(30, 60)))
        st, _, _, emin, emax = fo.fragment(g, 12, rnd.randint(14, 40))
        if st == fo.MIN_LT_12:
            assert emin < 12
            found = True
    assert found
    assert len(fo.next_overhangs([])[0]) == 240


# ---- an independent restatement of the GPU's incremental formulation -----------------------------------------------
T = fo.fidelity()
KEY = {k: i for i, k in enumerate(T["keys"])}
MM = T["counts"]
COMP = dict(zip(b"ABCDGHKMNRSTVWYabcdghkmnrstvwy", b"TVGHCDMKNYSABWRtvghcdmknysabwr"))


def rc(s: bytes) -> bytes:
    return bytes(COMP.get(c, 0) for c in reversed(s))


def keys_of(o: bytes):
    return KEY.get(o.decode("latin-1"), -1), KEY.get(rc(o).decode("latin-1"), -1)


def add(R, o):
    kx, krx = keys_of(o)
    for k in range(120):
        R[k] += (MM[k][kx] if kx >= 0 else 0) + (MM[k][krx] if krx >= 0 else 0)
    return kx


def extend(R, keyed, x):
    """SetEfficiency(S + x) from R over S and S's keyed members in order (x None: SetEfficiency(S))"""
    kx, krx = keys_of(x) if x is not None else (-1, -1)
    e = 1.0
    for k in keyed + ([kx] if kx >= 0 else []):
        nc = MM[k][k]
        nt = R[k] + (MM[k][kx] if kx >= 0 else 0) + (MM[k][krx] if krx >= 0 else 0)
        if nt != nc:
            e = e * (nc / nt)
    return e


def incremental_fragment(seq: bytes, mn: int, mx: int, exclude, include):
    if any(c >= 0x80 for c in seq):
        return fo.UNSUPPORTED, [], 0.0, 0, 0
    seq = seq.upper()
    if len(seq) < 4:
        return fo.PANIC, [], 0.0, 0, 0
    R, keyed, words = [0] * 120, [], set()
    for o in [seq[:4], seq[-4:]] + exclude:
        k = add(R, o)
        if k >= 0:
            keyed.append(k)
        words |= {o, rc(o)}
    incw = {w for o in include for w in (o, rc(o))}
    base, ln, ends = 0, len(seq), []
    while True:
        if ln < mx:
            return fo.OK, ends + [len(seq)], extend(R, keyed, None), 0, 0
        if mn > mx:
            return fo.MIN_GT_MAX, [], 0.0, mn, mx
        if mn < 12:
            return fo.MIN_LT_12, [], 0.0, mn, mx
        if ln < 2 * mx:
            d = mx - mn
            buf = min((ln + d) // 2, mx)
            mn, mx = buf - d, buf
        best, pos = 0.0, 0
        for p in range(mx, mn - 1, -1):
            x = seq[base + p - 4: base + p]
            if x in words or (include and x not in incw) or x == rc(x):
                continue
            e = extend(R, keyed, x)
            if e > best:
                best, pos = e, p
        if pos == 0:
            return fo.NO_POSITION, [], 0.0, 0, 0
        ends.append(base + pos)
        x = seq[base + pos - 4: base + pos]
        k = add(R, x)
        if k >= 0:
            keyed.append(k)
        words |= {x, rc(x)}
        base += pos - 4
        ln -= pos - 4


def gene(rnd, n):
    al = rnd.choice(["ACGT", "ACGT", "ACGTacgt", "ACGTN", "AT", "ACGTRYKM"])
    return "".join(rnd.choice(al) for _ in range(n)).encode()


def bits(x: float) -> bytes:
    return struct.pack("<d", x)


@pytest.mark.parametrize("seed", range(5))
def test_incremental_formulation_matches_oracle(seed):
    rnd = random.Random(seed)
    pool = [b"AAAA", b"TTTT", b"GTCT", b"AGAC", b"aaaa", b"NNNN", b"ACG", b"ACGTA", b"GGGG", b"CATG", b"NACG", b"", b"TCAC", b"ATAA"]
    for _ in range(120):
        g = gene(rnd, rnd.choice([3, 10, 40, 120, 400, 900]))
        mn = rnd.choice([5, 12, 20, 40, 60])
        mx = mn + rnd.choice([-3, 0, 5, 20, 40])
        ex = [rnd.choice(pool) if rnd.random() < 0.5 else gene(random.Random(rnd.random()), 4).upper() for _ in range(rnd.randint(0, 6))]
        inc = [] if rnd.random() < 0.6 else [gene(random.Random(rnd.random()), 4).upper() for _ in range(rnd.randint(1, 60))]
        st, frags, eff, emin, emax = fo.fragment(g, mn, mx, ex, inc)
        want_ends = []
        if st == fo.OK:
            pos = 0
            for f in frags:
                want_ends.append(pos + len(f) if not want_ends else want_ends[-1] - 4 + len(f))
        got = incremental_fragment(g, mn, mx, ex, inc)
        assert got[0] == st and got[1] == want_ends and bits(got[2]) == bits(eff) and got[3:] == (emin, emax), (g, mn, mx, ex, inc)
    for _ in range(40):
        s = [rnd.choice(pool + [b"ACGT"]) if rnd.random() < 0.3 else gene(random.Random(rnd.random()), 4).upper() for _ in range(rnd.randint(0, 30))]
        R, keyed = [0] * 120, []
        for o in s:
            k = add(R, o)
            if k >= 0:
                keyed.append(k)
        assert bits(extend(R, keyed, None)) == bits(fo.set_efficiency(s))
        cands, effs = fo.next_overhangs(s)
        for c, e in zip(cands, effs):
            x = c.encode()
            assert bits((extend(R, keyed, x) + extend(R, keyed, rc(x))) / 2) == bits(e)
