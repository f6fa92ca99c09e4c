"""GPU tier for synthesis/fragment: pg_fragment_batch, pg_fragment_set_efficiency_batch and
pg_fragment_next_overhangs_batch against the C restatement (tests/fragment_oracle.c), bit for bit: status,
fragment ends, error numbers and the float64 efficiency bytes of every item."""
import os
import random
import subprocess

import numpy as np
import pytest

import fragment_oracle as fo
from poly_b200 import _lib, fragment

pytestmark = pytest.mark.gpu
P = fo.pins()
THREADS = min(16, os.cpu_count() or 1)
STATUS = {fo.OK: fragment.ITEM_OK, fo.PANIC: fragment.ITEM_PANIC, fo.UNSUPPORTED: fragment.ITEM_UNSUPPORTED, fo.MIN_GT_MAX: fragment.ITEM_MIN_GT_MAX,
          fo.MIN_LT_12: fragment.ITEM_MIN_LT_12, fo.NO_POSITION: fragment.ITEM_NO_POSITION}


def check(seqs, mn, mx, exclude=(), include=()):
    raw = [s.encode("latin-1") if isinstance(s, str) else bytes(s) for s in seqs]
    flat, off = fo.ragged(raw)
    st, eff, emin, emax, foff, ends = fragment.fragment_arrays(flat, off, mn, mx, list(exclude), list(include))
    w_st, w_eff, w_emin, w_emax, w_ends = fo.fragment_batch(raw, mn, mx, list(exclude), list(include), threads=THREADS)
    for i, r in enumerate(raw):
        ctx = (r[:60], mn, mx)
        assert int(st[i]) == STATUS[int(w_st[i])], ctx
        assert np.float64(eff[i]).tobytes() == np.float64(w_eff[i]).tobytes(), ctx
        assert [int(x) for x in ends[int(foff[i]): int(foff[i + 1])]] == w_ends[i], ctx
        if int(w_st[i]) in (fo.MIN_GT_MAX, fo.MIN_LT_12):
            assert (int(emin[i]), int(emax[i])) == (int(w_emin[i]), int(w_emax[i])), ctx
    return st


def test_reference_pins():
    for name in ("TestFragment", "TestUnfragmentable", "TestSmallFragmentSize", "TestLongFragment"):
        b = P[name]
        check([b["seq"]], b["min"], b["max"])
    for b in P["TestFragmentSizes"]:
        check([b["seq"]], b["min"], b["max"])
    b = P["TestFragmentWithOverhangs"]
    check([b["seq"]], b["min"], b["max"], [], b["include"])
    b = P["Example_basic"]
    frags, _, err = fragment.Fragment(b["seq"], b["min"], b["max"], b["exclude"])
    assert err is None and frags == b["fragments"]
    b = P["ExampleFragment"]
    frags, eff, err = fragment.Fragment(b["seq"], b["min"], b["max"])
    assert frags[1] == b["fragment_1"] and "%f" % eff == b["efficiency_text"]
    s = list(P["ExampleNextOverhang"]["start"])
    for _ in range(3):
        s.append(fragment.NextOverhang(s))
    assert s == P["ExampleNextOverhang"]["output"]
    assert fragment.SetEfficiency(P["TestRegressionTestMatching12"]["set"]) == P["TestRegressionTestMatching12"]["efficiency"]
    assert "GTCT" not in fragment.NextOverhangs(["AGAC"])[0]
    _, _, err = fragment.Fragment(P["TestFragmentSizes"][0]["seq"], 105, 95)
    assert str(err) == "minFragmentSize (105) larger than maxFragmentSize (95)"
    _, _, err = fragment.Fragment(P["TestFragmentSizes"][1]["seq"], 7, 95)
    assert str(err) == "minFragmentSize must be equal to or greater than 12 . Got size of 7"
    frags, eff, err = fragment.Fragment(P["TestUnfragmentable"]["seq"], 40, 80)
    assert frags == [] and eff == 0 and str(err) == "bestOverhangPosition failed by equaling zero"
    with pytest.raises(_lib.GoPanic):
        fragment.Fragment("ACG", 12, 30)


def seeded_genes(n, seed):
    rnd = random.Random(seed)
    out = []
    for i in range(n):
        L = rnd.choice([4, 5, 11, 30, 90, 200, 600, 1500, 4000]) if i % 50 else rnd.randint(10_000, 20_000)
        # long genes stay A/C/G/T: the restatement's O(m^2) SetEfficiency would take minutes on a long N-rich one
        al = rnd.choice(["ACGT", "ACGT", "ACGT", "acgt", "ACGTN", "ACGTRYKMSWN", "AT"]) if L <= 4000 else rnd.choice(["ACGT", "acgt"])
        g = "".join(rnd.choice(al) for _ in range(L))
        if i % 97 == 0:
            g = g[: L // 2] + "NNNN" + g[L // 2:]
        if i % 211 == 0:
            g = g[:5] + "\xe9" + g[6:]
        out.append(g)
    return out + ["", "A", "ACG", "ACGT", "NNNN"]


EXCLUDES = [[], ["AAAA"], ["AAAA", "AAAA", "TTTT", "GTCT", "AGAC", "aaaa", "NNNN", "ACG", "ACGTAC", "", "NACG", "CGTN"],
            P["TestFragmentWithOverhangs"]["include"]]


@pytest.mark.parametrize("case", range(4))
def test_seeded_genes_against_oracle(case):
    mn, mx = [(90, 110), (12, 30), (40, 60), (200, 300)][case]
    genes = seeded_genes(500, case)
    check(genes, mn, mx, EXCLUDES[case])
    if case == 2:
        check(genes[:200], mn, mx, ["ACGT"], P["TestFragmentWithOverhangs"]["include"] + ["NNNA", "acgt"])


def test_argument_edges():
    rnd = random.Random(9)
    genes = ["".join(rnd.choice("ACGT") for _ in range(rnd.randint(20, 400))) for _ in range(200)]
    for mn, mx in ((105, 95), (7, 95), (5, 3), (12, 14), (12, 13), (20, 20), (-5, 40), (12, 10**12)):
        check(genes, mn, mx)
    # the end game reaches min < 12 in some of these
    st = check(["".join(rnd.choice("ACGT") for _ in range(rnd.randint(30, 60))) for _ in range(300)], 12, 20)
    assert (st == fragment.ITEM_MIN_LT_12).any() and (st == fragment.ITEM_OK).any()


def test_100kbp_gene():
    rnd = random.Random(100)
    g = "".join(rnd.choice("ACGT") for _ in range(100_000))
    check([g], 12, 30)
    gn = "".join(rnd.choice("ACGTN") for _ in range(6_000))  # overhangs with an N keep it going for many steps
    check([gn], 12, 30)


def test_empty_batch_and_capacity():
    assert fragment.FragmentBatch([], 90, 110) == []
    L = _lib.lib()
    z = np.zeros(8, dtype=np.uint8)
    off = np.zeros(1, dtype=np.uint64)
    foff, total = np.zeros(1, dtype=np.uint64), np.zeros(1, dtype=np.uint64)
    one = np.zeros(1)
    assert L.pg_fragment_batch(z.ctypes.data, off.ctypes.data, 0, 90, 110, z.ctypes.data, off.ctypes.data, 0, z.ctypes.data, off.ctypes.data, 0,
                               None, one.ctypes.data, one.ctypes.data, one.ctypes.data, foff.ctypes.data, None, 0, total.ctypes.data) == _lib.PG_OK
    # a NULL byte list with non-empty entries is an argument error, not a crash
    ex_off = np.array([0, 4], dtype=np.uint64)
    g, g_off = fo.ragged(["ACGTACGTACGT"])
    assert L.pg_fragment_batch(g.ctypes.data, g_off.ctypes.data, 1, 90, 110, None, ex_off.ctypes.data, 1, None, off.ctypes.data, 0, None,
                               one.ctypes.data, one.ctypes.data, one.ctypes.data, np.zeros(2, dtype=np.uint64).ctypes.data, None, 0,
                               total.ctypes.data) == _lib.PG_ERR_ARG
    assert L.pg_fragment_batch(None, g_off.ctypes.data, 1, 90, 110, None, off.ctypes.data, 0, None, off.ctypes.data, 0, None,
                               one.ctypes.data, one.ctypes.data, one.ctypes.data, np.zeros(2, dtype=np.uint64).ctypes.data, None, 0,
                               total.ctypes.data) == _lib.PG_ERR_ARG
    soff = np.array([0, 1], dtype=np.uint64)
    assert L.pg_fragment_set_efficiency_batch(None, ex_off.ctypes.data, soff.ctypes.data, 1, one.ctypes.data) == _lib.PG_ERR_ARG
    b = P["Example_basic"]
    flat, off = fo.ragged([b["seq"]] * 3)
    st, eff, _, _, foff, ends = fragment.fragment_arrays(flat, off, 95, 105, ["AAAA"], ends_cap=1)  # too small: one retry with the count
    assert list(foff) == [0, 4, 8, 12] and len(ends) == 12


def test_several_groups(monkeypatch):
    monkeypatch.setenv("PG_GROUP_BYTES", str(40_000))
    check(seeded_genes(120, 7), 40, 60, ["AAAA"])


def random_sets(n, seed):
    rnd = random.Random(seed)
    al = ["ACGT"] * 6 + ["ACGTN", "acgt"]
    sets = [[], ["AAAA"], ["AAAA", "TTTT"], ["AAAA", "AAAA"], ["ACG", "ACGTA", "", "NNNN"]]
    for _ in range(n - len(sets)):
        sets.append(["".join(rnd.choice(rnd.choice(al)) for _ in range(rnd.choice([4] * 12 + [3, 5])))
                     for _ in range(rnd.choice([0, 1, 2, 5, 10, 20, 40, 130, 300]) if rnd.random() < 0.2 else rnd.randint(0, 24))])
    return sets


def test_set_efficiency_and_next_overhangs():
    sets = random_sets(10_000, 1)
    eff = fragment.SetEfficiencyBatch(sets)
    want = fo.set_efficiency_batch(sets, threads=THREADS)
    assert eff.tobytes() == want.tobytes()
    assert max(sum(len(o) == 4 for o in s) for s in sets) > 128  # some sets spill their key list to global memory
    cands, nc, effs = fragment.next_overhangs_arrays(sets)
    w_c, w_n, w_e = fo.next_overhangs_batch(sets, threads=THREADS)
    assert (nc == w_n).all()
    for i in range(len(sets)):
        k = int(nc[i])
        assert cands[i, :k].tobytes() == w_c[i, :k].tobytes() and effs[i, :k].tobytes() == w_e[i, :k].tobytes(), sets[i]


def test_excludes_past_shared_memory():
    # more keyed excludes than the kernel keeps in shared memory (2 048): the rest are read from global memory
    rnd = random.Random(2100)
    keys = fo.fidelity()["keys"]
    ex = [rnd.choice(keys[:6]) for _ in range(2100)] + ["TTTT", "NNNA"]
    genes = ["".join(rnd.choice("ACGT") for _ in range(rnd.randint(50, 1500))) for _ in range(64)]
    st = check(genes, 40, 60, ex)
    assert (st == fragment.ITEM_OK).any()


def test_cpp_mirror_fragment_tests(tmp_path):
    rows = []

    def frow(name, seq, mn, mx, ex=(), inc=()):
        st, frags, eff, emin, emax = fo.fragment(seq, mn, mx, list(ex), list(inc))
        err = {fo.OK: "", fo.MIN_GT_MAX: f"minFragmentSize ({emin}) larger than maxFragmentSize ({emax})",
               fo.MIN_LT_12: f"minFragmentSize must be equal to or greater than 12 . Got size of {emin}",
               fo.NO_POSITION: "bestOverhangPosition failed by equaling zero"}[st]
        rows.append("\t".join(["F", name, seq, str(mn), str(mx), ",".join(ex), ",".join(inc), str(STATUS[st]), float(eff).hex(),
                                ",".join(f.decode() for f in frags), err]))
        return frags

    for name in ("TestFragment", "TestUnfragmentable", "TestSmallFragmentSize", "TestLongFragment"):
        b = P[name]
        frow(name, b["seq"], b["min"], b["max"])
    for b in P["TestFragmentSizes"]:
        frow("TestFragmentSizes", b["seq"], b["min"], b["max"])
    b = P["TestFragmentWithOverhangs"]
    frow("TestFragmentWithOverhangs", b["seq"], b["min"], b["max"], [], b["include"])
    b = P["Example_basic"]
    assert [f.decode() for f in frow("Example_basic", b["seq"], b["min"], b["max"], b["exclude"])] == b["fragments"]
    b = P["ExampleFragment"]
    assert frow("ExampleFragment", b["seq"], b["min"], b["max"])[1].decode() == b["fragment_1"]
    rnd = random.Random(12)
    for g in seeded_genes(60, 12):
        if g and "\xe9" not in g and len(g) >= 4:
            frow("random", g, 40, 60, ["AAAA", "GTCT"], [] if rnd.random() < 0.7 else EXCLUDES[3])
    for s in random_sets(60, 12):
        if "" not in s:
            rows.append("\t".join(["S", ",".join(s), float(fo.set_efficiency(s)).hex()]))
            c, e = fo.next_overhangs(s)
            rows.append("\t".join(["N", ",".join(s), ",".join(c), ",".join(float(x).hex() for x in e)]))
    tsv = tmp_path / "fragment_expected.tsv"
    tsv.write_text("\n".join(rows) + "\n")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "fragment_tests"
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-o", str(exe), os.path.join(root, "hostcpp", "fragment_tests.cpp"),
                           "-L" + os.path.join(root, "poly_b200", "lib"), "-lpolyb200", "-Wl,-rpath," + os.path.join(root, "poly_b200", "lib")])
    out = subprocess.run([str(exe), str(tsv)], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "fragment_tests: all passed" in out.stdout
