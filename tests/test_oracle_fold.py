"""CPU tier for fold: the C restatement (oracle/fold_oracle.c) reproduces every pin of poly's fold tests
(fold_test.go, seqfold_test.go, example_test.go), and the library's energy tables equal
tests/golden/fold/energies.json entry by entry."""
import math
import os
import re

import pytest

import fold_oracle as fo

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def mfe(seq: str, temp: float = 37.0) -> float:
    st, e, _ = fo.fold(seq.encode(), temp)
    assert st == fo.OK
    return e


UNAFOLD_DNA = {
    "GGGAGGTCGTTACATCTGGGTAACACCGGTACTGATCCGGTGACCTCCC": -10.94,
    "GGGAGGTCGCTCCAGCTGGGAGGAGCGTTGGGGGTATATACCCCCAACACCGGTACTGATCCGGTGACCTCCC": -23.4,
    "CGCAGGGAUACCCGCG": -3.8,
    "TAGCTCAGCTGGGAGAGCGCCTGCTTTGCACGCAGGAGGT": -6.85,
    "GGGGGCATAGCTCAGCTGGGAGAGCGCCTGCTTTGCACGCAGGAGGTCTGCGGTTCGATCCCGCGCGCTCCCACCA": -15.50,
    "TGAGACGGAAGGGGATGATTGTCCCCTTCCGTCTCA": -18.10,
    "ACCCCCTCCTTCCTTGGATCAAGGGGCTCAA": -3.65,
}
UNAFOLD_RNA = {
    "ACCCCCUCCUUCCUUGGAUCAAGGGGCUCAA": -9.5,
    "AAGGGGUUGGUCGCCUCGACUAAGCGGCUUGGAAUUCC": -10.1,
    "UUGGAGUACACAACCUGUACACUCUUUC": -4.3,
    "AGGGAAAAUCCC": -3.3,
    "GCUUACGAGCAAGUUAAGCAAC": -4.6,
    "UGGGAGGUCGUCUAACGGUAGGACGGCGGACUCUGGAUCCGCUGGUGGAGGUUCGAGUCCUCCCCUCCCAGCCA": -32.8,
    "GGGCGAUGAGGCCCGCCCAAACUGCCCUGAAAAGGGCUGAUGGCCUCUACUG": -20.7,
    "GGGGGCAUAGCUCAGCUGGGAGAGCGCCUGCUUUGCACGCAGGAGGUCUGCGGUUCGAUCCCGCGCGCUCCCACCA": -31.4,
}


@pytest.mark.parametrize("table,frac", [(UNAFOLD_DNA, 0.6), (UNAFOLD_RNA, 0.5)])
def test_unafold_tolerances(table, frac):
    for seq, ufold in table.items():
        d = mfe(seq)
        assert abs(d - ufold) <= abs(frac * min(d, ufold)), seq


def test_fold_cache_matches_w():
    seq = "ATGGATTTAGATAGAT"
    st, w = fo.probe(seq.encode(), 37.0, "W", 0, len(seq) - 1)
    assert st == fo.OK and abs(mfe(seq) - w) <= 1


def test_dot_bracket_and_example():
    st, _, db = fo.fold(b"GGGAGGTCGTTACATCTGGGTAACACCGGTACTGATCCGGTGACCTCCC", 37.0)
    assert db == b"((((((((.((((......))))..((((.......)))).))))))))"
    st, _, db = fo.fold(b"ACCCCCUCCUUCCUUGGAUCAAGGGGCUCAA", 37.0)
    assert db == b".((((.(((......)))....))))"  # 26 characters for 31 nt: DotBracket stops at the last ')'


def test_multibranch_has_7_41():
    _, _, _, structs = fo.fold(b"GGGAGGTCGTTACATCTGGGTAACACCGGTACTGATCCGGTGACCTCCC", 37.0, with_structs=True)
    assert any("BIFURCATION" in d and (7, 41) in inner for _, d, inner in structs)


def test_pair_stack_bulge_hairpin_internal_loop_w():
    assert fo.pair(b"ATGGAATAGTG", 0, 1, 9, 10) == "AT/TG"
    st, e = fo.probe(b"GCUCAGCUGGGAGAGC", 37.0, "stack", 1, 2, 14, 13)
    assert st == fo.OK and abs(e - -2.1) <= 0.1
    st, e = fo.probe(b"ACCCCCATCCTTCCTTGAGTCAAGGGGCTCAA", 37.0, "Bulge", 5, 7, 18, 17)
    assert st == fo.OK and abs(e - 3.22) <= 0.4
    for seq, i, j, want, tol in ((b"ACCCCCTCCTTCCTTGGATCAAGGGGCTCAA", 11, 16, 4.3, 1.0), (b"ACCCGCAAGCCCTCCTTCCTTGGATCAAGGGGCTCAA", 3, 8, 0.67, 0.1),
                                 (b"CUUUGCACG", 0, 8, 4.5, 0.2)):
        st, e = fo.probe(seq, 37.0, "hairpin", i, j)
        assert st == fo.OK and abs(e - want) <= tol
    st, e = fo.probe(b"ACCCCCTCCTTCCTTGGATCAAGGGGCTCAA", 37.0, "internalLoop", 6, 10, 21, 17)
    assert st == fo.OK and abs(e - 3.5) <= 0.1
    for seq, want in ((b"GCUCAGCUGGGAGAGC", -3.8), (b"CCUGCUUUGCACGCAGG", -6.4), (b"GCGGUUCGAUCCCGC", -4.2)):
        st, e = fo.probe(seq, 37.0, "W", 0, len(seq) - 1)
        assert st == fo.OK and abs(e - want) <= 0.2


def test_errors_and_panics():
    assert fo.fold(b"ATGGATTTAGATAGATADFQ#(RSDOFIA)", 4000.0)[0] == fo.NOT_NUCLEIC
    assert fo.fold(b"XYZ", 37.0)[0] == fo.NOT_NUCLEIC
    assert fo.fold(b"ACGUT", 37.0)[0] == fo.NOT_NUCLEIC  # T and U together
    assert fo.fold(b"", 37.0)[0] == fo.PANIC
    assert fo.fold(b"A", 37.0)[0] == fo.PANIC
    assert fo.fold(b"ACG\xc3\xa9", 37.0)[0] == fo.UNSUPPORTED


def test_never_computed_cells():
    # 2..4 nt: W[0][n-1] is invalid and V[0][n-1] was never computed: MFE -inf, brackets at both ends
    for s, db in ((b"AC", b"()"), (b"ACG", b"(.)"), (b"ACGT", b"(..)")):
        st, e, got = fo.fold(s, 37.0)
        assert st == fo.OK and e == -math.inf and got == db
    st, e, db = fo.fold(b"AAAAAAAAAA", 37.0)  # no pair at all
    assert st == fo.OK and e == -math.inf and db == b"........()"


def test_empty_result_mfe_is_inf():
    # Result{}.MinimumFreeEnergy() is +inf and DotBracket() is "": the library's Result() default
    from poly_b200 import fold

    assert fold.Result().MinimumFreeEnergy() == math.inf and fold.Result().DotBracket() == ""


NAN, INF = math.nan, math.inf


@pytest.mark.parametrize("a,b,want", [
    (-1.0, 1.0, -1.0), (1.0, -1.0, -1.0),     # ordered operands
    (1.0, -INF, -INF), (-INF, 1.0, -INF),     # -Inf wins over anything ...
    (NAN, -INF, -INF), (-INF, NAN, -INF),     # ... NaN included
    (NAN, 1.0, NAN), (1.0, NAN, NAN),         # NaN next, whichever side it is on
    (INF, NAN, NAN), (NAN, NAN, NAN),
    (-0.0, 0.0, -0.0), (0.0, -0.0, -0.0),     # -0 below +0
    (0.0, 0.0, 0.0), (-0.0, -0.0, -0.0), (INF, 1.0, 1.0),
])
def test_go_min_is_math_min(a, b, want):
    # Go's math.Min: Min(x, -Inf) = Min(-Inf, x) = -Inf, Min(x, NaN) = Min(NaN, x) = NaN,
    # Min(-0, +-0) = Min(+-0, -0) = -0, in that order of precedence
    got = fo.go_min(a, b)
    if math.isnan(want):
        assert math.isnan(got)
    else:
        assert got == want and math.copysign(1.0, got) == math.copysign(1.0, want)


def test_branch_heavy_item_fits_the_kernel_capacities():
    # fold.cu keeps a W cell's branch list in an arena slot of (d + 1) / 5 entries (d = end - start) and the
    # traceback's pending branches in a 256-entry stack.  Replay the traceback's order on the restatement's
    # structure list: each chain of V cells pops one pending branch; a multibranch ends its chain and pushes
    # its branches (its "BIFURCATION:<u>n/<h>h" description counts the closing pair too).
    import fold_designs

    st, _, _, structs = fo.fold(fold_designs.branch_heavy().encode(), 37.0, with_structs=True)
    assert st == fo.OK
    largest, largest_cap, depth, pending, chain = 0, 0, 0, 1, False
    for _, desc, [(s, e)] in structs:
        if not chain:
            pending -= 1
            chain = True
        if desc.startswith("BIFURCATION"):
            nb = int(desc.split("/")[1].rstrip("h")) - 1
            cap = (e - s + 1) // 5
            assert nb <= cap, (s, e, nb, cap)
            largest, largest_cap = max((largest, largest_cap), (nb, cap))
            pending += nb
            depth = max(depth, pending)
            chain = False
        elif desc.startswith("HAIRPIN") or desc == "":  # no inner pair: the chain ends
            chain = False
    assert pending == 0 and not chain
    print(f"largest branch list {largest} of a slot of {largest_cap}; deepest pending branches {depth} of 256")
    assert largest >= 3 and 10 <= depth <= 256


def _inc_tables():
    text = open(os.path.join(ROOT, "poly_b200", "csrc", "fold_tables.inc")).read()
    out = {}
    for kind, name, body in re.findall(r"static const (?:KeyEnergy|LenEnergy) k_(dna|rna)_(\w+)\[\] = \{(.*?)\};", text, re.S):
        ent = {}
        for k, h, s in re.findall(r'\{"?([^",]+?)"?, ([-0-9.e]+), ([-0-9.e]+)\}', body):
            if k not in ("nullptr", "-1"):
                ent[k] = [float(h), float(s)]
        out.setdefault(kind, {})[name] = ent
    for kind, body in re.findall(r"static const double k_(dna|rna)_multibranch\[4\] = \{(.*?)\};", text):
        out[kind]["multibranch"] = [float(x) for x in body.split(",")]
    return out


def test_library_tables_equal_golden():
    golden = fo.energies()
    lib = _inc_tables()
    for kind in ("dna", "rna"):
        g = {k: v for k, v in golden[kind].items() if k == "multibranch" or v}
        l = {k: v for k, v in lib[kind].items() if k == "multibranch" or v}
        assert l == g, kind
