"""GPU parity for the secondary kernels (K4 Smith-Waterman score, K5 SantaLucia Tm)
through the C ABI: the reference's own known answers, then seeded batches vs the oracle."""
import json
import os

import numpy as np
import pytest

from poly_b200 import _lib, align, mash, primers, synth
from test_oracle_align_primers import GENE, NUC_4, TEST_LUT, TEST_MAT, design_primers, lut
from test_oracle_tm_restatement import same_bits

pytestmark = pytest.mark.gpu
GOLD = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "survey_goldens.json")))


def _make_scoring():
    a = align.NewAlphabet(["-", "A", "C", "G", "T"])
    return align.NewScoring(align.NewSubstitutionMatrix(a, a, TEST_MAT), -2)


SC = _make_scoring()


def last_kernel():
    return _lib.lib().pg_last_kernel().decode()


def test_reference_TestSmithWaterman(gpu):
    """search/align/align_test.go:139-292 (scores)."""
    assert align.SmithWatermanScore("TGTTACGG", "GGTTGACTA", SC) == 13
    assert align.SmithWatermanScore("ACACACTA", "AGCACACA", SC) == 17
    assert align.SmithWatermanScore("", "GAT", SC) == 0
    assert align.SmithWatermanScore("", "", SC) == 0
    assert align.SmithWatermanScore("G", "A", SC) == 0
    assert align.SmithWatermanScore("G", "G", SC) == 3
    assert align.SmithWatermanScore("G", "GATTACA", SC) == 3


def test_reference_examples(gpu):
    """search/align/example_test.go:49-111."""
    a5 = align.NewAlphabet(["A", "C", "G", "T", "U"])
    sc = align.NewScoring(align.NewSubstitutionMatrix(a5, a5, 2 * np.eye(5, dtype=np.int64) - 1), -1)
    assert align.SmithWatermanScore("GATTACA", "GCATGCU", sc) == 2
    an = align.NewAlphabet(["A", "C", "G", "T", "-"])
    sc = align.NewScoring(align.NewSubstitutionMatrix(an, an, align.NUC_4), -1)
    assert align.SmithWatermanScore("GATTACA", "GCATGCT", sc) == 15  # literal index mapping, not 17
    assert align.SmithWatermanScore("GATTACA", "GCATGCU", align.NewScoring(None, -1)) == 2  # matrix.Default


def test_sw_errors_match_reference_order(gpu, oracle):
    for a, b in [("ANA", "GAT"), ("NAA", "GXT"), ("ANA", "GXT"), ("AAN", "GAT"), ("", "X"), ("X", ""), ("ACGT", "ACGX")]:
        w = oracle.sw_score(a, b, TEST_LUT, TEST_LUT, TEST_MAT, -2)
        for query_is_a in (True, False):
            q, t = (a, b) if query_is_a else (b, a)
            scores, errs = align.SmithWatermanScores([q], t, SC, query_is_a=query_is_a)
            if w[3] == 0:
                assert errs[0] is None and scores[0] == w[0]
            else:
                bad = (a if w[3] == 1 else b)[w[4]]
                assert scores[0] == 0 and str(errs[0]) == f"Symbol {bad} not in alphabet"
    with pytest.raises(align.AlphabetError, match="Symbol X not in alphabet"):
        align.SmithWatermanScore("ACGT", "ACGX", SC)


@pytest.mark.parametrize("maxq,tlen", [(25, 10000), (32, 777), (33, 500), (64, 9000), (65, 300), (200, 1000)])
def test_sw_batch_vs_oracle(gpu, oracle, maxq, tlen):
    """All three kernel variants (<=32, <=64 register columns; long = global column), both
    orientations, ragged query lengths, a template longer than one smem chunk."""
    rng = np.random.default_rng(maxq)
    nq = 300
    qs = [bytes(rng.choice(list(b"ACGT-"), size=int(rng.integers(0, maxq + 1))).astype(np.uint8)) for _ in range(nq - 1)]
    qs.append(bytes(rng.choice(list(b"ACGT"), size=maxq).astype(np.uint8)))
    t = bytes(rng.choice(list(b"ACGT"), size=tlen).astype(np.uint8))
    for query_is_a in (True, False):
        scores, errs = align.SmithWatermanScores(qs, t, SC, query_is_a=query_is_a)
        assert last_kernel() in (("sw_score_kernel", "sw_score_x2_kernel") if maxq <= 64 else ("sw_score_long_kernel",))
        for i in range(0, nq, 7):
            a, b = (qs[i], t) if query_is_a else (t, qs[i])
            w = oracle.sw_score(a, b, TEST_LUT, TEST_LUT, TEST_MAT, -2)
            assert errs[i] is None and scores[i] == w[0], (i, query_is_a)


def test_sw_protein_matrix_and_wide_scores(gpu, oracle):
    """Non-square use of Default (26 letters) and values that force the int64 kernel."""
    rng = np.random.default_rng(9)
    letters = [chr(65 + i) for i in range(26)]
    qs = [bytes(rng.choice(list(range(65, 91)), size=30).astype(np.uint8)) for _ in range(40)]
    t = bytes(rng.choice(list(range(65, 91)), size=400).astype(np.uint8))
    sc = align.NewScoring(None, -1)
    scores, errs = align.SmithWatermanScores(qs, t, sc)
    l = lut(letters)
    for i in range(40):
        assert scores[i] == oracle.sw_score(qs[i], t, l, l, 2 * np.eye(26, dtype=np.int64) - 1, -1)[0]
    big = np.array(TEST_MAT, dtype=np.int64) * (1 << 33)
    a = align.NewAlphabet(["-", "A", "C", "G", "T"])
    scb = align.NewScoring(align.NewSubstitutionMatrix(a, a, big), -(1 << 34))
    q = [bytes(rng.choice(list(b"ACGT"), size=20).astype(np.uint8)) for _ in range(33)]
    tt = bytes(rng.choice(list(b"ACGT"), size=300).astype(np.uint8))
    scores, errs = align.SmithWatermanScores(q, tt, scb)
    for i in range(33):
        assert scores[i] == oracle.sw_score(q[i], tt, TEST_LUT, TEST_LUT, big, -(1 << 34))[0]


def test_cfg5_goldens_and_sample(gpu, oracle):
    """BASELINE configs[4] shape: 25-bp primers vs the 10 kb template."""
    n = 4096
    pr = synth.primers(n)
    off = synth.uniform_offsets(n, 25)
    tpl = synth.template()
    score, ec, ep = align.sw_scores_arrays(pr, off, tpl, SC)
    assert not ec.any()
    assert score[:6].tolist() == GOLD["cfg5"]["sw"]
    for i in range(0, n, 97):
        assert score[i] == oracle.sw_score(bytes(pr[25 * i:25 * i + 25]), bytes(tpl), TEST_LUT, TEST_LUT, TEST_MAT, -2)[0]
    tm, dh, ds, st = primers.santalucia_arrays(pr, off, primers.DEFAULT_CP, primers.DEFAULT_NA, primers.DEFAULT_MG)
    assert not st.any()
    assert tm[:6] == pytest.approx(GOLD["cfg5"]["tm"], rel=1e-6)  # north_star tolerance: 1e-6 relative
    for i in range(n):
        rc, wt, wh, ws = oracle.santalucia(bytes(pr[25 * i:25 * i + 25]), primers.DEFAULT_CP, primers.DEFAULT_NA, primers.DEFAULT_MG)
        assert rc == 0 and same_bits([tm[i], dh[i], ds[i]], [wt, wh, ws]).all(), i


def test_reference_tm_tests(gpu):
    """primers/primers_test.go:29-84."""
    tm, dh, ds = primers.SantaLucia("ACGATGGCAGTAGCATGC", 0.1e-6, 350e-3, 0.0)
    assert abs(62.7 - tm) / 62.7 < 0.02
    assert (tm, dh, ds) == pytest.approx(tuple(GOLD["tm"]["ACGATGGCAGTAGCATGC"]), rel=1e-6)
    tm, dh, ds = primers.SantaLucia("ACGTAGATCTACGT", 0.1e-6, 350e-3, 0.0)
    assert abs(47.428514 - tm) / 47.428514 < 0.02
    assert (tm, dh, ds) == pytest.approx(tuple(GOLD["tm"]["ACGTAGATCTACGT"]), rel=1e-6)
    tm = primers.MeltingTemp("GTAAAACGACGGCCAGT")
    assert abs(52.8 - tm) / 52.8 < 0.02 and tm == pytest.approx(GOLD["tm"]["GTAAAACGACGGCCAGT_meltingtemp"], rel=1e-6)
    assert primers.MeltingTemp("gtaaaacgacggccagt") == tm
    with pytest.raises(IndexError):
        primers.MeltingTemp("")
    with pytest.raises(ValueError):
        primers.MeltingTemp(b"AC\xc3\xa9")


def test_tm_edge_symbols_vs_oracle(gpu, oracle):
    """Unknown neighbours contribute {0,0} (primers.go:98), IUPAC palindromes, lower case."""
    rng = np.random.default_rng(4)
    seqs = [b"A", b"T", b"N", b"AT", b"ACGT", b"NNNN", b"RY", b"acgt", b"AcGtNnRy", b"SSSS", b"WWWW", b"A\x00T"]
    seqs += [bytes(rng.choice(list(b"ACGTNacgtnRYSWKMBDHV\x00 "), size=int(rng.integers(1, 60))).astype(np.uint8)) for _ in range(300)]
    bases, off = mash.flatten(seqs)
    for (cp, na, mg) in [(500e-9, 50e-3, 0.0), (0.1e-6, 350e-3, 0.0), (1e-6, 10e-3, 2e-3)]:
        tm, dh, ds, st = primers.santalucia_arrays(bases, off, cp, na, mg)
        for i, q in enumerate(seqs):
            rc, wt, wh, ws = oracle.santalucia(q, cp, na, mg)
            assert rc == 0 and st[i] == 0
            assert same_bits([tm[i], dh[i], ds[i]], [wt, wh, ws]).all(), q


def test_reference_design_primers_through_gpu(gpu):
    """primers/pcr/example_test.go:36,46,54: primer strings pinned by Tm threshold crossings,
    with every MeltingTemp evaluated on the GPU."""
    assert design_primers(primers.MeltingTemp, GENE, 55.0) == ("AATAATTACACCGAGATAACACATCATGG", "TTAAGAAAGCGCATTTTCCAGC")


def test_reference_TestNeedlemanWunsch(gpu):
    """search/align/align_test.go:11-137 and example_test.go:10-47 (scores)."""
    a5 = align.NewAlphabet(["A", "C", "G", "T", "U"])
    sc = align.NewScoring(align.NewSubstitutionMatrix(a5, a5, 2 * np.eye(5, dtype=np.int64) - 1), -1)
    for a, b, want in [("GATTACA", "GCATGCU", 0), ("GATTACA", "GATTACA", 7), ("GATTACA", "GAT", -1), ("", "GAT", -3), ("", "", 0),
                       ("G", "A", -1), ("G", "G", 1), ("G", "GATTACA", -5), ("GAT", "", -3)]:
        assert align.NeedlemanWunschScore(a, b, sc) == want, (a, b)
    with pytest.raises(align.AlphabetError, match="Symbol X not in alphabet"):
        align.NeedlemanWunschScore("GATX", "GAT", sc)


@pytest.mark.parametrize("maxq,tlen", [(25, 3000), (40, 9000), (64, 500), (150, 400)])
def test_nw_batch_vs_oracle(gpu, oracle, maxq, tlen):
    rng = np.random.default_rng(maxq + 1)
    nq = 200
    qs = [bytes(rng.choice(list(b"ACGT"), size=int(rng.integers(0, maxq + 1))).astype(np.uint8)) for _ in range(nq - 1)]
    qs.append(bytes(rng.choice(list(b"ACGT"), size=maxq).astype(np.uint8)))
    t = bytes(rng.choice(list(b"ACGT"), size=tlen).astype(np.uint8))
    for query_is_a in (True, False):
        scores, errs = align.NeedlemanWunschScores(qs, t, SC, query_is_a=query_is_a)
        assert last_kernel() == ("nw_score_kernel" if maxq <= 64 else "sw_score_long_kernel")
        for i in range(0, nq, 5):
            a, b = (qs[i], t) if query_is_a else (t, qs[i])
            w = oracle.nw_score(a, b, TEST_LUT, TEST_LUT, TEST_MAT, -2)
            assert errs[i] is None and scores[i] == w[0], (i, query_is_a, len(qs[i]))
    # positive "gap" (a reward) exercises the masked Smith-Waterman variant
    scp = align.NewScoring(SC.SubstitutionMatrix, 1)
    scores, errs = align.SmithWatermanScores(qs[:60], t[:300], scp)
    for i in range(60):
        assert scores[i] == oracle.sw_score(qs[i], t[:300], TEST_LUT, TEST_LUT, TEST_MAT, 1)[0]


def test_cfg5_full_size_properties(gpu, oracle):
    """BASELINE configs[4] at full size: 1M x 25 bp primers vs the 10 kb template."""
    n = 1_000_000
    pr = synth.primers(n)
    off = synth.uniform_offsets(n, 25)
    tpl = synth.template()
    score, ec, ep = align.sw_scores_arrays(pr, off, tpl, SC)
    assert not ec.any() and score.min() >= 0 and score.max() <= 75        # 25 matches x 3
    idx = np.random.default_rng(8).integers(0, n, 200)
    for i in idx:
        assert score[i] == oracle.sw_score(bytes(pr[25 * i:25 * i + 25]), bytes(tpl), TEST_LUT, TEST_LUT, TEST_MAT, -2)[0]
    # the same primers in two halves give the same scores (chunk independence)
    s2, _, _ = align.sw_scores_arrays(pr[: 25 * 1000], off[:1001], tpl, SC)
    assert np.array_equal(s2, score[:1000])
    tm, dh, ds, st = primers.santalucia_arrays(pr, off, primers.DEFAULT_CP, primers.DEFAULT_NA, primers.DEFAULT_MG)
    assert not st.any() and np.isfinite(tm).all() and 20 < tm.min() and tm.max() < 90
    for i in idx:
        assert same_bits(tm[i], oracle.melting_temp(bytes(pr[25 * i:25 * i + 25]))), i


def test_reference_alignment_strings(gpu):
    """The aligned strings of align.SmithWaterman: search/align/align_test.go:157-291 and
    search/align/example_test.go:82,110."""
    assert align.SmithWatermanAlign("TGTTACGG", "GGTTGACTA", SC) == (13, "GTT-AC", "GTTGAC")
    assert align.SmithWatermanAlign("ACACACTA", "AGCACACA", SC) == (17, "A-CACACTA", "AGCACAC-A")
    assert align.SmithWatermanAlign("", "GAT", SC) == (0, "", "")
    assert align.SmithWatermanAlign("", "", SC) == (0, "", "")
    assert align.SmithWatermanAlign("G", "A", SC) == (0, "", "")
    assert align.SmithWatermanAlign("G", "G", SC) == (3, "G", "G")
    assert align.SmithWatermanAlign("G", "GATTACA", SC) == (3, "G", "G")
    a5 = align.NewAlphabet(["A", "C", "G", "T", "U"])
    sc = align.NewScoring(align.NewSubstitutionMatrix(a5, a5, 2 * np.eye(5, dtype=np.int64) - 1), -1)
    assert align.SmithWatermanAlign("GATTACA", "GCATGCU", sc) == (2, "AT", "AT")
    an = align.NewAlphabet(["A", "C", "G", "T", "-"])
    sc = align.NewScoring(align.NewSubstitutionMatrix(an, an, align.NUC_4), -1)
    assert align.SmithWatermanAlign("GATTACA", "GCATGCT", sc) == (15, "GATTAC", "GCATGC")
    with pytest.raises(align.AlphabetError, match="Symbol X not in alphabet"):
        align.SmithWatermanAlign("ACGT", "ACGX", SC)


@pytest.mark.parametrize("maxq,tlen,gap", [(25, 10000, -2), (32, 700, -1), (33, 500, -2), (64, 3000, -3), (20, 400, 0), (12, 300, 1)])
def test_sw_align_batch_vs_oracle(gpu, oracle, maxq, tlen, gap):
    """Tie-breaking of the first maximum and of the traceback, both orientations, ragged
    queries, gap 0 / positive gap (long gap runs leave the default window: full-window retry)."""
    rng = np.random.default_rng(maxq * 7 + tlen)
    nq = 150
    qs = [bytes(rng.choice(list(b"ACGT"), size=int(rng.integers(0, maxq + 1))).astype(np.uint8)) for _ in range(nq - 1)]
    qs.append(bytes(rng.choice(list(b"ACGT"), size=maxq).astype(np.uint8)))
    t = bytes(rng.choice(list(b"ACGT"), size=tlen).astype(np.uint8))
    # plant near-copies of some queries (with an indel) so that real gapped alignments occur
    tl = bytearray(t)
    for k_, q in enumerate(qs[:40]):
        if len(q) > 8:
            pos = 50 + k_ * (tlen - 200) // 40
            ins = q[: len(q) // 2] + b"T" + q[len(q) // 2:]
            tl[pos: pos + len(ins)] = ins[: max(0, min(len(ins), tlen - pos))]
    t = bytes(tl[:tlen])
    sc = align.NewScoring(SC.SubstitutionMatrix, gap)
    for query_is_a in (True, False):
        res = align.SmithWatermanAligns(qs, t, sc, query_is_a=query_is_a)
        assert last_kernel() == "sw_align_kernel"
        step = 1 if tlen <= 1000 else 3
        for i in range(0, nq, step):
            a, b = (qs[i], t) if query_is_a else (t, qs[i])
            w = oracle.sw_align(a, b, TEST_LUT, TEST_LUT, TEST_MAT, gap)
            assert res[i][3] is None
            assert (res[i][0], res[i][1].encode(), res[i][2].encode()) == (w[0], w[1], w[2]), (i, query_is_a, qs[i])


def test_reference_pcr_examples_batched(gpu):
    """primers/pcr/example_test.go:10-55: DesignPrimers / DesignPrimersWithOverhangs strings from the
    batched GPU search (pg_design_primers_batch)."""
    from poly_b200 import pcr

    assert pcr.DesignPrimers(GENE, 55.0) == ("AATAATTACACCGAGATAACACATCATGG", "TTAAGAAAGCGCATTTTCCAGC")
    assert pcr.DesignPrimersWithOverhangs(GENE, "TTATAGGTCTCATACT", "ATGAAGAGACCATATA", 55.0) == (
        "TTATAGGTCTCATACTAATAATTACACCGAGATAACACATCATGG", "TATATGGTCTCTTCATTTAAGAAAGCGCATTTTCCAGC")
    with pytest.raises(IndexError):
        pcr.DesignPrimers("ACGTACGTAC", 55.0)          # shorter than 15 nt: sequence[0:15] panics
    with pytest.raises(IndexError):
        pcr.DesignPrimers("AT" * 12, 95.0)             # exhausted before the target is reached


def test_design_primers_batch_vs_oracle(gpu, oracle):
    from poly_b200 import pcr

    rng = np.random.default_rng(12)
    genes = [bytes(rng.choice(list(b"ACGTacgtN"), size=int(rng.integers(40, 400)), p=[.22, .22, .22, .22, .02, .02, .02, .02, .04]).astype(np.uint8)) for _ in range(300)]
    for target in (48.0, 55.0, 62.5):
        fwd, rev, st = pcr.design_primer_lengths(genes, target)
        for i, g in enumerate(genes):
            try:
                wf, wr = design_primers(oracle.melting_temp, g.decode("latin-1"), target)
            except (IndexError, ValueError):
                assert st[i] == 1, i
                continue
            assert st[i] == 0 and (fwd[i], rev[i]) == (len(wf), len(wr)), (i, target)


def test_reference_nw_alignment_strings(gpu, oracle):
    """ExampleNeedlemanWunsch (search/align/example_test.go:10-47): score 0, G-ATTACA / GCA-TGCU;
    plus the reference's loop condition (traceback stops when one string is exhausted)."""
    a5 = align.NewAlphabet(["A", "C", "G", "T", "U"])
    sc = align.NewScoring(align.NewSubstitutionMatrix(a5, a5, 2 * np.eye(5, dtype=np.int64) - 1), -1)
    assert align.NeedlemanWunschAlign("GATTACA", "GCATGCU", sc) == (0, "G-ATTACA", "GCA-TGCU")
    assert align.NeedlemanWunschAlign("GATTACA", "GATTACA", sc) == (7, "GATTACA", "GATTACA")
    assert align.NeedlemanWunschAlign("", "GAT", sc) == (-3, "", "")
    l5 = lut(["A", "C", "G", "T", "U"])
    m5 = 2 * np.eye(5, dtype=np.int64) - 1
    for a, b in [("GATTACA", "GAT"), ("G", "GATTACA"), ("G", "A"), ("GAT", "GATTACA"), ("GCATGCU", "GATTACA")]:
        w = oracle.nw_align(a, b, l5, l5, m5, -1)
        assert align.NeedlemanWunschAlign(a, b, sc) == (w[0], w[1].decode(), w[2].decode()), (a, b)


@pytest.mark.parametrize("maxq,tlen,gap", [(25, 600, -2), (40, 300, -1), (64, 150, -3), (10, 50, 0)])
def test_nw_align_batch_vs_oracle(gpu, oracle, maxq, tlen, gap):
    rng = np.random.default_rng(maxq + tlen)
    nq = 80
    qs = [bytes(rng.choice(list(b"ACGT"), size=int(rng.integers(0, maxq + 1))).astype(np.uint8)) for _ in range(nq - 1)]
    qs.append(bytes(rng.choice(list(b"ACGT"), size=maxq).astype(np.uint8)))
    t = bytes(rng.choice(list(b"ACGT"), size=tlen).astype(np.uint8))
    sc = align.NewScoring(SC.SubstitutionMatrix, gap)
    for query_is_a in (True, False):
        res = align.SmithWatermanAligns(qs, t, sc, query_is_a=query_is_a, global_alignment=True)
        for i in range(nq):
            a, b = (qs[i], t) if query_is_a else (t, qs[i])
            w = oracle.nw_align(a, b, TEST_LUT, TEST_LUT, TEST_MAT, gap)
            assert res[i][3] is None and (res[i][0], res[i][1].encode(), res[i][2].encode()) == (w[0], w[1], w[2]), (i, query_is_a)


def test_reference_return_shape_and_long_pairs(gpu, oracle):
    """align.SmithWaterman / NeedlemanWunsch return (score, alignA, alignB, err) like the reference
    (align.go:100,171); pairs with BOTH strings longer than 64 symbols keep the whole matrix in HBM
    (sw_align_long.cu) and must give the oracle's strings, including the first-maximum rule and the
    diagonal > up > left preference."""
    assert align.SmithWaterman("TGTTACGG", "GGTTGACTA", SC) == (13, "GTT-AC", "GTTGAC", None)
    sc5 = align.NewScoring(None, -1)
    assert align.NeedlemanWunsch("GATTACA", "GATTACA", sc5) == (7, "GATTACA", "GATTACA", None)
    score, a, b, err = align.SmithWaterman("ACGT", "ACGX", SC)
    assert (score, a, b) == (0, "", "") and str(err) == "Symbol X not in alphabet"
    rng = np.random.default_rng(64)
    ALPHA = align.NewAlphabet(["-", "A", "C", "G", "T"])
    MAT = TEST_MAT
    lut = ALPHA.byte_lut()
    mat = np.array(MAT, dtype=np.int64)
    for la, lb in [(65, 65), (70, 300), (300, 70), (257, 1000), (1000, 999), (129, 65)]:
        base = rng.choice(list(b"ACGT"), size=max(la, lb) + 50).astype(np.uint8)
        a = bytes(base[:la])
        mut = base[10: 10 + lb].copy()
        flip = rng.random(lb) < 0.08
        mut[flip] = rng.choice(list(b"ACGT"), size=int(flip.sum()))
        b = bytes(np.delete(mut, rng.integers(0, lb, 3)))            # a few deletions -> gaps in the alignment
        for gap in (-2, -5):
            scg = align.NewScoring(align.NewSubstitutionMatrix(ALPHA, ALPHA, MAT), gap)
            w = oracle.sw_align(a, b, lut, lut, mat, gap)
            assert align.SmithWaterman(a, b, scg) == (w[0], w[1].decode(), w[2].decode(), None), (la, lb, gap)
            w = oracle.nw_align(a, b, lut, lut, mat, gap)
            assert align.NeedlemanWunsch(a, b, scg) == (w[0], w[1].decode(), w[2].decode(), None), (la, lb, gap)
    # ties everywhere: homopolymers (first maximum in row-major order, diagonal preference)
    a, b = b"A" * 100, b"A" * 90
    w = oracle.sw_align(a, b, lut, lut, mat, -2)
    assert align.SmithWaterman(a, b, SC) == (w[0], w[1].decode(), w[2].decode(), None)
    # an error in a long pair: same (0, "", "", err) as the reference
    score, sa, sb, err = align.SmithWaterman(b"ACGT" * 30 + b"N", b"ACGT" * 40, SC)
    assert (score, sa, sb) == (0, "", "") and str(err) == "Symbol N not in alphabet"


def test_sw_packed_int16_kernel(gpu, oracle):
    """sw_score_x2_kernel (two queries per register, DPX s16x2): odd batch sizes, empty queries, queries whose
    partner is longer / shorter / invalid, tables with larger magnitudes, gap 0, both orientations; and the
    bound that sends larger scores back to the 32-bit kernel."""
    rng = np.random.default_rng(16)
    a5 = align.NewAlphabet(["-", "A", "C", "G", "T"])
    lut5 = a5.byte_lut()
    for nq, maxq, tlen, gap, scale in [(3, 25, 2000, -2, 1), (301, 32, 9000, -7, 60), (77, 28, 500, 0, 1), (2, 8, 100, -1, 100), (129, 16, 8200, -3, 9)]:
        mat = (np.array(TEST_MAT, dtype=np.int64) * scale)
        mat[2, 3] = mat[3, 2] = scale * 2                     # not just a match / mismatch table
        sc = align.NewScoring(align.NewSubstitutionMatrix(a5, a5, mat.tolist()), gap)
        qs = [bytes(rng.choice(list(b"ACGT-"), size=int(rng.integers(0, maxq + 1))).astype(np.uint8)) for _ in range(nq)]
        qs[0] = bytes(rng.choice(list(b"ACGT"), size=maxq).astype(np.uint8))
        if nq > 2:
            qs[1] = b""
            qs[2] = qs[2][:3] + b"N" + qs[2][3:maxq - 1]      # invalid symbol: (0, err) for this query only
        t = bytes(rng.choice(list(b"ACGT"), size=tlen).astype(np.uint8))
        for query_is_a in (True, False):
            scores, errs = align.SmithWatermanScores(qs, t, sc, query_is_a=query_is_a)
            assert last_kernel() == "sw_score_x2_kernel"
            for i in range(nq):
                x, y = (qs[i], t) if query_is_a else (t, qs[i])
                w = oracle.sw_score(x, y, lut5, lut5, mat, gap)
                assert scores[i] == w[0] and (errs[i] is None) == (w[3] == 0), (nq, i, query_is_a)
    # 25 x 700 = 17500 > 2^14: the packed kernel must not be chosen (values would wrap)
    mat = np.array(TEST_MAT, dtype=np.int64) * 700
    sc = align.NewScoring(align.NewSubstitutionMatrix(a5, a5, mat.tolist()), -2)
    q = [bytes(rng.choice(list(b"ACGT"), size=25).astype(np.uint8)) for _ in range(10)]
    t = q[3] + bytes(rng.choice(list(b"ACGT"), size=300).astype(np.uint8))
    scores, _ = align.SmithWatermanScores(q, t, sc)
    assert last_kernel() == "sw_score_kernel"
    assert scores[3] == 25 * 3 * 700 and all(scores[i] == oracle.sw_score(q[i], t, lut5, lut5, mat, -2)[0] for i in range(10))
