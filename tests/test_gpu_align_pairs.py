"""GPU parity of the pair-list alignment calls (pg_sw/nw_score_pairs, _dev, pg_sw/nw_align_pairs):
the reference's known answers as one pair batch, then seeded ragged pairs against the oracle on
both sides of every kernel boundary."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import pair_oracle
from poly_b200 import _lib, align, mash, synth
from poly_b200.mash import flatten
from test_oracle_align_primers import TEST_LUT, TEST_MAT

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ALPHA = align.NewAlphabet(["-", "A", "C", "G", "T"])


def scoring(gap=-2, mat=TEST_MAT):
    return align.NewScoring(align.NewSubstitutionMatrix(ALPHA, ALPHA, mat), gap)


def oracle_pairs(oracle, A, B, pairs, lut_a, lut_b, mat, gap, global_alignment=False):
    """The C pair driver over po_sw_score / po_nw_score on all host threads: [(score, err_code, err_pos)]."""
    return list(zip(*(x.tolist() for x in pair_oracle.scores(A, B, pairs, lut_a, lut_b, mat, gap, global_alignment))))


def check_vs_oracle(oracle, A, B, pairs, sc, lut_a=TEST_LUT, lut_b=TEST_LUT, mat=TEST_MAT):
    for g in (False, True):
        score, ec, ep = align.pair_scores_arrays(A, B, pairs, sc, g)
        want = oracle_pairs(oracle, A, B, pairs, lut_a, lut_b, np.asarray(mat), sc.GapPenalty, g)
        got = list(zip(score.tolist(), ec.tolist(), ep.tolist()))
        bad = [(k, len(A[int(pairs[k][0])]), len(B[int(pairs[k][1])]), got[k], tuple(want[k])) for k in range(len(pairs)) if got[k] != tuple(want[k])]
        assert not bad, (g, sc.GapPenalty, bad[:5])


def rand_seqs(rng, lens, alphabet=b"ACGT"):
    return [bytes(rng.choice(list(alphabet), size=int(n)).astype(np.uint8)) for n in lens]


def test_reference_known_answers_as_one_batch(gpu):
    """align_test.go / example_test.go answers, every pair in one call."""
    cases = [("TGTTACGG", "GGTTGACTA", 13), ("ACACACTA", "AGCACACA", 17), ("", "GAT", 0), ("", "", 0), ("G", "A", 0),
             ("G", "G", 3), ("G", "GATTACA", 3)]
    A = [a for a, _, _ in cases]
    B = [b for _, b, _ in cases]
    pairs = np.stack([np.arange(len(cases)), np.arange(len(cases))], 1)
    scores, errs = align.SmithWatermanPairScores(A, B, pairs, scoring())
    assert scores == [w for _, _, w in cases] and errs == [None] * len(cases)
    al = align.SmithWatermanPairAligns(A, B, pairs, scoring())
    assert [x[:3] for x in al] == [(13, "GTT-AC", "GTTGAC"), (17, "A-CACACTA", "AGCACAC-A"), (0, "", ""), (0, "", ""), (0, "", ""),
                                   (3, "G", "G"), (3, "G", "G")]
    an = align.NewAlphabet(["A", "C", "G", "T", "-"])
    nuc = align.NewScoring(align.NewSubstitutionMatrix(an, an, align.NUC_4), -1)
    assert align.SmithWatermanPairScores(["GATTACA"], ["GCATGCT"], [[0, 0]], nuc)[0] == [15]  # literal index mapping
    assert align.SmithWatermanPairScores(["GATTACA"], ["GCATGCU"], [[0, 0]], align.NewScoring(None, -1))[0] == [2]
    a5 = align.NewAlphabet(["A", "C", "G", "T", "U"])
    sc5 = align.NewScoring(align.NewSubstitutionMatrix(a5, a5, 2 * np.eye(5, dtype=np.int64) - 1), -1)
    nw = [("GATTACA", "GCATGCU", 0), ("GATTACA", "GATTACA", 7), ("GATTACA", "GAT", -1), ("", "GAT", -3), ("", "", 0),
          ("G", "A", -1), ("G", "G", 1), ("G", "GATTACA", -5), ("GAT", "", -3)]
    p = np.stack([np.arange(len(nw))] * 2, 1)
    assert align.NeedlemanWunschPairScores([a for a, _, _ in nw], [b for _, b, _ in nw], p, sc5)[0] == [w for _, _, w in nw]
    assert align.SmithWatermanPairAligns(["GATTACA"], ["GCATGCU"], [[0, 0]], sc5)[0][:3] == (2, "AT", "AT")
    assert align.SmithWatermanPairAligns(["GATTACA"], ["GCATGCT"], [[0, 0]], nuc)[0][:3] == (15, "GATTAC", "GCATGC")


BOUNDS = [0, 1, 31, 32, 33, 63, 64, 65, 127, 128, 129, 159, 160, 161, 255, 256, 257, 511, 512, 513, 2047, 2048, 2049]


@pytest.mark.parametrize("gap", [-3, -2, -1, 0, 1])
def test_random_ragged_pairs_vs_oracle(gpu, oracle, gap):
    rng = np.random.default_rng(100 + gap)
    lens = BOUNDS + [int(x) for x in rng.integers(0, 3000, 40)]
    A = rand_seqs(rng, lens)
    B = rand_seqs(rng, lens[::-1] + [700, 5])
    n = 1500
    pairs = np.stack([rng.integers(0, len(A), n), rng.integers(0, len(B), n)], 1)
    # every boundary length against a few others, with the shorter string on either side
    edge = [(i, j) for i in range(len(BOUNDS)) for j in (0, 1, 5, 10, 22, len(B) - 2, len(B) - 1)]
    pairs = np.concatenate([pairs, np.array(edge)])
    # plant related strings so that alignments are gapped and scores are high
    for k in range(0, 40):
        i, j = int(pairs[k, 0]), int(pairs[k, 1])
        src = bytearray(A[i])
        if len(src) > 10:
            del src[len(src) // 2]
            B[j] = bytes(src)
    check_vs_oracle(oracle, A, B, pairs, scoring(gap))


def test_long_pair_vs_oracle(gpu, oracle):
    rng = np.random.default_rng(7)
    a = rand_seqs(rng, [5000])[0]
    b = bytearray(a + rand_seqs(rng, [2000])[0])
    for p in range(100, 5000, 700):
        b[p] = ord("A")
    A, B = [a, rand_seqs(rng, [7000])[0]], [bytes(b), a[:6999]]
    check_vs_oracle(oracle, A, B, np.array([[0, 0], [1, 1], [1, 0], [0, 1]]), scoring(-2))
    check_vs_oracle(oracle, B, A, np.array([[0, 0], [1, 1]]), scoring(-1))
    align.pair_scores_arrays(A, B, np.array([[0, 0], [1, 1]]), scoring(-2), False)
    assert _lib.lib().pg_last_kernel() == b"sw_pair_long_kernel"


def test_default_matrix_and_int64_table(gpu, oracle):
    rng = np.random.default_rng(11)
    letters = bytes(range(ord("A"), ord("Z") + 1))
    lens = [0, 1, 31, 33, 100, 257, 600]
    A, B = rand_seqs(rng, lens, letters), rand_seqs(rng, lens[::-1], letters)
    pairs = np.array([(i, j) for i in range(len(A)) for j in range(len(B))])
    dm = align.Default
    lut = dm.FirstAlphabet.byte_lut()
    check_vs_oracle(oracle, A, B, pairs, align.NewScoring(None, -2), lut, lut, dm.scores)
    big = np.asarray(TEST_MAT, np.int64) * (1 << 33)
    A, B = rand_seqs(rng, lens), rand_seqs(rng, lens[::-1])
    check_vs_oracle(oracle, A, B, pairs, scoring(-(1 << 34), big), TEST_LUT, TEST_LUT, big)


def test_error_order_vs_oracle(gpu, oracle):
    A = [b"XACGT", b"ACXGT", b"ACGT", b"", b"ACGTX", b"X", b"AC" * 200 + b"X"]
    B = [b"ACGT", b"XCGT", b"ACGX", b"", b"X", b"AC" * 200 + b"XX"]
    pairs = np.array([(i, j) for i in range(len(A)) for j in range(len(B))])
    check_vs_oracle(oracle, A, B, pairs, scoring(-2))
    scores, errs = align.SmithWatermanPairScores(A, B, pairs, scoring(-2))
    assert str(errs[0]) == "Symbol X not in alphabet"


def test_pair_list_shapes(gpu, oracle):
    rng = np.random.default_rng(3)
    A = rand_seqs(rng, rng.integers(0, 400, 50))
    B = rand_seqs(rng, rng.integers(0, 400, 9))
    pairs = np.stack([rng.integers(0, 50, 300), rng.integers(0, 9, 300)], 1)
    pairs[100:150] = pairs[0]  # repeated pairs
    check_vs_oracle(oracle, A, B, pairs, scoring(-2))
    # A and B the same buffers (all-pairs of one read set)
    ba, oa = flatten(A)
    same = np.stack(np.triu_indices(50, 1), 1)
    got = align.pair_scores_arrays((ba, oa), (ba, oa), same, scoring(-2))
    want = oracle_pairs(oracle, A, A, same, TEST_LUT, TEST_LUT, TEST_MAT, -2)
    assert [tuple(x) for x in zip(*[g.tolist() for g in got])] == [tuple(w) for w in want]
    assert [len(x) for x in align.pair_scores_arrays(A, B, np.zeros((0, 2), np.int64), scoring())] == [0, 0, 0]


def test_pair_groups_match_one_group(gpu, monkeypatch):
    """A small group budget cuts one call into many pair groups; every output matches the one-group call."""
    rng = np.random.default_rng(13)
    A = rand_seqs(rng, rng.integers(0, 200, 60))
    B = rand_seqs(rng, rng.integers(0, 200, 40))
    A[3], B[5] = b"ACXGT", b"GGTXA"  # errors, with their positions, in several groups
    pairs = np.stack([rng.integers(0, len(A), 2000), rng.integers(0, len(B), 2000)], 1)

    def run():
        before = _lib.lib().pg_launch_count()
        out = ([align.pair_scores_arrays(A, B, pairs, scoring(-2), g) for g in (False, True)],
               align.SmithWatermanPairAligns(A, B, pairs, scoring(-2)), align.NeedlemanWunschPairAligns(A, B, pairs, scoring(-2)))
        return out, _lib.lib().pg_launch_count() - before

    def key(aligns):  # errors compare by their text
        return [(s, a, b, str(e)) for s, a, b, e in aligns]

    (scores, sw, nw), launches = run()
    monkeypatch.setenv("PG_GROUP_BYTES", str(8_000))  # about 240 pairs per score group, 9 per string group
    (g_scores, g_sw, g_nw), g_launches = run()
    assert g_launches > launches
    for w, x in zip(scores, g_scores):
        for a, b in zip(w, x):
            assert np.array_equal(a, b)
    assert key(g_sw) == key(sw) and key(g_nw) == key(nw)


def test_host_out_of_range_index_writes_nothing(gpu):
    A, B = [b"ACGT", b"GG"], [b"ACG"]
    ba, oa = flatten(A)
    bb, ob = flatten(B)
    m = scoring().SubstitutionMatrix
    table = np.ascontiguousarray(m.scores, np.int64)
    for pa_, pb_ in (([0, 2], [0, 0]), ([0, 1], [0, 1])):
        pa, pb = np.array(pa_, np.uint32), np.array(pb_, np.uint32)
        score, ec, ep = np.full(2, 77, np.int64), np.full(2, 77, np.int32), np.full(2, 77, np.int64)
        before = _lib.lib().pg_launch_count()
        for fn in (_lib.lib().pg_sw_score_pairs, _lib.lib().pg_nw_score_pairs):
            rc = fn(ba.ctypes.data, oa.ctypes.data, 2, bb.ctypes.data, ob.ctypes.data, 1, pa.ctypes.data, pb.ctypes.data, 2, TEST_LUT.ctypes.data,
                    TEST_LUT.ctypes.data, table.ctypes.data, 5, 5, -2, score.ctypes.data, ec.ctypes.data, ep.ctypes.data)
            assert rc == _lib.PG_ERR_ARG
        assert _lib.lib().pg_launch_count() == before
        assert (score == 77).all() and (ec == 77).all() and (ep == 77).all()


def _to_dev(seqs):
    import torch
    b, o = flatten(seqs)
    return torch.from_numpy(b.copy() if len(b) else np.zeros(1, np.uint8)).cuda(), torch.from_numpy(o.astype(np.int64)).cuda()


def test_dev_matches_host_and_flags_bad_indices(gpu):
    import torch
    rng = np.random.default_rng(5)
    A = rand_seqs(rng, list(rng.integers(0, 700, 200)) + [1500])
    B = rand_seqs(rng, list(rng.integers(0, 300, 80)) + [40])
    pairs = np.stack([rng.integers(0, len(A), 3000), rng.integers(0, len(B), 3000)], 1)
    da, oa = _to_dev(A)
    db, ob = _to_dev(B)
    ma, mb = max(len(x) for x in A), max(len(x) for x in B)
    for g in (False, True):
        want = align.pair_scores_arrays(A, B, pairs, scoring(-2), g)
        got = align.pair_scores_device(da, oa, ma, db, ob, mb, torch.from_numpy(pairs).cuda(), scoring(-2), g)
        torch.cuda.synchronize()
        for w, x in zip(want, got):
            assert np.array_equal(w, x.cpu().numpy())
        bad = pairs.copy()
        bad[7, 0] = len(A)
        bad[9, 1] = 1 << 31
        bad[11, 0] = (1 << 32) + 1  # must not wrap to the valid index 1
        bad[13, 1] = -2
        got = [x.cpu().numpy() for x in align.pair_scores_device(da, oa, ma, db, ob, mb, torch.from_numpy(bad).cuda(), scoring(-2), g)]
        ok = np.ones(len(pairs), bool)
        ok[[7, 9, 11, 13]] = False
        for w, x in zip(want, got):
            assert np.array_equal(w[ok], x[ok])
        assert (got[1][~ok] == 3).all() and (got[0][~ok] == 0).all() and (got[2][~ok] == -1).all()
        # a sequence longer than the max_len passed is flagged too, not read past its scratch row
        got = [x.cpu().numpy() for x in align.pair_scores_device(da, oa, ma - 1, db, ob, mb, torch.from_numpy(pairs).cuda(), scoring(-2), g)]
        longest = np.array([len(A[i]) for i in pairs[:, 0]]) == ma
        assert (got[1][longest] == 3).all() and np.array_equal(got[0][~longest], want[0][~longest])


@pytest.mark.parametrize("global_alignment", [False, True])
def test_cross_check_against_one_template_api(gpu, global_alignment):
    rng = np.random.default_rng(9)
    qs = rand_seqs(rng, rng.integers(0, 301, 10_000), b"ACGTN")
    t = rand_seqs(rng, [10_000])[0]
    n = len(qs)
    for query_is_a in (True, False):
        want = align.sw_scores_arrays(*flatten(qs), t, scoring(-2), query_is_a, global_alignment)
        if query_is_a:
            got = align.pair_scores_arrays(qs, [t], np.stack([np.arange(n), np.zeros(n, np.int64)], 1), scoring(-2), global_alignment)
        else:
            got = align.pair_scores_arrays([t], qs, np.stack([np.zeros(n, np.int64), np.arange(n)], 1), scoring(-2), global_alignment)
        for w, g in zip(want, got):
            assert np.array_equal(w, g), query_is_a


def test_aligned_strings_vs_oracle(gpu, oracle):
    rng = np.random.default_rng(21)
    A = rand_seqs(rng, [0, 1, 5, 40, 70, 100, 150, 300])
    B = [a[3:] + rand_seqs(rng, [10])[0] for a in A] + rand_seqs(rng, [65, 200])
    pairs = np.array([(i, j) for i in range(len(A)) for j in range(len(B))])
    for g, fn, ofn in ((False, align.SmithWatermanPairAligns, oracle.sw_align), (True, align.NeedlemanWunschPairAligns, oracle.nw_align)):
        got = fn(A, B, pairs, scoring(-2))
        for k, (i, j) in enumerate(pairs):
            w = ofn(A[i], B[j], TEST_LUT, TEST_LUT, TEST_MAT, -2)
            assert (got[k][0], got[k][1].encode(), got[k][2].encode()) == (w[0], w[1], w[2]), (g, i, j)
    # a short out_stride: PG_ITEM_UNSUPPORTED with the needed length
    ba, oa = flatten(A)
    bb, ob = flatten(B)
    pa, pb = np.array([7], np.uint32), np.array([7], np.uint32)
    table = np.ascontiguousarray(TEST_MAT, np.int64)
    for fn, ofn in ((_lib.lib().pg_sw_align_pairs, oracle.sw_align), (_lib.lib().pg_nw_align_pairs, oracle.nw_align)):
        score, ec, ep = np.zeros(1, np.int64), np.zeros(1, np.int32), np.zeros(1, np.int64)
        out_a, out_b, ln, st = np.zeros(8, np.uint8), np.zeros(8, np.uint8), np.zeros(1, np.uint32), np.zeros(1, np.int32)
        _lib.check(fn(ba.ctypes.data, oa.ctypes.data, len(A), bb.ctypes.data, ob.ctypes.data, len(B), pa.ctypes.data, pb.ctypes.data, 1,
                      TEST_LUT.ctypes.data, TEST_LUT.ctypes.data, table.ctypes.data, 5, 5, -2, score.ctypes.data, ec.ctypes.data, ep.ctypes.data,
                      out_a.ctypes.data, out_b.ctypes.data, 8, ln.ctypes.data, st.ctypes.data))
        w = ofn(A[7], B[7], TEST_LUT, TEST_LUT, TEST_MAT, -2)
        assert st[0] == _lib.PG_ITEM_UNSUPPORTED and ln[0] == len(w[1]) > 8 and score[0] == w[0], fn


def test_index_workflow(gpu, oracle):
    """Family reads -> sketches -> index top-k -> pairs -> scores; the best hit is in the query's family."""
    L, k, s, fam, n = 2000, 21, 500, 10, 80
    reads = synth.family_reads(n, L, family=fam)
    seqs = [bytes(reads[i * L:(i + 1) * L]) for i in range(n)]
    sk = mash.sketch_uniform(reads, n, L, k, s)
    qi, ri = np.arange(0, n, 5), np.array([i for i in range(n) if i % 5])  # two queries per family, the rest indexed
    ix = mash.SketchIndex(sk[ri])
    ref = np.asarray(ix.nearest(sk[qi], 4)[0]).astype(np.int64)
    assert (ref != 0xFFFFFFFF).all()
    pairs = np.stack([np.repeat(np.arange(len(qi)), 4), ref.reshape(-1)], 1)
    Q, R = [seqs[i] for i in qi], [seqs[i] for i in ri]
    score, ec, _ = align.pair_scores_arrays(Q, R, pairs, scoring(-2))
    assert not ec.any()
    want = oracle_pairs(oracle, Q, R, pairs[::3], TEST_LUT, TEST_LUT, TEST_MAT, -2)
    assert score[::3].tolist() == [w[0] for w in want]
    best = ri[pairs[np.arange(len(qi)) * 4 + score.reshape(-1, 4).argmax(1), 1]]
    assert ((best // fam) == (qi // fam)).all()


def test_hostcpp_pairs(gpu, tmp_path):
    src = os.path.join(ROOT, "hostcpp", "pairs_tests.cpp")
    exe = str(tmp_path / "pairs_tests")
    subprocess.check_call(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "hostcpp"), "-I", os.path.join(ROOT, "include"), src, "-o", exe,
                           "-L", os.path.join(ROOT, "poly_b200", "lib"), "-lpolyb200", "-Wl,-rpath," + os.path.join(ROOT, "poly_b200", "lib")])
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
