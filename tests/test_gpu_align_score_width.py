"""GPU tier: the alignment kernels at the limits of their score types.  Every kernel picks 2 x int16, int32 or int64
cells on the host (score_bound in poly_b200/csrc/align_core.cuh); each case here is built so that its exact score
lands on one of those limits -- planted perfect copies, so the maximum is reached and not only allowed -- and is
compared, as an exact integer (and as strings for the tracebacks), with the int64 C restatement of the reference.
int32 and int64 share kernel names, so on either side of that switch the score value is the evidence."""
import ctypes as C

import numpy as np
import pytest

import pair_oracle
from poly_b200 import _lib, align, synth
from poly_b200.mash import flatten
from test_oracle_align_primers import TEST_LUT, TEST_MAT

pytestmark = pytest.mark.gpu

LIMIT = 2_000_000_000  # a call takes 32-bit scores while its bound is below this (SCORE32_LIMIT)
INT32_MAX = 2**31 - 1
DNA = ["-", "A", "C", "G", "T"]
A5 = align.NewAlphabet(DNA)
LUT5 = A5.byte_lut()


def last_kernel():
    return _lib.lib().pg_last_kernel().decode()


def mat5(match, mismatch):
    """The '-' row and column score 0; A/C/G/T score `match` on the diagonal and `mismatch` off it."""
    m = np.zeros((5, 5), np.int64)
    m[1:, 1:] = mismatch
    m[np.arange(1, 5), np.arange(1, 5)] = match
    return m


def scoring(mat, gap, alpha=A5):
    return align.NewScoring(align.NewSubstitutionMatrix(alpha, alpha, mat), gap)


def rand(rng, n, letters=b"ACGT"):
    return bytes(rng.choice(list(letters), size=int(n)).astype(np.uint8))


def planted(rng, qs, tlen, letters=b"ACGT"):
    """A random template of tlen symbols holding a copy of every non-empty query (as many as fit)."""
    t = bytearray(rand(rng, tlen, letters))
    pos = 0
    for q in sorted((q for q in qs if q), key=len, reverse=True):
        if pos + len(q) > tlen:
            break
        t[pos:pos + len(q)] = q
        pos += len(q) + 3
    return bytes(t)


def batch_vs_oracle(oracle, qs, t, mat, gap, lut=LUT5, alpha=A5, global_alignment=False, kernel=None):
    """pg_sw/nw_score_batch in both orientations against po_sw_score / po_nw_score; returns the scores of query_is_a."""
    sc = scoring(mat, gap, alpha)
    ofn = oracle.nw_score if global_alignment else oracle.sw_score
    out = None
    for query_is_a in (True, False):
        got, errs = align.SmithWatermanScores(qs, t, sc, query_is_a=query_is_a, global_alignment=global_alignment)
        if kernel:
            assert last_kernel() == kernel, (query_is_a, last_kernel())
        want = [ofn(*((q, t) if query_is_a else (t, q)), lut, lut, mat, gap)[0] for q in qs]
        bad = [(i, len(qs[i]), got[i], want[i]) for i in range(len(qs)) if got[i] != want[i] or errs[i] is not None]
        assert not bad, (query_is_a, gap, bad[:4])
        out = out or got
    return out


def batch_dev(qs, t, mat, gap, lut=LUT5, global_alignment=False):
    """pg_sw/nw_score_batch_dev on device buffers: the scores, query_is_a = 1."""
    import torch

    b, o = flatten(qs)
    d_q = torch.from_numpy(b.copy() if len(b) else np.zeros(1, np.uint8)).cuda()
    d_o = torch.from_numpy(o.astype(np.int64)).cuda()
    d_t = torch.from_numpy(np.frombuffer(t, np.uint8).copy() if t else np.zeros(1, np.uint8)).cuda()
    n = len(qs)
    score = torch.empty(n, dtype=torch.int64, device="cuda")
    code = torch.empty(n, dtype=torch.int32, device="cuda")
    pos = torch.empty(n, dtype=torch.int64, device="cuda")
    table = np.ascontiguousarray(mat, np.int64)
    fn = _lib.lib().pg_nw_score_batch_dev if global_alignment else _lib.lib().pg_sw_score_batch_dev
    _lib.check(fn(d_q.data_ptr(), d_o.data_ptr(), n, max(len(q) for q in qs), d_t.data_ptr(), len(t), 1, lut.ctypes.data, lut.ctypes.data,
                  table.ctypes.data, table.shape[0], table.shape[1], gap, score.data_ptr(), code.data_ptr(), pos.data_ptr(),
                  C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert not code.any().item()
    return score.cpu().tolist()


def aligns_vs_oracle(oracle, qs, t, mat, gap, expect, global_alignment=False):
    """pg_sw/nw_align_batch in both orientations: the oracle's score and strings for every query ("ok"), or
    PG_ERR_UNSUPPORTED for the whole call ("unsupported")."""
    sc = scoring(mat, gap)
    ofn = oracle.nw_align if global_alignment else oracle.sw_align
    for query_is_a in (True, False):
        try:
            got = align.SmithWatermanAligns(qs, t, sc, query_is_a=query_is_a, global_alignment=global_alignment)
        except _lib.PolyError as e:
            assert expect == "unsupported" and e.code == _lib.PG_ERR_UNSUPPORTED, (expect, str(e))
            continue
        assert expect == "ok", [g[0] for g in got]
        for i, q in enumerate(qs):
            w = ofn(*((q, t) if query_is_a else (t, q)), LUT5, LUT5, mat, gap)
            assert (got[i][0], got[i][1].encode(), got[i][2].encode(), got[i][3]) == (w[0], w[1], w[2], None), (i, len(q), query_is_a, got[i][0], w[0])


def pairs_vs_oracle(oracle, A, B, pairs, mat, gap, global_alignment=False, lut=LUT5, alpha=A5, dev=True):
    """pg_sw/nw_score_pairs (and the _dev form) against the C pair driver over po_sw_score / po_nw_score."""
    sc = scoring(mat, gap, alpha)
    want = pair_oracle.scores(A, B, pairs, lut, lut, mat, gap, global_alignment)[0]
    got = align.pair_scores_arrays(A, B, pairs, sc, global_alignment)
    bad = [(k, len(A[pairs[k][0]]), len(B[pairs[k][1]]), int(got[0][k]), int(want[k])) for k in range(len(pairs)) if got[0][k] != want[k]]
    assert not bad and not got[1].any(), (gap, bad[:4])
    if dev:
        import torch

        def to_dev(seqs):
            b, o = flatten(seqs)
            return torch.from_numpy(b.copy()).cuda(), torch.from_numpy(o.astype(np.int64)).cuda()

        (da, oa), (db, ob) = to_dev(A), to_dev(B)
        d = align.pair_scores_device(da, oa, max(map(len, A)), db, ob, max(map(len, B)), torch.from_numpy(np.asarray(pairs)).cuda(), sc,
                                     global_alignment)
        torch.cuda.synchronize()
        assert d[0].cpu().tolist() == want.tolist() and not d[1].any().item(), gap
    return want


# ---- 2 x int16 (packed) <-> int32 ---------------------------------------------------------------------------------

@pytest.mark.parametrize("m,kernel", [(615, "sw_score_x2_kernel"), (616, "sw_score_kernel")])
def test_packed_int16_edge(gpu, oracle, m, kernel):
    """25-bp queries, local, gap -1: the bound is 26 max|S| = 15 990 (packed) or 16 016 (int32).  Planted copies
    reach 25 max|S| = 15 375 / 15 400; an odd batch with an empty query next to a full one."""
    rng = np.random.default_rng(m)
    qs = [rand(rng, 25) for _ in range(101)] + [rand(rng, rng.integers(0, 26)) for _ in range(30)]
    qs[6] = b""
    t = planted(rng, qs[:60], 2500)
    got = batch_vs_oracle(oracle, qs, t, mat5(m, -m), -1, kernel=kernel)
    assert max(got) == 25 * m and got[6] == 0


def test_cfg5_shape_takes_packed_kernel(gpu, oracle):
    """The headline primer shape (25-bp primers, +-3 table, gap -2, the 10 kb template) stays on the packed kernel."""
    n = 1001
    pr, off, tpl = synth.primers(n), synth.uniform_offsets(n, 25), synth.template()
    score, ec, _ = align.sw_scores_arrays(pr, off, tpl, scoring(TEST_MAT, -2))
    assert last_kernel() == "sw_score_x2_kernel" and not ec.any()
    for i in range(0, n, 50):
        assert score[i] == oracle.sw_score(bytes(pr[25 * i:25 * i + 25]), bytes(tpl), TEST_LUT, TEST_LUT, TEST_MAT, -2)[0], i


# ---- the top of int32: local alignments ---------------------------------------------------------------------------

def top_tables(qlen):
    """max|S| for a query of qlen symbols: the largest that keeps the bound max|S| (qlen + 1) under the limit
    (int32), one more (int64), and one whose perfect match scores 2^31 + a few (only int64 holds it)."""
    lo = (LIMIT - 1) // (qlen + 1)
    return [lo, lo + 1, 2**31 // qlen + 1]


@pytest.mark.parametrize("qlen,tlen,kernel", [(8, 400, "sw_score_kernel"), (25, 3000, "sw_score_kernel"), (32, 700, "sw_score_kernel"),
                                              (64, 900, "sw_score_kernel"), (100, 500, "sw_score_long_kernel")])
def test_local_int32_top(gpu, oracle, qlen, tlen, kernel):
    """Rows 8 / 32 / 64 and a query longer than 64 (global-memory column), both orientations: the last int32
    table, the first int64 one and a score past 2^31."""
    rng = np.random.default_rng(qlen)
    qs = [rand(rng, qlen) for _ in range(9)] + [rand(rng, rng.integers(0, qlen + 1)) for _ in range(24)] + [b""]
    t = planted(rng, qs[:9], tlen)
    for m in top_tables(qlen):
        mat = mat5(m, -m)
        got = batch_vs_oracle(oracle, qs, t, mat, -1, kernel=kernel)
        assert max(got) == qlen * m, (m, max(got))
        assert batch_dev(qs, t, mat, -1) == got
    if qlen == 25:  # bound 1 999 999 976 and score 1 923 076 900; int64; score 2^31 + 2
        assert top_tables(qlen) == [76_923_076, 76_923_077, 85_899_346]


@pytest.mark.parametrize("n_sym", [26, 255])
def test_local_int32_top_large_alphabets(gpu, oracle, n_sym):
    """No query profile (26 symbols), and a 255 x 255 table (no shared-memory copy at all); the pair calls keep the
    tables in shared memory (26) or read them from global memory (255: more than 48 KB)."""
    rng = np.random.default_rng(n_sym)
    codes = list(range(65, 91)) if n_sym == 26 else list(range(1, 256))
    alpha = align.NewAlphabet([chr(c) for c in codes])
    lut = alpha.byte_lut()
    letters = bytes(codes)
    qlen = 30
    qs = [rand(rng, qlen, letters) for _ in range(7)] + [rand(rng, rng.integers(0, qlen + 1), letters) for _ in range(10)] + [b""]
    t = planted(rng, qs[:7], 600, letters)
    for m in top_tables(qlen):
        mat = np.full((n_sym, n_sym), -m, np.int64)
        np.fill_diagonal(mat, m)
        got = batch_vs_oracle(oracle, qs, t, mat, -1, lut=lut, alpha=alpha, kernel="sw_score_kernel" if n_sym == 26 else "sw_score_long_kernel")
        assert max(got) == qlen * m
        A, B = qs[:17], [t]
        want = pairs_vs_oracle(oracle, A, B, [(i, 0) for i in range(len(A))], mat, -1, lut=lut, alpha=alpha)
        assert int(want.max()) == qlen * m


# ---- the bottom of int32: global alignments -----------------------------------------------------------------------

@pytest.mark.parametrize("rows,tlen,kernel", [(8, 3000, "nw_score_kernel"), (32, 3000, "nw_score_kernel"), (64, 2000, "nw_score_kernel"),
                                              (100, 1000, "sw_score_long_kernel"), (8, 0, "nw_score_kernel"), (64, 0, "nw_score_kernel")])
def test_global_int32_bottom(gpu, oracle, rows, tlen, kernel):
    """gap = -(limit / (sum + 2)): gap ramps and corners near -2e9 (the empty query scores tlen * gap, an empty
    template qlen * gap).  Queries of every length up to the row count, so the kernels run rows beyond the query."""
    rng = np.random.default_rng(rows + tlen)
    qs = [rand(rng, n) for n in range(rows + 1)] + [rand(rng, rows) for _ in range(4)]
    t = rand(rng, tlen)
    g = -((LIMIT - 1) // (rows + tlen + 2))
    for gap in (g, g - 1):  # int32, int64
        got = batch_vs_oracle(oracle, qs, t, TEST_MAT, gap, lut=TEST_LUT, global_alignment=True, kernel=kernel)
        assert min(got) == (tlen or rows) * gap < -1.5e9, (gap, min(got))
        assert batch_dev(qs, t, TEST_MAT, gap, lut=TEST_LUT, global_alignment=True) == got
    if rows <= 64 and tlen:  # the traceback reads the same values from its column ring
        aligns_vs_oracle(oracle, qs[::3], t, TEST_MAT, g, "ok" if rows == 64 else "unsupported", global_alignment=True)


# ---- positive gaps: values grow with the longer string ------------------------------------------------------------

def pos_gaps(sum_len):
    """+1, the largest gap whose values (about gap * sum) still fit int32 under the bound, and 2^20 (values ~ 3e9)."""
    return [1, (LIMIT - 1) // (sum_len + 2), 2**20]


@pytest.mark.parametrize("qlen,tlen,kernel", [(10, 3000, "sw_score_kernel"), (64, 3000, "sw_score_kernel"), (100, 2500, "sw_score_long_kernel")])
def test_positive_gap_batch(gpu, oracle, qlen, tlen, kernel):
    rng = np.random.default_rng(qlen * 3)
    qs = [rand(rng, qlen) for _ in range(3)] + [rand(rng, n) for n in rng.integers(0, qlen + 1, 12)] + [b""]
    t = planted(rng, qs[:3], tlen)
    for gap in pos_gaps(qlen + tlen):
        got = batch_vs_oracle(oracle, qs, t, TEST_MAT, gap, lut=TEST_LUT, kernel=kernel)
        assert batch_dev(qs, t, TEST_MAT, gap, lut=TEST_LUT) == got
        if gap > 1:  # a gap step beats half a match: the best path is all gaps, H[i][j] = (i + j - 1) gap
            assert max(got) == (qlen + tlen - 1) * gap
        if gap == 2**20:
            assert max(got) > INT32_MAX


@pytest.mark.parametrize("qlen,tlen", [(12, 300), (64, 3000)])
def test_positive_gap_align_batch(gpu, oracle, qlen, tlen):
    """The traceback kernels return the oracle's strings, or refuse the call: never a wrong score."""
    rng = np.random.default_rng(qlen + 5)
    qs = [rand(rng, qlen)] + [rand(rng, n) for n in rng.integers(0, qlen + 1, 6)]
    t = planted(rng, qs[:1], tlen)
    g1, mid, big = pos_gaps(qlen + tlen)
    aligns_vs_oracle(oracle, qs, t, TEST_MAT, g1, "ok")
    aligns_vs_oracle(oracle, qs[:3], t, TEST_MAT, mid, "ok" if qlen == 64 else "unsupported")
    aligns_vs_oracle(oracle, qs[:3], t, TEST_MAT, big, "unsupported" if tlen > 2000 else "ok")


# short classes R = 1 / 2 / 4 / 5 / 8 (shorter string <= 32 / 64 / 128 / 160 / 256 symbols) and long pairs
PAIR_SHORT = [20, 50, 100, 150, 200, 300]


@pytest.mark.parametrize("short", PAIR_SHORT)
def test_positive_gap_pairs(gpu, oracle, short):
    rng = np.random.default_rng(short)
    long_len = 2500
    S = [rand(rng, short), rand(rng, short - 7), b""]
    L = [rand(rng, long_len), rand(rng, long_len - 100)]
    for gap in pos_gaps(short + long_len):
        for A, B in ((S, L), (L, S)):  # the shorter string as a, then as b
            pairs = [(i, j) for i in range(len(A)) for j in range(len(B))]
            want = pairs_vs_oracle(oracle, A, B, pairs, TEST_MAT, gap)
            if gap > 1:
                assert int(want.max()) == (short + long_len - 1) * gap
    # aligned strings of pair lists: the oracle's, or PG_ERR_UNSUPPORTED
    A, B = S[:1], L[1:]
    for gap in pos_gaps(short + long_len - 100):
        try:
            got = align.SmithWatermanPairAligns(A, B, [(0, 0)], scoring(TEST_MAT, gap))
        except _lib.PolyError as e:
            assert e.code == _lib.PG_ERR_UNSUPPORTED and gap == 2**20, (gap, str(e))
            continue
        w = oracle.sw_align(A[0], B[0], LUT5, LUT5, TEST_MAT, gap)
        assert (got[0][0], got[0][1].encode(), got[0][2].encode()) == (w[0], w[1], w[2]), gap


# ---- pairs: the int32 / int64 switch ------------------------------------------------------------------------------

@pytest.mark.parametrize("short", [32, 64, 128, 160, 256, 300])
def test_pairs_local_int32_top(gpu, oracle, short):
    """Every short class at its own top (the bound follows the shorter of the call's longest a and b), and a long pair."""
    rng = np.random.default_rng(short + 1)
    S = [rand(rng, short), rand(rng, short - 5), rand(rng, 1)]
    L = [rand(rng, 20) + S[0] + rand(rng, 20), rand(rng, short + 40)]
    for m in top_tables(short):
        mat = mat5(m, -m)
        for A, B in ((S, L), (L, S)):
            pairs = [(i, j) for i in range(len(A)) for j in range(len(B))]
            want = pairs_vs_oracle(oracle, A, B, pairs, mat, -1)
            assert int(want.max()) == short * m


@pytest.mark.parametrize("short,long_len", [(40, 6000), (150, 6000), (300, 12000), (520, 12000)])
def test_pairs_global_int32_bottom(gpu, oracle, short, long_len):
    """NW pairs near -2e9; long pairs (> 256) hand each 256-row strip's bottom row to the next through global scratch."""
    rng = np.random.default_rng(short + 2)
    S = [rand(rng, short), rand(rng, short // 2)]
    L = [rand(rng, long_len), rand(rng, long_len - 1000)]
    g = -((LIMIT - 1) // (short + long_len + 2))
    for gap in (g, g - 1):
        for A, B in ((S, L), (L, S)):
            pairs = [(i, j) for i in range(len(A)) for j in range(len(B))]
            want = pairs_vs_oracle(oracle, A, B, pairs, TEST_MAT, gap, global_alignment=True)
            assert int(want.min()) < -1.5e9, int(want.min())
