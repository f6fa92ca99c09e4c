"""CPU tier for the pair-list alignment calls: without a usable GPU every new entry point fails
loudly with PG_ERR_NO_DEVICE (no CPU fallback), and the C pair driver the GPU tests compare against
equals the restated functions called pair by pair."""
import ctypes as C

import numpy as np
import pytest

import oracle_ffi
import pair_oracle
from poly_b200 import _lib, align
from test_oracle_align_primers import TEST_LUT, TEST_MAT

PAIR_CALLS = ("pg_sw_score_pairs", "pg_nw_score_pairs", "pg_sw_score_pairs_dev", "pg_nw_score_pairs_dev", "pg_sw_align_pairs",
              "pg_nw_align_pairs")


def _no_gpu():
    n = C.c_int(0)
    _lib.lib().pg_device_count(C.byref(n))
    return n.value == 0


def test_pair_calls_are_exported():
    for name in PAIR_CALLS:
        assert name in _lib.EXPORTS and hasattr(_lib.lib(), name)


@pytest.mark.skipif(not _no_gpu(), reason="this check is for the GPU-less tier")
def test_pair_calls_fail_without_a_device():
    seqs = np.frombuffer(b"ACGTACGT", np.uint8).copy()
    off = np.array([0, 4, 8], np.uint64)
    pa, pb = np.array([0, 1], np.uint32), np.array([1, 0], np.uint32)
    table = np.ascontiguousarray(TEST_MAT, np.int64)
    out = [np.zeros(2, np.int64), np.zeros(2, np.int32), np.zeros(2, np.int64)]
    common = [TEST_LUT.ctypes.data, TEST_LUT.ctypes.data, table.ctypes.data, 5, 5, -2] + [o.ctypes.data for o in out]
    host = [seqs.ctypes.data, off.ctypes.data, 2, seqs.ctypes.data, off.ctypes.data, 2, pa.ctypes.data, pb.ctypes.data, 2]
    dev = [seqs.ctypes.data, off.ctypes.data, 2, 4, seqs.ctypes.data, off.ctypes.data, 2, 4, pa.ctypes.data, pb.ctypes.data, 2]
    al = [np.zeros(16, np.uint8), np.zeros(16, np.uint8), np.zeros(2, np.uint32), np.zeros(2, np.int32)]
    lib = _lib.lib()
    assert lib.pg_sw_score_pairs(*host, *common) == _lib.PG_ERR_NO_DEVICE
    assert lib.pg_nw_score_pairs(*host, *common) == _lib.PG_ERR_NO_DEVICE
    assert lib.pg_sw_score_pairs_dev(*dev, *common, None) == _lib.PG_ERR_NO_DEVICE
    assert lib.pg_nw_score_pairs_dev(*dev, *common, None) == _lib.PG_ERR_NO_DEVICE
    tail = [al[0].ctypes.data, al[1].ctypes.data, 8, al[2].ctypes.data, al[3].ctypes.data]
    assert lib.pg_sw_align_pairs(*host, *common, *tail) == _lib.PG_ERR_NO_DEVICE
    assert lib.pg_nw_align_pairs(*host, *common, *tail) == _lib.PG_ERR_NO_DEVICE
    with pytest.raises(_lib.PolyError):
        align.SmithWatermanPairScores(["ACGT"], ["ACG"], [[0, 0]], align.NewScoring(None, -1))


@pytest.mark.parametrize("gap", [-3, -2, 0, 1])
def test_pair_driver_matches_per_pair_oracle(gap):
    """The C pair driver (oracle/pair_oracle.c) equals po_sw_score / po_nw_score called pair by pair, errors
    and empty strings included, on random pairs of two ragged sets."""
    rng = np.random.default_rng(40 + gap)
    A = [bytes(rng.choice(list(b"ACGT"), size=int(n)).astype(np.uint8)) for n in rng.integers(0, 300, 120)]
    B = [bytes(rng.choice(list(b"ACGT"), size=int(n)).astype(np.uint8)) for n in rng.integers(0, 300, 45)]
    A[3], A[4], B[5], B[6] = b"XACG", b"ACGX" * 20, b"", b"AXC"
    pairs = np.stack([rng.integers(0, len(A), 3000), rng.integers(0, len(B), 3000)], 1)
    pairs[:4] = [(3, 6), (4, 6), (3, 5), (4, 0)]
    for g in (False, True):
        got = list(zip(*(x.tolist() for x in pair_oracle.scores(A, B, pairs, TEST_LUT, TEST_LUT, TEST_MAT, gap, g, nthreads=4))))
        if g:
            want = [oracle_ffi.nw_score(A[i], B[j], TEST_LUT, TEST_LUT, TEST_MAT, gap) for i, j in pairs]
        else:
            want = [tuple(oracle_ffi.sw_score(A[i], B[j], TEST_LUT, TEST_LUT, TEST_MAT, gap)[k] for k in (0, 3, 4)) for i, j in pairs]
        assert got == [tuple(w) for w in want], g


def test_pairs_must_be_n_by_2():
    """A (2, n) array is not silently read as n pairs; the check runs before any library call."""
    sc = align.NewScoring(None, -1)
    with pytest.raises(ValueError, match=r"\(n, 2\)"):
        align.pair_scores_arrays(["ACGT", "AC", "G"], ["ACG", "T", "A"], np.array([[0, 1, 2], [2, 1, 0]]), sc)
    with pytest.raises(ValueError):
        align.pair_scores_arrays(["ACGT"], ["ACG"], np.array([0, 0]), sc)
    with pytest.raises(ValueError, match="2\\^32"):
        align.pair_scores_arrays(["ACGT"], ["ACG"], np.array([[-1, 0]]), sc)
