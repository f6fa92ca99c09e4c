"""GPU tier: the host-pointer entry points reject ragged offsets that decrease inside the batch
(here [0, 6, 3, 9], which still rises end to end) with PG_ERR_ARG before any kernel is launched."""
import ctypes as C

import numpy as np
import pytest

from poly_b200 import _lib

pytestmark = pytest.mark.gpu

BAD = np.array([0, 6, 3, 9], dtype=np.uint64)
GOOD = np.array([0, 9], dtype=np.uint64)
N = len(BAD) - 1
SEQS = np.frombuffer(b"ACGTACGTA", dtype=np.uint8).copy()
LUT = np.full(256, -1, dtype=np.int16)
LUT[list(b"-ACGT")] = np.arange(5, dtype=np.int16)
TABLE = np.eye(5, dtype=np.int64) * 4 - 2


class Out:
    """Output buffers that stay alive for the whole call; out(dtype, n) is the address of a new one."""

    def __init__(self):
        self.keep = []

    def __call__(self, dtype, n=N):
        self.keep.append(np.zeros(n, dtype))
        return self.keep[-1].ctypes.data


def _p(a):
    return a.ctypes.data


def _score(L, name):
    o = Out()
    return getattr(L, name)(_p(SEQS), _p(BAD), N, _p(SEQS), len(SEQS), 1, _p(LUT), _p(LUT), _p(TABLE), 5, 5, -2,
                            o(np.int64), o(np.int32), o(np.int64))


def _align(L, name):
    o, stride = Out(), 32
    return getattr(L, name)(_p(SEQS), _p(BAD), N, _p(SEQS), len(SEQS), 1, _p(LUT), _p(LUT), _p(TABLE), 5, 5, -2,
                            o(np.int64), o(np.int32), o(np.int64), o(np.uint8, N * stride), o(np.uint8, N * stride), stride,
                            o(np.uint32), o(np.int32))


def _similarity_pairs(L):
    o = Out()
    sk, a, b = np.arange(9, dtype=np.uint32), np.array([0, 1], np.uint32), np.array([2, 2], np.uint32)
    return L.pg_mash_similarity_pairs(_p(sk), _p(BAD), N, _p(a), _p(b), 2, o(np.int64, 2), o(np.float64, 2), o(np.float64, 2), o(np.int32, 2))


def _find_sites(L, seq_off, pat_off):
    o, n = Out(), C.c_uint64(0)
    return L.pg_find_sites_batch(_p(SEQS), _p(seq_off), len(seq_off) - 1, _p(SEQS), _p(pat_off), len(pat_off) - 1, 0,
                                 o(np.uint32, 16), o(np.uint64, 16), o(np.uint32, 16), 16, C.byref(n))


def _tm(L):
    o = Out()
    return L.pg_tm_batch(_p(SEQS), _p(BAD), N, 500e-9, 50e-3, 0.0, o(np.float64), o(np.float64), o(np.float64), o(np.int32))


def _design_primers(L):
    o = Out()
    return L.pg_design_primers_batch(_p(SEQS), _p(BAD), N, 55.0, o(np.uint32), o(np.uint32), o(np.int32))


def _minimal_primer(L):
    o = Out()
    return L.pg_pcr_minimal_primer_batch(_p(SEQS), _p(BAD), N, 55.0, o(np.uint32), o(np.int32))


def _seqhash(L):
    o = Out()
    return L.pg_seqhash_batch(_p(SEQS), _p(BAD), N, 0, 0, o(np.uint8, 32 * N), o(np.int32), o(np.uint64))


def _least_rotation(L):
    o = Out()
    return L.pg_least_rotation_batch(_p(SEQS), _p(BAD), N, o(np.uint64))


def _sketch(L, multi):
    o, k, s = Out(), 3, 4
    args = (_p(SEQS), _p(BAD), N, k, s, 0, o(np.uint32, N * s), s, o(np.uint32), o(np.int32))
    return L.pg_mash_sketch_batch_multi(*args, None, 0) if multi else L.pg_mash_sketch_batch(*args)


CALLS = {
    "pg_mash_sketch_batch": lambda L: _sketch(L, False),
    "pg_mash_sketch_batch_multi": lambda L: _sketch(L, True),
    "pg_mash_similarity_pairs": _similarity_pairs,
    "pg_sw_score_batch": lambda L: _score(L, "pg_sw_score_batch"),
    "pg_nw_score_batch": lambda L: _score(L, "pg_nw_score_batch"),
    "pg_sw_align_batch": lambda L: _align(L, "pg_sw_align_batch"),
    "pg_nw_align_batch": lambda L: _align(L, "pg_nw_align_batch"),
    "pg_tm_batch": _tm,
    "pg_design_primers_batch": _design_primers,
    "pg_pcr_minimal_primer_batch": _minimal_primer,
    "pg_find_sites_batch-seq_offsets": lambda L: _find_sites(L, BAD, GOOD),
    "pg_find_sites_batch-pat_offsets": lambda L: _find_sites(L, GOOD, BAD),
    "pg_seqhash_batch": _seqhash,
    "pg_least_rotation_batch": _least_rotation,
}


@pytest.mark.parametrize("name", sorted(CALLS))
def test_decreasing_offsets_rejected_before_launch(gpu, name):
    L = gpu.lib()
    before = L.pg_launch_count()
    assert CALLS[name](L) == _lib.PG_ERR_ARG
    assert "offsets decrease at 1" in _lib.last_error()
    assert L.pg_launch_count() == before
