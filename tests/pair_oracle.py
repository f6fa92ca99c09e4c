"""ctypes binding of oracle/pair_oracle.c, the pair-list driver over the restated po_sw_score /
po_nw_score, in oracle/liboracle.so.  TEST INFRASTRUCTURE ONLY (tests/ and tools/bench_align_pairs.py)."""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

import oracle_ffi

SIGS = {
    "po_pair_scores": (C.c_int, [C.c_int] + [C.c_void_p] * 6 + [C.c_uint64] + [C.c_void_p] * 3 + [C.c_int, C.c_int64, C.c_int] + [C.c_void_p] * 3),
}
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        _LIB = oracle_ffi.bind(SIGS)
    return _LIB


flat = oracle_ffi.ragged  # a list of byte strings, or a (bases, offsets) tuple, as contiguous uint8 / uint64 arrays


def scores(A, B, pairs, lut_a, lut_b, table, gap, global_alignment=False, nthreads=None):
    """(score int64[n], err_code int32[n], err_pos int64[n]) of every (i, j) row of pairs."""
    ba, oa = flat(A)
    bb, ob = flat(B)
    pairs = np.asarray(pairs).reshape(-1, 2)
    pa = np.ascontiguousarray(pairs[:, 0], np.uint32)
    pb = np.ascontiguousarray(pairs[:, 1], np.uint32)
    assert (pa < len(oa) - 1).all() and (pb < len(ob) - 1).all()
    lut_a = np.ascontiguousarray(lut_a, np.int16)
    lut_b = np.ascontiguousarray(lut_b, np.int16)
    table = np.ascontiguousarray(table, np.int64)
    n = len(pa)
    sc, ec, ep = np.zeros(n, np.int64), np.zeros(n, np.int32), np.zeros(n, np.int64)
    rc = lib().po_pair_scores(int(global_alignment), ba.ctypes.data, oa.ctypes.data, bb.ctypes.data, ob.ctypes.data, pa.ctypes.data,
                              pb.ctypes.data, n, lut_a.ctypes.data, lut_b.ctypes.data, table.ctypes.data, table.shape[1], gap,
                              nthreads or len(os.sched_getaffinity(0)), sc.ctypes.data, ec.ctypes.data, ep.ctypes.data)
    assert rc == oracle_ffi.PO_OK, rc
    return sc, ec, ep
