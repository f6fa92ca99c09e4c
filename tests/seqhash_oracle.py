"""ctypes binding of oracle/seqhash_oracle.c, the CPU restatement of seqhash, in oracle/liboracle.so.

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__ (build and smoke) and tools/bench_seqhash.py's
parity check and CPU arm.  Never imported by poly_b200/.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

import oracle_ffi
from oracle_ffi import _b

TYPES = {"DNA": 0, "RNA": 1, "PROTEIN": 2}
SIGS = {
    "po_blake3": (None, [C.c_char_p, C.c_uint64, C.c_char_p]),
    "po_booth_least_rotation": (C.c_int64, [C.c_char_p, C.c_int64]),
    "po_rotate_sequence": (None, [C.c_char_p, C.c_int64, C.c_char_p]),
    "po_seqhash": (C.c_int, [C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_char_p, C.POINTER(C.c_int64)]),
    "po_seqhash_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                   C.c_void_p]),
}
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        _LIB = oracle_ffi.bind(SIGS)
    return _LIB


def blake3(data) -> bytes:
    d = _b(data)
    out = C.create_string_buffer(32)
    lib().po_blake3(d, len(d), out)
    return out.raw


def booth_least_rotation(seq) -> int:
    d = _b(seq)
    return lib().po_booth_least_rotation(d, len(d))


def rotate_sequence(seq) -> bytes:
    d = _b(seq)
    out = C.create_string_buffer(max(len(d), 1))
    lib().po_rotate_sequence(d, len(d), out)
    return out.raw[: len(d)]


def seqhash(seq, seq_type: str, circular: bool, double_stranded: bool):
    """(err code, digest bytes or None, error byte position) of seqhash.Hash on one sequence."""
    d = _b(seq)
    out = C.create_string_buffer(32)
    pos = C.c_int64(0)
    code = lib().po_seqhash(d, len(d), TYPES[seq_type], int(circular), int(double_stranded), out, C.byref(pos))
    return code, (out.raw if code == 0 else None), pos.value


def seqhash_string(seq, seq_type: str, circular: bool, double_stranded: bool):
    code, dig, _ = seqhash(seq, seq_type, circular, double_stranded)
    if code:
        return None
    return "v1_" + seq_type[0] + ("C" if circular else "L") + ("D" if double_stranded else "S") + "_" + dig.hex()


def seqhash_batch(seqs: np.ndarray, offsets: np.ndarray, seq_type: str, circular: bool, double_stranded: bool, nthreads: int = 1):
    """(digest n x 32 uint8, err_code int32[n], err_pos int64[n]) over a dense batch."""
    seqs = np.ascontiguousarray(seqs, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = len(offsets) - 1
    dig = np.zeros((n, 32), dtype=np.uint8)
    code = np.zeros(n, dtype=np.int32)
    pos = np.zeros(n, dtype=np.int64)
    rc = lib().po_seqhash_batch(seqs.ctypes.data, offsets.ctypes.data, n, TYPES[seq_type], int(circular), int(double_stranded),
                                nthreads, dig.ctypes.data, code.ctypes.data, pos.ctypes.data)
    assert rc == oracle_ffi.PO_OK, rc
    return dig, code, pos
