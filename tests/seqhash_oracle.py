"""ctypes binding for oracle/libseqhash_oracle.so -- the CPU restatement of seqhash (oracle/seqhash_oracle.c).

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__ (build and smoke) and tools/bench_seqhash.py's
parity check and CPU arm.  Never imported by poly_b200/.  The library is built on its own, next to
oracle/liboracle.so, by build() below (called from __graft_entry__.build(), and again here when missing or stale).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_DIR = os.path.join(os.path.dirname(_HERE), "oracle")
SRC = os.path.join(ORACLE_DIR, "seqhash_oracle.c")
SO = os.path.join(ORACLE_DIR, "libseqhash_oracle.so")
TYPES = {"DNA": 0, "RNA": 1, "PROTEIN": 2}
_LIB = None


def build(force: bool = False) -> str:
    """Compile oracle/libseqhash_oracle.so when missing or stale, under an exclusive file lock (several test
    processes may get here at once), replacing the library atomically."""
    import fcntl

    def stale():
        return force or not os.path.exists(SO) or os.path.getmtime(SRC) > os.path.getmtime(SO)

    if stale():
        with open(os.path.join(ORACLE_DIR, ".build.lock"), "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if stale():
                tmp = os.path.join(ORACLE_DIR, f"libseqhash_oracle.{os.getpid()}.tmp.so")
                subprocess.check_call(["gcc", "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-pthread", "-shared", "-o", tmp, SRC])
                os.replace(tmp, SO)
    return SO


def lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.po_blake3.restype = None
        L.po_blake3.argtypes = [C.c_char_p, C.c_uint64, C.c_char_p]
        L.po_booth_least_rotation.restype = C.c_int64
        L.po_booth_least_rotation.argtypes = [C.c_char_p, C.c_int64]
        L.po_rotate_sequence.restype = None
        L.po_rotate_sequence.argtypes = [C.c_char_p, C.c_int64, C.c_char_p]
        L.po_seqhash.restype = C.c_int
        L.po_seqhash.argtypes = [C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_char_p, C.POINTER(C.c_int64)]
        L.po_seqhash_batch.restype = None
        L.po_seqhash_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _LIB = L
    return _LIB


def _b(s) -> bytes:
    return s.encode("latin-1") if isinstance(s, str) else bytes(s)


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
    lib().po_seqhash_batch(seqs.ctypes.data, offsets.ctypes.data, n, TYPES[seq_type], int(circular), int(double_stranded),
                           nthreads, dig.ctypes.data, code.ctypes.data, pos.ctypes.data)
    return dig, code, pos
