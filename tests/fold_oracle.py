"""ctypes binding of oracle/fold_oracle.c, the CPU restatement of poly's fold package (Zuker), in
oracle/liboracle.so.

TEST INFRASTRUCTURE ONLY (tests/ and tools/bench_fold.py).  Its energy tables are read from
tests/golden/fold/energies.json and handed to the library on first use."""
from __future__ import annotations

import ctypes as C
import json
import math
import os

import numpy as np

import oracle_ffi

_HERE = os.path.dirname(os.path.abspath(__file__))
ENERGIES = os.path.join(_HERE, "golden", "fold", "energies.json")
OK, PANIC, UNSUPPORTED, NOT_NUCLEIC, INTERNAL = 0, 1, 2, 3, 4
TABLES = ("nearestNeighbors", "internalMismatches", "terminalMismatches", "danglingEnds", "triTetraLoops", "internalLoops", "bulgeLoops",
          "hairpinLoops")
SIGS = {
    "fo_set_table": (None, [C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_void_p, C.c_void_p]),
    "fo_set_multibranch": (None, [C.c_int, C.c_void_p]),
    "fo_fold": (C.c_int, [C.c_char_p, C.c_int64, C.c_double, C.POINTER(C.c_double), C.c_char_p, C.POINTER(C.c_int64), C.POINTER(C.c_void_p)]),
    "fo_probe": (C.c_int, [C.c_char_p, C.c_int64, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double)]),
    "fo_pair": (None, [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p]),
    "fo_free": (None, [C.c_void_p]),
    "fo_fold_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]),
}
_LIB = None


def energies() -> dict:
    with open(ENERGIES) as f:
        return json.load(f)


def lib():
    global _LIB
    if _LIB is None:
        L = oracle_ffi.bind(SIGS)
        tabs = energies()
        for kind, name in enumerate(("dna", "rna")):
            t = tabs[name]
            L.fo_set_multibranch(kind, np.array(t["multibranch"], dtype=np.float64).ctypes.data)
            for ti, tname in enumerate(TABLES):
                ent = t.get(tname, {})
                keys = b"".join(k.encode().ljust(8, b"\0") for k in ent)
                h = np.array([v[0] for v in ent.values()] or [0.0], dtype=np.float64)
                s = np.array([v[1] for v in ent.values()] or [0.0], dtype=np.float64)
                L.fo_set_table(kind, ti, len(ent), keys or b"\0" * 8, h.ctypes.data, s.ctypes.data)
        _LIB = L
    return _LIB


def fold(seq: bytes, temp: float, with_structs: bool = False):
    """(status, mfe, dot_bracket bytes[, structs]) of Zuker(seq, temp) + MinimumFreeEnergy + DotBracket.
    structs: [(energy, description, [(start, end), ...]), ...] in the traceback's order."""
    mfe, n = C.c_double(), C.c_int64()
    buf = C.create_string_buffer(max(len(seq), 1))
    p = C.c_void_p()
    st = lib().fo_fold(seq, len(seq), temp, C.byref(mfe), buf, C.byref(n), C.byref(p) if with_structs else None)
    db = buf.raw[: n.value]
    if not with_structs:
        return st, mfe.value, db
    structs = []
    if p.value:
        text = C.string_at(p.value).decode()
        lib().fo_free(p)
        for line in text.splitlines():
            e, desc, inner = (line.split(" ") + [""])[:3]
            pairs = [tuple(int(x) for x in ij.split(",")) for ij in inner.split(";") if ij]
            structs.append((float.fromhex(e), "" if desc == "-" else desc, pairs))
    return st, mfe.value, db, structs


def probe(seq: bytes, temp: float, which: str, *idx) -> tuple:
    """(status, value) of stack / Bulge / hairpin / internalLoop / W on the filled context of seq, or of
    go_min on operands named by index (go_min below)."""
    code = {"stack": 0, "Bulge": 1, "hairpin": 2, "internalLoop": 3, "W": 4, "go_min": 5}[which]
    a = list(idx) + [0] * (4 - len(idx))
    out = C.c_double()
    st = lib().fo_probe(seq, len(seq), temp, code, a[0], a[1], a[2], a[3], C.byref(out))
    return st, out.value


def pair(seq: bytes, a: int, b: int, c: int, d: int) -> str:
    out = C.create_string_buffer(6)
    lib().fo_pair(seq, a, b, c, d, out)
    return out.value.decode()


GO_MIN_OPERANDS = (-math.inf, -1.0, -0.0, 0.0, 1.0, math.inf, math.nan)  # fold_oracle.c's go_min_operands


def go_min(a: float, b: float) -> float:
    """The restatement's math.Min of two operands from GO_MIN_OPERANDS."""
    ix = lambda x: next(i for i, v in enumerate(GO_MIN_OPERANDS) if (math.isnan(v) and math.isnan(x)) or
                        (v == x and math.copysign(1, v) == math.copysign(1, x)))
    st, out = probe(b"ACGT", 37.0, "go_min", ix(a), ix(b))
    assert st == OK
    return out


def fold_batch(seqs, temp: float, threads: int = 16):
    """(mfe float64[n], dot-brackets [bytes], status int32[n]) over `threads` host threads."""
    flat, off = oracle_ffi.ragged(seqs)
    n = len(off) - 1
    mfe = np.zeros(max(n, 1), dtype=np.float64)
    db = np.zeros(max(int(off[-1]), 1), dtype=np.uint8)
    dbl = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    rc = lib().fo_fold_batch(flat.ctypes.data, off.ctypes.data, n, temp, mfe.ctypes.data, db.ctypes.data, dbl.ctypes.data, st.ctypes.data, threads)
    assert rc == oracle_ffi.PO_OK, rc
    dbs = [db[int(off[i]): int(off[i]) + int(dbl[i])].tobytes() for i in range(n)]
    return mfe[:n], dbs, st[:n]
