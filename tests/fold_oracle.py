"""ctypes binding of tests/fold_oracle.c, the CPU restatement of poly's fold package (Zuker).

TEST INFRASTRUCTURE ONLY (tests/ and tools/bench_fold.py).  The C file is compiled on first use into a
temporary directory, so nothing is written into the tree.  Its energy tables are read from
tests/golden/fold/energies.json."""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ENERGIES = os.path.join(_HERE, "golden", "fold", "energies.json")
OK, PANIC, UNSUPPORTED, NOT_NUCLEIC, INTERNAL = 0, 1, 2, 3, 4
TABLES = ("nearestNeighbors", "internalMismatches", "terminalMismatches", "danglingEnds", "triTetraLoops", "internalLoops", "bulgeLoops",
          "hairpinLoops")
_LIB = None


def energies() -> dict:
    with open(ENERGIES) as f:
        return json.load(f)


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="fold_oracle_"), "libfold_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-Wall",
                               os.path.join(_HERE, "fold_oracle.c"), "-o", out, "-lm"])
        L = C.CDLL(out)
        L.fo_set_table.restype = None
        L.fo_set_table.argtypes = [C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_void_p, C.c_void_p]
        L.fo_set_multibranch.restype = None
        L.fo_set_multibranch.argtypes = [C.c_int, C.c_void_p]
        L.fo_fold.restype = C.c_int
        L.fo_fold.argtypes = [C.c_char_p, C.c_int64, C.c_double, C.POINTER(C.c_double), C.c_char_p, C.POINTER(C.c_int64),
                              C.POINTER(C.c_void_p)]
        L.fo_probe.restype = C.c_int
        L.fo_probe.argtypes = [C.c_char_p, C.c_int64, C.c_double, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double)]
        L.fo_pair.restype = None
        L.fo_pair.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p]
        L.fo_free.restype = None
        L.fo_free.argtypes = [C.c_void_p]
        L.fo_fold_batch.restype = None
        L.fo_fold_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int]
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
    """(status, value) of stack / Bulge / hairpin / internalLoop / W on the filled context of seq."""
    code = {"stack": 0, "Bulge": 1, "hairpin": 2, "internalLoop": 3, "W": 4}[which]
    a = list(idx) + [0] * (4 - len(idx))
    out = C.c_double()
    st = lib().fo_probe(seq, len(seq), temp, code, a[0], a[1], a[2], a[3], C.byref(out))
    return st, out.value


def pair(seq: bytes, a: int, b: int, c: int, d: int) -> str:
    out = C.create_string_buffer(6)
    lib().fo_pair(seq, a, b, c, d, out)
    return out.value.decode()


def fold_batch(seqs, temp: float, threads: int = 16):
    """(mfe float64[n], dot-brackets [bytes], status int32[n]) over `threads` host threads."""
    raw = [bytes(s) for s in seqs]
    off = np.zeros(len(raw) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    flat = np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8)
    mfe = np.zeros(max(len(raw), 1), dtype=np.float64)
    db = np.zeros(max(int(off[-1]), 1), dtype=np.uint8)
    dbl = np.zeros(max(len(raw), 1), dtype=np.uint64)
    st = np.zeros(max(len(raw), 1), dtype=np.int32)
    lib().fo_fold_batch(flat.ctypes.data, off.ctypes.data, len(raw), temp, mfe.ctypes.data, db.ctypes.data, dbl.ctypes.data, st.ctypes.data, threads)
    dbs = [db[int(off[i]): int(off[i]) + int(dbl[i])].tobytes() for i in range(len(raw))]
    return mfe[: len(raw)], dbs, st[: len(raw)]
