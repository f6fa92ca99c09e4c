"""ctypes binding of tests/fragment_oracle.c, the CPU restatement of poly's synthesis/fragment.

TEST INFRASTRUCTURE ONLY (tests/, smoke() and tools/bench_fragment.py).  The C file is compiled on first
use into a temporary directory, so nothing is written into the tree.  Its fidelity table is read from
tests/golden/fragment/ligation_fidelity.json."""
from __future__ import annotations

import ctypes as C
import json
import os
import subprocess
import tempfile

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
FIDELITY = os.path.join(_HERE, "golden", "fragment", "ligation_fidelity.json")
PINS = os.path.join(_HERE, "golden", "fragment", "pins.json")
OK, PANIC, UNSUPPORTED, MIN_GT_MAX, MIN_LT_12, NO_POSITION = 0, 1, 2, 3, 4, 5
_LIB = None


def fidelity() -> dict:
    with open(FIDELITY) as f:
        return json.load(f)


def pins() -> dict:
    with open(PINS) as f:
        return json.load(f)


def lib():
    global _LIB
    if _LIB is None:
        out = os.path.join(tempfile.mkdtemp(prefix="fragment_oracle_"), "libfragment_oracle.so")
        subprocess.check_call(["gcc", "-O2", "-std=gnu11", "-ffp-contract=off", "-fPIC", "-shared", "-pthread", "-Wall",
                               os.path.join(_HERE, "fragment_oracle.c"), "-o", out])
        L = C.CDLL(out)
        vp, u64, i64 = C.c_void_p, C.c_uint64, C.c_int64
        L.fr_set_table.restype = None
        L.fr_set_table.argtypes = [vp, vp]
        L.fr_set_efficiency.restype = C.c_double
        L.fr_set_efficiency.argtypes = [vp, vp, u64]
        L.fr_next_overhangs.restype = C.c_int
        L.fr_next_overhangs.argtypes = [vp, vp, u64, vp, vp]
        L.fr_fragment.restype = C.c_int
        L.fr_fragment.argtypes = [vp, i64, i64, i64, vp, vp, u64, vp, vp, u64, vp, vp, vp, vp, vp]
        L.fr_fragment_batch.restype = None
        L.fr_fragment_batch.argtypes = [vp, vp, u64, i64, i64, vp, vp, u64, vp, vp, u64, vp, vp, vp, vp, vp, vp, vp, C.c_int]
        L.fr_set_efficiency_batch.restype = None
        L.fr_set_efficiency_batch.argtypes = [vp, vp, vp, u64, vp, C.c_int]
        L.fr_next_overhangs_batch.restype = None
        L.fr_next_overhangs_batch.argtypes = [vp, vp, vp, u64, vp, vp, vp, C.c_int]
        t = fidelity()
        keys = np.frombuffer("".join(t["keys"]).encode(), dtype=np.uint8).copy()
        counts = np.array(t["counts"], dtype=np.int32)
        L.fr_set_table(keys.ctypes.data, counts.ctypes.data)
        _LIB = L
    return _LIB


def ragged(items):
    """(flat uint8, offsets uint64[n + 1]) of a list of str / bytes"""
    raw = [s.encode("latin-1") if isinstance(s, str) else bytes(s) for s in items]
    off = np.zeros(len(raw) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    return np.frombuffer(b"".join(raw) + b"\0", dtype=np.uint8).copy(), off


def max_ends(length: int) -> int:
    """the most fragment ends an item of `length` bytes can have: every step advances by at least 2 and
    needs at least 12 bytes left (DESIGN.md "Fragment")"""
    return (length - 12) // 2 + 2 if length >= 12 else 1


def fragment(seq, mn: int, mx: int, exclude=(), include=()):
    """(status, fragments [bytes], efficiency, err_min, err_max) of Fragment / FragmentWithOverhangs"""
    raw = seq.encode("latin-1") if isinstance(seq, str) else bytes(seq)
    s = np.frombuffer(raw + b"\0", dtype=np.uint8)
    ex, exo = ragged(exclude)
    inc, inco = ragged(include)
    ends = np.zeros(max_ends(len(raw)), dtype=np.uint64)
    eff, emin, emax, ne = C.c_double(), C.c_int64(), C.c_int64(), C.c_uint64()
    st = lib().fr_fragment(s.ctypes.data, len(raw), mn, mx, ex.ctypes.data, exo.ctypes.data, len(exclude), inc.ctypes.data, inco.ctypes.data,
                           len(include), C.byref(eff), C.byref(emin), C.byref(emax), ends.ctypes.data, C.byref(ne))
    up = raw.upper()
    e = [int(x) for x in ends[: ne.value]]
    frags = [up[(e[k - 1] - 4 if k else 0): e[k]] for k in range(len(e))]
    return st, frags, eff.value, emin.value, emax.value


def set_efficiency(overhangs) -> float:
    b, o = ragged(overhangs)
    return lib().fr_set_efficiency(b.ctypes.data, o.ctypes.data, len(overhangs))


def next_overhangs(overhangs):
    """(candidates [str], efficiencies [float]) of NextOverhangs"""
    b, o = ragged(overhangs)
    cands = np.zeros(1024, dtype=np.uint8)
    eff = np.zeros(256, dtype=np.float64)
    n = lib().fr_next_overhangs(b.ctypes.data, o.ctypes.data, len(overhangs), cands.ctypes.data, eff.ctypes.data)
    return [cands[4 * i: 4 * i + 4].tobytes().decode("latin-1") for i in range(n)], [float(x) for x in eff[:n]]


def fragment_batch(seqs, mn: int, mx: int, exclude=(), include=(), threads: int = 16):
    """(status int32[n], efficiency float64[n], err_min int64[n], err_max int64[n], ends [[int]]) over host threads"""
    flat, off = ragged(seqs)
    n = len(seqs)
    ex, exo = ragged(exclude)
    inc, inco = ragged(include)
    eoff = np.zeros(n + 1, dtype=np.uint64)
    np.cumsum([max_ends(int(off[i + 1] - off[i])) for i in range(n)], out=eoff[1:])
    ends = np.zeros(max(int(eoff[-1]), 1), dtype=np.uint64)
    st, ne = np.zeros(max(n, 1), dtype=np.int32), np.zeros(max(n, 1), dtype=np.uint64)
    eff, emin, emax = np.zeros(max(n, 1)), np.zeros(max(n, 1), dtype=np.int64), np.zeros(max(n, 1), dtype=np.int64)
    lib().fr_fragment_batch(flat.ctypes.data, off.ctypes.data, n, mn, mx, ex.ctypes.data, exo.ctypes.data, len(exclude), inc.ctypes.data,
                            inco.ctypes.data, len(include), st.ctypes.data, eff.ctypes.data, emin.ctypes.data, emax.ctypes.data, ends.ctypes.data,
                            eoff.ctypes.data, ne.ctypes.data, threads)
    return st[:n], eff[:n], emin[:n], emax[:n], [[int(x) for x in ends[int(eoff[i]): int(eoff[i]) + int(ne[i])]] for i in range(n)]


def _sets(sets):
    flat, off = ragged([o for s in sets for o in s])
    soff = np.zeros(len(sets) + 1, dtype=np.uint64)
    np.cumsum([len(s) for s in sets], out=soff[1:])
    return flat, off, soff


def set_efficiency_batch(sets, threads: int = 16) -> np.ndarray:
    flat, off, soff = _sets(sets)
    eff = np.zeros(max(len(sets), 1))
    lib().fr_set_efficiency_batch(flat.ctypes.data, off.ctypes.data, soff.ctypes.data, len(sets), eff.ctypes.data, threads)
    return eff[: len(sets)]


def next_overhangs_batch(sets, threads: int = 16):
    """(cands uint8[n, 256, 4], n_cands uint32[n], eff float64[n, 256])"""
    flat, off, soff = _sets(sets)
    n = len(sets)
    cands = np.zeros((max(n, 1), 256, 4), dtype=np.uint8)
    nc = np.zeros(max(n, 1), dtype=np.uint32)
    eff = np.zeros((max(n, 1), 256))
    lib().fr_next_overhangs_batch(flat.ctypes.data, off.ctypes.data, soff.ctypes.data, n, cands.ctypes.data, nc.ctypes.data, eff.ctypes.data, threads)
    return cands[:n], nc[:n], eff[:n]
