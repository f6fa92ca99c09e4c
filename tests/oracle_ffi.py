"""ctypes binding for oracle/liboracle.so -- the CPU restatement of the reference -- and the one place
that builds and loads it.  The other binding modules (seqhash_oracle, clone_oracle, fold_oracle,
fragment_oracle, pair_oracle) keep their own signature tables and apply them to the same handle with bind().

TEST INFRASTRUCTURE ONLY: imported by tests/, __graft_entry__ (build and smoke) and bench.py's
cpu_baseline / --impl reference legs.  Never imported by poly_b200/.
"""
from __future__ import annotations

import ctypes as C
import glob
import importlib
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_DIR = os.path.join(os.path.dirname(_HERE), "oracle")
LIB_PATH = os.path.join(ORACLE_DIR, "liboracle.so")
BINDINGS = ("oracle_ffi", "seqhash_oracle", "clone_oracle", "fold_oracle", "fragment_oracle", "pair_oracle")
_LIB = None

PO_OK, PO_PANIC, PO_UNSUPPORTED = 0, -1, -2

_i32p, _i64p, _u64p, _f64p = C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_uint64), C.POINTER(C.c_double)
_ALIGN = [C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int64, _i64p]

SIGS = {
    "po_murmur3_32": (C.c_uint32, [C.c_char_p, C.c_size_t, C.c_uint32]),
    "po_mash_sketch_faithful": (C.c_int, [C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_void_p]),
    "po_mash_sketch_closed": (C.c_int, [C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_void_p]),
    "po_mash_similarity": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, _i64p, _f64p]),
    "po_mash_distance": (C.c_int, [C.c_void_p, C.c_int, C.c_void_p, C.c_int, _f64p]),
    "po_mash_sketch_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, _u64p]),
    "po_sw_score": (C.c_int, _ALIGN + [_i64p, _i64p, _i32p, _i64p]),
    "po_sw_align": (C.c_int, _ALIGN + [C.c_char_p, C.c_char_p, C.c_int64, _i64p, _i32p, _i64p]),
    "po_nw_align": (C.c_int, _ALIGN + [C.c_char_p, C.c_char_p, C.c_int64, _i64p, _i32p, _i64p]),
    "po_nw_score": (C.c_int, _ALIGN + [_i32p, _i64p]),
    "po_fastq_parse": (C.c_int, [C.c_char_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64, _u64p, _i32p, _u64p]),
    "po_fasta_parse": (C.c_int, [C.c_char_p, C.c_uint64, C.c_uint32, C.c_int, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_uint64,
                                 C.c_void_p, C.c_uint64, _u64p, _i32p, _u64p]),
    "po_reverse_complement": (None, [C.c_char_p, C.c_int64, C.c_char_p]),
    "po_santalucia": (C.c_int, [C.c_char_p, C.c_int64, C.c_double, C.c_double, C.c_double, _f64p, _f64p, _f64p]),
    "po_melting_temp": (C.c_int, [C.c_char_p, C.c_int64, _f64p]),
    "po_sw_score_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                    C.c_int64, C.c_int, C.c_void_p, _u64p]),
    "po_melting_temp_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_uint64, C.c_int, C.c_void_p, _u64p]),
    "po_mash_similarity_block": (C.c_int, [C.c_void_p, C.c_uint64, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, C.c_uint64, C.c_int,
                                           C.c_void_p, _u64p]),
}


def build(force: bool = False) -> str:
    """Compile oracle/liboracle.so (oracle/Makefile) when it is missing or older than any oracle/*.c, *.h or the
    Makefile.  Several ranks of a torchrun job may get here at once: the build runs under an exclusive file lock
    and replaces the library atomically."""
    import fcntl

    deps = glob.glob(os.path.join(ORACLE_DIR, "*.[ch]")) + [os.path.join(ORACLE_DIR, "Makefile")]

    def stale():
        return force or not os.path.exists(LIB_PATH) or any(os.path.getmtime(d) > os.path.getmtime(LIB_PATH) for d in deps)

    if stale():
        with open(os.path.join(ORACLE_DIR, ".build.lock"), "w") as lk:
            fcntl.flock(lk, fcntl.LOCK_EX)
            if stale():  # nobody built it while we waited
                tmp = f"liboracle.{os.getpid()}.tmp.so"
                subprocess.check_call(["make", "-C", ORACLE_DIR, "-s", "-B", f"OUT={tmp}"])
                os.replace(os.path.join(ORACLE_DIR, tmp), LIB_PATH)
    return LIB_PATH


def lib():
    """The one handle on liboracle.so (built first when missing or stale), with this module's table bound."""
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        bind(SIGS)
    return _LIB


def bind(sigs: dict):
    """Apply a {name: (restype, argtypes)} table to the shared handle and return the handle."""
    L = lib()
    for name, (res, args) in sigs.items():
        f = getattr(L, name)
        f.restype = res
        f.argtypes = args
    return L


def signatures() -> dict:
    """The signature tables of every binding module, merged: every oracle function bound in Python."""
    out = {}
    for m in BINDINGS:
        out.update(importlib.import_module(m).SIGS)
    return out


def _b(s) -> bytes:
    return s.encode("latin-1") if isinstance(s, str) else bytes(s)


def ragged(items):
    """(flat uint8, offsets uint64[n + 1]) of a sequence of str / bytes, with a NUL after the last item so that
    the pointer is valid for an empty list.  A (bases, offsets) tuple of arrays is returned as contiguous arrays."""
    if isinstance(items, tuple) and len(items) == 2 and isinstance(items[0], np.ndarray):
        return np.ascontiguousarray(items[0], np.uint8), np.ascontiguousarray(items[1], np.uint64)
    raw = [_b(s) for s in items]
    off = np.zeros(len(raw) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    return np.frombuffer(b"".join(raw) + b"\0", dtype=np.uint8).copy(), off


def murmur3_32(data, seed: int = 0) -> int:
    d = _b(data)
    return lib().po_murmur3_32(d, len(d), seed)


class OracleMash:
    """Mirror of mash.Mash (search/mash/mash.go:52-56) over the oracle."""

    def __init__(self, kmer_size: int, sketch_size: int):
        self.KmerSize, self.SketchSize = kmer_size, sketch_size
        self.Sketches = np.zeros(sketch_size, dtype=np.uint32)

    def Sketch(self, seq, faithful: bool = True) -> int:
        d = _b(seq)
        f = lib().po_mash_sketch_faithful if faithful else lib().po_mash_sketch_closed
        return f(d, len(d), self.KmerSize, self.SketchSize, self.Sketches.ctypes.data)

    def SimilarityCount(self, other: "OracleMash"):
        same, sim = C.c_int64(0), C.c_double(0)
        rc = lib().po_mash_similarity(self.Sketches.ctypes.data, self.SketchSize, other.Sketches.ctypes.data,
                                      other.SketchSize, C.byref(same), C.byref(sim))
        if rc != PO_OK:
            raise IndexError("reference would panic: index out of range")
        return same.value, sim.value

    def Similarity(self, other) -> float:
        return self.SimilarityCount(other)[1]

    def Distance(self, other) -> float:
        d = C.c_double(0)
        rc = lib().po_mash_distance(self.Sketches.ctypes.data, self.SketchSize, other.Sketches.ctypes.data, other.SketchSize, C.byref(d))
        if rc != PO_OK:
            raise IndexError("reference would panic: index out of range")
        return d.value


def sketch_batch(bases: np.ndarray, offsets: np.ndarray, k: int, s: int, variant: int = 1, nthreads: int = 1,
                 padded: bool = True):
    """Returns (rc, out[n,s] uint32) -- fresh zeroed sketch per read."""
    bases = np.ascontiguousarray(bases, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = len(offsets) - 1
    out = np.zeros((n, max(s, 0)), dtype=np.uint32)
    rc = lib().po_mash_sketch_batch(bases.ctypes.data, offsets.ctypes.data, n, k, s, variant, nthreads, out.ctypes.data, None)
    return rc, out


def sketch_batch_timing(bases, offsets, k, s, variant, nthreads):
    bases = np.ascontiguousarray(bases, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    ck = C.c_uint64(0)
    rc = lib().po_mash_sketch_batch(bases.ctypes.data, offsets.ctypes.data, len(offsets) - 1, k, s, variant, nthreads, None, C.byref(ck))
    return rc, ck.value


def sw_score(a, b, lut_a, lut_b, table, gap):
    """Returns (score, max_row, max_col, err_code, err_pos)."""
    a, b = _b(a), _b(b)
    lut_a = np.ascontiguousarray(lut_a, dtype=np.int16)
    lut_b = np.ascontiguousarray(lut_b, dtype=np.int16)
    table = np.ascontiguousarray(table, dtype=np.int64)
    sc, mr, mc, ep = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int64(0)
    ec = C.c_int32(0)
    rc = lib().po_sw_score(a, len(a), b, len(b), lut_a.ctypes.data, lut_b.ctypes.data, table.ctypes.data, table.shape[1], gap,
                           C.byref(sc), C.byref(mr), C.byref(mc), C.byref(ec), C.byref(ep))
    assert rc == PO_OK
    return sc.value, mr.value, mc.value, ec.value, ep.value


def nw_align(a, b, lut_a, lut_b, table, gap):
    """Returns (score, alignA, alignB, err_code, err_pos) of the full align.NeedlemanWunsch."""
    return sw_align(a, b, lut_a, lut_b, table, gap, _fn="po_nw_align")


def sw_align(a, b, lut_a, lut_b, table, gap, _fn="po_sw_align"):
    """Returns (score, alignA, alignB, err_code, err_pos) of the full align.SmithWaterman."""
    a, b = _b(a), _b(b)
    lut_a = np.ascontiguousarray(lut_a, dtype=np.int16)
    lut_b = np.ascontiguousarray(lut_b, dtype=np.int16)
    table = np.ascontiguousarray(table, dtype=np.int64)
    cap = len(a) + len(b) + 1
    oa, ob = C.create_string_buffer(cap), C.create_string_buffer(cap)
    sc, n, ep, ec = C.c_int64(0), C.c_int64(0), C.c_int64(0), C.c_int32(0)
    rc = getattr(lib(), _fn)(a, len(a), b, len(b), lut_a.ctypes.data, lut_b.ctypes.data, table.ctypes.data, table.shape[1], gap,
                           C.byref(sc), oa, ob, cap, C.byref(n), C.byref(ec), C.byref(ep))
    assert rc == PO_OK, rc
    return sc.value, oa.raw[: n.value], ob.raw[: n.value], ec.value, ep.value


def fastq_parse(text: bytes):
    """Returns (sequences list, err_code, err_line) as fastq.Parse would (valid prefix + error)."""
    cap = text.count(b"\n") // 4 + 2
    st, ln = np.zeros(cap, np.uint64), np.zeros(cap, np.uint64)
    n, ec, el = C.c_uint64(0), C.c_int32(0), C.c_uint64(0)
    rc = lib().po_fastq_parse(text, len(text), st.ctypes.data, ln.ctypes.data, cap, C.byref(n), C.byref(ec), C.byref(el))
    assert rc == PO_OK
    return [text[int(st[i]): int(st[i] + ln[i])] for i in range(n.value)], ec.value, el.value


def fasta_parse(text: bytes, max_line_size: int = 65536, alias: bool = True):
    """Returns ([(name, sequence)], err_code, err_line) as fasta.Parse / NewParser(r, max_line_size).ParseAll would."""
    cap = text.count(b"\n") + 2
    seq, name = np.zeros(len(text) + 1, np.uint8), np.zeros(len(text) + 1, np.uint8)
    so, no = np.zeros(cap + 1, np.uint64), np.zeros(cap + 1, np.uint64)
    n, ec, el = C.c_uint64(0), C.c_int32(0), C.c_uint64(0)
    rc = lib().po_fasta_parse(text, len(text), max_line_size, int(alias), seq.ctypes.data, len(seq), so.ctypes.data,
                              name.ctypes.data, len(name), no.ctypes.data, cap, C.byref(n), C.byref(ec), C.byref(el))
    assert rc == PO_OK
    sb, nb = seq.tobytes(), name.tobytes()
    recs = [(nb[int(no[i]): int(no[i + 1])], sb[int(so[i]): int(so[i + 1])]) for i in range(n.value)]
    return recs, ec.value, el.value


def nw_score(a, b, lut_a, lut_b, table, gap):
    a, b = _b(a), _b(b)
    lut_a = np.ascontiguousarray(lut_a, dtype=np.int16)
    lut_b = np.ascontiguousarray(lut_b, dtype=np.int16)
    table = np.ascontiguousarray(table, dtype=np.int64)
    sc, ep, ec = C.c_int64(0), C.c_int64(0), C.c_int32(0)
    rc = lib().po_nw_score(a, len(a), b, len(b), lut_a.ctypes.data, lut_b.ctypes.data, table.ctypes.data, table.shape[1], gap,
                           C.byref(sc), C.byref(ec), C.byref(ep))
    assert rc == PO_OK
    return sc.value, ec.value, ep.value


def reverse_complement(seq) -> bytes:
    d = _b(seq)
    out = C.create_string_buffer(len(d))
    lib().po_reverse_complement(d, len(d), out)
    return out.raw


def santalucia(seq, cp, na, mg):
    d = _b(seq)
    tm, dh, ds = C.c_double(0), C.c_double(0), C.c_double(0)
    rc = lib().po_santalucia(d, len(d), cp, na, mg, C.byref(tm), C.byref(dh), C.byref(ds))
    return rc, tm.value, dh.value, ds.value


def melting_temp(seq) -> float:
    rc, tm, _, _ = santalucia(seq, 500e-9, 50e-3, 0.0)
    if rc == PO_PANIC:
        raise IndexError("reference would panic: index out of range [-1]")
    if rc != PO_OK:
        raise ValueError("unsupported input")
    return tm


# ---- batch drivers (bench.py's CPU legs) ---------------------------------------------------------
def sw_score_batch(queries: np.ndarray, offsets: np.ndarray, templ: np.ndarray, lut_a, lut_b, table, gap: int, nthreads: int = 1):
    queries = np.ascontiguousarray(queries, dtype=np.uint8); offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    templ = np.ascontiguousarray(templ, dtype=np.uint8)
    lut_a = np.ascontiguousarray(lut_a, dtype=np.int16); lut_b = np.ascontiguousarray(lut_b, dtype=np.int16)
    table = np.ascontiguousarray(table, dtype=np.int64)
    n = len(offsets) - 1
    score = np.zeros(n, dtype=np.int64)
    rc = lib().po_sw_score_batch(queries.ctypes.data, offsets.ctypes.data, n, templ.ctypes.data, len(templ), lut_a.ctypes.data, lut_b.ctypes.data,
                                 table.ctypes.data, table.shape[1], gap, nthreads, score.ctypes.data, None)
    return rc, score


def melting_temp_batch(bases: np.ndarray, offsets: np.ndarray, nthreads: int = 1):
    bases = np.ascontiguousarray(bases, dtype=np.uint8); offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = len(offsets) - 1
    tm = np.zeros(n, dtype=np.float64)
    rc = lib().po_melting_temp_batch(bases.ctypes.data, offsets.ctypes.data, n, nthreads, tm.ctypes.data, None)
    return rc, tm


def similarity_block(sk: np.ndarray, row_lo: int, row_hi: int, col_lo: int, col_hi: int, nthreads: int = 1):
    sk = np.ascontiguousarray(sk, dtype=np.uint32)
    n, s = sk.shape
    same = np.zeros((row_hi - row_lo, col_hi - col_lo), dtype=np.uint32)
    rc = lib().po_mash_similarity_block(sk.ctypes.data, n, s, row_lo, row_hi, col_lo, col_hi, nthreads, same.ctypes.data, None)
    return rc, same
