"""ctypes binding of oracle/clone_oracle.c, the CPU restatement of clone.go (CutWithEnzyme, CircularLigate,
GoldenGate), in oracle/liboracle.so, and a Python restatement of the deferred-hash ligation that libpolyb200
runs (DESIGN.md "Clone").

TEST INFRASTRUCTURE ONLY (tests/ and tools/bench_clone.py)."""
from __future__ import annotations

import ctypes as C
import struct

import numpy as np

import oracle_ffi
import seqhash_oracle

_LIB = None
OK, PANIC, UNSUPPORTED = 0, 1, 2
_vpp, _u64p, _i64p = C.POINTER(C.c_void_p), C.POINTER(C.c_uint64), C.POINTER(C.c_int64)
SIGS = {
    "co_free": (None, [C.c_void_p]),
    "co_cut": (C.c_int, [C.c_char_p, C.c_int64, C.c_int, C.c_int, C.c_char_p, C.c_int64, C.c_char_p, C.c_int64, C.c_char_p, C.c_int64,
                         C.c_int64, C.c_int64, _vpp, _u64p, _i64p]),
    "co_cut_batch": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                               C.c_int, C.c_void_p, C.c_void_p]),
    "co_circular_ligate": (None, [C.c_char_p, C.c_int64, _vpp, _u64p, _i64p, _vpp, _u64p, _i64p]),
}

# clone.GetBaseRestrictionEnzymes (clone.go:358-364): name -> (forward site, reverse site, skip, overhang length,
# recognition site)
BASE_ENZYMES = {
    "BsaI": (b"GGTCTC", b"GAGACC", 1, 4, b"GGTCTC"),
    "BbsI": (b"GAAGAC", b"GTCTTC", 2, 4, b"GAAGAC"),
    "BtgZI": (b"GCGATG", b"CATCGC", 10, 4, b"GCGATG"),
}


def lib():
    global _LIB
    if _LIB is None:
        _LIB = oracle_ffi.bind(SIGS)
    return _LIB


def _take(p: C.c_void_p, nbytes: int, count: int) -> list[bytes]:
    raw = C.string_at(p.value, nbytes) if nbytes else b""
    lib().co_free(p)
    out, i = [], 0
    for _ in range(count):
        (n,) = struct.unpack_from("<Q", raw, i)
        out.append(raw[i + 8: i + 8 + n])
        i += 8 + n
    return out


def _ser(strings) -> bytes:
    return b"".join(struct.pack("<Q", len(s)) + s for s in strings)


def _enzyme(enzyme):
    return BASE_ENZYMES[enzyme] if isinstance(enzyme, str) else enzyme


def cut(part: bytes, circular: bool, directional: bool, enzyme):
    """(status, [(Sequence, ForwardOverhang, ReverseOverhang), ...]) of CutWithEnzyme."""
    fsite, rsite, skip, ohl, recog = _enzyme(enzyme)
    p, nb, nf = C.c_void_p(), C.c_uint64(), C.c_int64()
    rc = lib().co_cut(part, len(part), int(circular), int(directional), fsite, len(fsite), rsite, len(rsite), recog, len(recog), skip, ohl,
                      C.byref(p), C.byref(nb), C.byref(nf))
    s = _take(p, nb.value, 3 * nf.value)
    return rc, [tuple(s[3 * i: 3 * i + 3]) for i in range(nf.value)]


def cut_counts(parts: np.ndarray, offsets: np.ndarray, circular: np.ndarray, enzymes, directional: bool, nthreads: int):
    """(fragment count, status) of every (part, enzyme) item on nthreads threads -- the timed CPU arm."""
    enz = [_enzyme(e) for e in enzymes]
    bufs = [C.create_string_buffer(s, len(s)) for e in enz for s in (e[0], e[1], e[4])]
    sites = (C.c_void_p * len(bufs))(*[C.addressof(b) for b in bufs])
    lens = np.array([len(s) for e in enz for s in (e[0], e[1], e[4])], np.int64)
    so = np.array([v for e in enz for v in (e[2], e[3])], np.int64)
    n = (len(offsets) - 1) * len(enz)
    nfrag, status = np.zeros(n, np.int64), np.zeros(n, np.int32)
    parts = np.ascontiguousarray(parts, np.uint8)
    offsets = np.ascontiguousarray(offsets, np.uint64)
    circ = np.ascontiguousarray(circular, np.uint8)
    rc = lib().co_cut_batch(parts.ctypes.data, offsets.ctypes.data, circ.ctypes.data, len(offsets) - 1, sites, lens.ctypes.data,
                            so.ctypes.data, len(enz), int(directional), nthreads, nfrag.ctypes.data, status.ctypes.data)
    assert rc == oracle_ffi.PO_OK, rc
    return nfrag, status


def circular_ligate(fragments):
    """(clones, loops) of CircularLigate, hashed eagerly at the reference's call sites."""
    buf = _ser([s for f in fragments for s in f])
    pc, cb, nc, pl, lb, nl = C.c_void_p(), C.c_uint64(), C.c_int64(), C.c_void_p(), C.c_uint64(), C.c_int64()
    lib().co_circular_ligate(buf, len(fragments), C.byref(pc), C.byref(cb), C.byref(nc), C.byref(pl), C.byref(lb), C.byref(nl))
    return _take(pc, cb.value, nc.value), _take(pl, lb.value, nl.value)


def golden_gate(parts, enzyme):
    """(status, clones, loops) of GoldenGate; parts = [(sequence, circular), ...].  A digest that panics
    (or is unsupported) makes the whole reaction do so, with no constructs."""
    frags = []
    for seq, circ in parts:
        rc, f = cut(seq, circ, True, enzyme)
        if rc:
            return rc, [], []
        frags += f
    clones, loops = circular_ligate(frags)
    return OK, clones, loops


# ---- the deferred-hash ligation (the design of libpolyb200's host enumeration) ------------------------------
_COMP = bytes.maketrans(b"ABCDGHKMNRSTVWYabcdghkmnrstvwy", b"TVGHCDMKNYSABWRtvghcdmknysabwr")
_ZERO = bytes(c if chr(c) in "ABCDGHKMNRSTVWYabcdghkmnrstvwy" else 0 for c in range(256))


def rc(s: bytes) -> bytes:
    """transform.ReverseComplement: unlisted bytes become 0"""
    return s.translate(_ZERO).translate(_COMP)[::-1]


def emits(fragments):
    """recurseLigate without hashing: the ordered list of (kind, kept, construct) it would hash.  kind 0 is a
    closed clone (clone.go:274), 1 a looping construct (:304).  kept is False when a later early return of an
    enclosing call drops the construct from that call's result (its hash still enters the set)."""
    out = []

    def rec(seed, used):
        fwd_oh, seq, rev_oh = seed
        if fwd_oh == rev_oh:
            out.append([0, True, fwd_oh + seq])
            return
        start = len(out)
        used = list(used)
        for nf in fragments:
            nseq, nfwd, nrev = nf
            new_seed, attached = None, False
            if rev_oh == nfwd:
                attached, new_seed = True, (fwd_oh, seq + rev_oh + nseq, nrev)
            if rev_oh == rc(nrev) and rev_oh != rc(rev_oh):
                attached, new_seed = True, (fwd_oh, seq + rev_oh + rc(nseq), rc(nfwd))
            if not attached:
                continue
            for u in used:
                if u[0] == nseq:
                    for e in out[start:]:
                        e[1] = False
                    out.append([1, True, u[1] + u[0] + u[2]])
                    return
            used.append(nf)
            rec(new_seed, used)

    for f in fragments:
        rec((f[1], f[0], f[2]), [])
    return out


def ligate_deferred(fragments):
    """(clones, loops) from emits() followed by one walk that keeps the first construct of each seqhash."""
    seen, clones, loops = set(), [], []
    for kind, kept, construct in emits(fragments):
        key = seqhash_oracle.seqhash_string(construct, "DNA", kind == 0, True) or ""
        if key in seen:
            continue
        seen.add(key)
        if kept:
            (clones if kind == 0 else loops).append(construct)
    return clones, loops
