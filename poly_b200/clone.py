"""clone on the GPU: restriction digests and Golden Gate assemblies.

Mirrors clone/clone.go of poly: `CutWithEnzyme` (:138-268), `CircularLigate` (:326-338), `GoldenGate`
(:342-355), the enzyme manager and `GetBaseRestrictionEnzymes` (:358-364), with the reference's names and
quirks.  The digest runs in CUDA kernels (pg_clone_digest_batch); the ligation recursion runs once, in
libpolyb200's host code, and every construct it closes is built and seqhashed on the device
(pg_clone_golden_gate_batch, pg_clone_circular_ligate_batch).  This module only marshals the batches.

Enzyme sites must be plain literals (the reference compiles them as regexps; this library does not
implement Go's regexp language): a pattern with a regexp metacharacter raises `UnsupportedError`, as does
a part with a byte >= 0x80 (strings.ToUpper would re-encode it).  Skip and OverheadLength must fit in
int32 (the C ABI's width); a wider value raises `UnsupportedError` rather than wrapping.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Dict, List, Sequence, Tuple

import numpy as np

from . import _lib
from .seqhash import UnsupportedError

_META = set("\\.+*?()|[]{}^$")


@dataclass
class Part:
    """A circular or linear DNA sequence (clone.go:56-59)."""

    Sequence: str
    Circular: bool = False


@dataclass
class Fragment:
    """A linear sequence with sticky ends (clone.go:70-74)."""

    Sequence: str
    ForwardOverhang: str
    ReverseOverhang: str


@dataclass
class Enzyme:
    """A restriction enzyme (clone.go:77-84).  RegexpFor / RegexpRev are the reference's patterns as
    strings; they must be literals."""

    Name: str
    RegexpFor: str
    RegexpRev: str
    Skip: int
    OverheadLength: int
    RecognitionSite: str

    def __post_init__(self):
        for p in (self.RegexpFor, self.RegexpRev):
            if not p or any(ch in _META for ch in p) or not p.isascii() or "\0" in p or len(p) > 32:
                raise UnsupportedError(f"enzyme {self.Name}: pattern {p!r} is not a literal of 1..32 ASCII bytes (only literal sites are supported)")
        for field in ("Skip", "OverheadLength"):  # pg_clone_enzyme holds them as int32; a wider value would wrap
            v = getattr(self, field)
            if not -(1 << 31) <= v < (1 << 31):
                raise UnsupportedError(f"enzyme {self.Name}: {field} = {v} is outside int32 (only -2^31 .. 2^31 - 1 are supported)")


class EnzymeNotFound(KeyError):
    def __str__(self):
        return self.args[0]


class EnzymeManager:
    """Enzymes by name (clone.go:88-107)."""

    def __init__(self, enzymes: Sequence[Enzyme]):
        self.enzymeMap: Dict[str, Enzyme] = {e.Name: e for e in enzymes}

    def GetEnzymeByName(self, name: str) -> Enzyme:
        if name in self.enzymeMap:
            return self.enzymeMap[name]
        raise EnzymeNotFound("Enzyme " + name + " not found")

    def CutWithEnzymeByName(self, part: Part, directional: bool, name: str) -> List[Fragment]:
        return CutWithEnzyme(part, directional, self.GetEnzymeByName(name))


def NewEnzymeManager(enzymes: Sequence[Enzyme]) -> EnzymeManager:
    return EnzymeManager(enzymes)


def GetBaseRestrictionEnzymes() -> List[Enzyme]:
    return [
        Enzyme("BsaI", "GGTCTC", "GAGACC", 1, 4, "GGTCTC"),
        Enzyme("BbsI", "GAAGAC", "GTCTTC", 2, 4, "GAAGAC"),
        Enzyme("BtgZI", "GCGATG", "CATCGC", 10, 4, "GCGATG"),
    ]


# ---- marshalling ------------------------------------------------------------------------------------------
class _Enzyme(C.Structure):
    _fields_ = [("forward_site", C.c_char_p), ("forward_len", C.c_uint32), ("reverse_site", C.c_char_p), ("reverse_len", C.c_uint32),
                ("recognition_site", C.c_char_p), ("recognition_len", C.c_uint32), ("skip", C.c_int32), ("overhang_length", C.c_int32)]


def _enzymes(enzymes: Sequence[Enzyme]):
    arr = (_Enzyme * len(enzymes))()
    keep = []
    for i, e in enumerate(enzymes):
        f, r, s = e.RegexpFor.encode(), e.RegexpRev.encode(), e.RecognitionSite.encode("utf-8")
        keep += [f, r, s]
        arr[i] = _Enzyme(f, len(f), r, len(r), s, len(s), e.Skip, e.OverheadLength)
    return arr, keep


def _b(s) -> bytes:
    return s.encode("utf-8") if isinstance(s, str) else bytes(s)


def _s(b: bytes) -> str:
    return b.decode("latin-1")


def _ragged(items: Sequence[bytes]):
    off = np.zeros(len(items) + 1, np.uint64)
    np.cumsum([len(x) for x in items], out=off[1:])
    return np.frombuffer(b"".join(items) or b"\0", np.uint8), off


def _item_error(status: int, what: str) -> Exception:
    if status == _lib.PG_ITEM_PANIC:
        return _lib.GoPanic(f"{what}: clone.CutWithEnzyme panics (slice bounds out of range)")
    return UnsupportedError(f"{what}: a byte >= 0x80 (strings.ToUpper would re-encode it; unsupported)")


def CutWithEnzymeBatch(parts: Sequence[Part], directional: bool, enzymes: Sequence[Enzyme]):
    """CutWithEnzyme(part, directional, enzyme) for every part x enzyme, in one call.  Returns
    (fragments, status): fragments[p][e] is the list of Fragments, status[p][e] a PG_ITEM_* code (a panic or
    unsupported item has no fragments)."""
    n, ne = len(parts), len(enzymes)
    if n == 0 or ne == 0:
        return [[[] for _ in range(ne)] for _ in range(n)], [[0] * ne for _ in range(n)]
    seqs, off = _ragged([_b(p.Sequence) for p in parts])
    circ = np.array([bool(p.Circular) for p in parts], np.uint8)
    enz, keep = _enzymes(enzymes)
    cnt, st = np.zeros(n * ne, np.uint32), np.zeros(n * ne, np.int32)
    nf, ns, no = C.c_uint64(), C.c_uint64(), C.c_uint64()
    caps = (0, 0, 0)
    L = _lib.lib()
    for _ in range(2):  # a first call with guessed capacities; the second, if needed, at the reported sizes
        fcap, scap, ocap = caps
        sb, so = np.zeros(max(scap, 1), np.uint8), np.zeros(fcap + 1, np.uint64)
        ob, oo = np.zeros(max(ocap, 1), np.uint8), np.zeros(2 * fcap + 1, np.uint64)
        rc = L.pg_clone_digest_batch(_lib.ptr(seqs), _lib.ptr(off), _lib.ptr(circ), n, C.cast(enz, C.c_void_p), ne, int(bool(directional)),
                                     _lib.ptr(cnt), _lib.ptr(st), _lib.ptr(sb), scap, _lib.ptr(so), _lib.ptr(ob), ocap, _lib.ptr(oo), fcap,
                                     C.byref(nf), C.byref(ns), C.byref(no))
        if rc != _lib.PG_ERR_ARG or (nf.value, ns.value, no.value) == caps:
            break
        caps = (nf.value, ns.value, no.value)
    _lib.check(rc, allow=(_lib.PG_ERR_PANIC, _lib.PG_ERR_UNSUPPORTED))
    del keep
    out, f = [], 0
    for p in range(n):
        row = []
        for e in range(ne):
            frs = []
            for _ in range(int(cnt[p * ne + e])):
                frs.append(Fragment(_s(sb[so[f]: so[f + 1]].tobytes()), _s(ob[oo[2 * f]: oo[2 * f + 1]].tobytes()),
                                    _s(ob[oo[2 * f + 1]: oo[2 * f + 2]].tobytes())))
                f += 1
            row.append(frs)
        out.append(row)
    return out, st.reshape(n, ne).tolist()


def CutWithEnzyme(part: Part, directional: bool, enzyme: Enzyme) -> List[Fragment]:
    """CutWithEnzyme (clone.go:138).  Raises GoPanic where the reference panics."""
    frags, st = CutWithEnzymeBatch([part], directional, [enzyme])
    if st[0][0]:
        raise _item_error(st[0][0], "CutWithEnzyme")
    return frags[0][0]


def _ligation_outputs(call, n_reactions: int, max_bytes: int, per_reaction: bool = True):
    """Runs call(bytes_cap, constructs_cap, outputs...) with growing buffers; returns per reaction
    (clones, loops, clone digests, loop digests) and the reaction statuses."""
    caps = (1 << 20, 1 << 12)
    L = _lib.lib()
    while True:
        bcap, ccap = caps
        out, coff = np.zeros(max(bcap, 1), np.uint8), np.zeros(ccap + 1, np.uint64)
        kinds, dig = np.zeros(max(ccap, 1), np.uint8), np.zeros((max(ccap, 1), 32), np.uint8)
        counts, st = np.zeros(2 * max(n_reactions, 1), np.uint64), np.zeros(max(n_reactions, 1), np.int32)
        nb, nc = C.c_uint64(), C.c_uint64()
        rc = call(L, bcap, ccap, _lib.ptr(out), _lib.ptr(coff), _lib.ptr(kinds), _lib.ptr(dig), _lib.ptr(counts), _lib.ptr(st), C.byref(nb), C.byref(nc))
        if rc == _lib.PG_ERR_ARG and (nb.value > bcap or nc.value > ccap):
            if nb.value > max_bytes:
                raise MemoryError(f"the ligation hashes {nb.value} bytes of constructs, more than max_bytes = {max_bytes}")
            caps = (max(bcap, nb.value), max(ccap, nc.value))
            continue
        if rc == _lib.PG_ERR_UNSUPPORTED and not per_reaction:  # the call refused its input: nothing was written
            raise UnsupportedError(_lib.last_error())
        _lib.check(rc, allow=(_lib.PG_ERR_PANIC, _lib.PG_ERR_UNSUPPORTED) if per_reaction else ())
        break
    res, k = [], 0
    for r in range(n_reactions):
        n = int(counts[2 * r] + counts[2 * r + 1])
        clones, loops, cd, ld = [], [], [], []
        for j in range(k, k + n):
            s = _s(out[coff[j]: coff[j + 1]].tobytes())
            (clones if kinds[j] == 0 else loops).append(s)
            (cd if kinds[j] == 0 else ld).append(dig[j].tobytes())
        k += n
        res.append((clones, loops, cd, ld))
    return res, st[:n_reactions].tolist()


def GoldenGateBatch(reactions: Sequence[Sequence[Part]], enzyme: Enzyme, max_bytes: int = 1 << 34, digests: bool = False):
    """GoldenGate(parts, enzyme) for every reaction in one call: a list of (clones, loops) per reaction (with
    digests=True, (clones, loops, clone digests, loop digests), each digest the 32 bytes of the construct's
    seqhash).  A reaction whose digest panics raises GoPanic, as GoldenGate would.  max_bytes bounds the
    bytes of all constructs the ligation hashes (MemoryError past it)."""
    parts = [p for r in reactions for p in r]
    seqs, off = _ragged([_b(p.Sequence) for p in parts])
    circ = np.array([bool(p.Circular) for p in parts] or [0], np.uint8)
    roff = np.zeros(len(reactions) + 1, np.uint64)
    np.cumsum([len(r) for r in reactions], out=roff[1:])
    enz, keep = _enzymes([enzyme])

    def call(L, bcap, ccap, *outs):
        return L.pg_clone_golden_gate_batch(_lib.ptr(seqs), _lib.ptr(off), _lib.ptr(circ), len(parts), _lib.ptr(roff), len(reactions),
                                            C.cast(enz, C.c_void_p), bcap, ccap, *outs)

    res, st = _ligation_outputs(call, len(reactions), max_bytes)
    del keep
    for r, s in enumerate(st):
        if s:
            raise _item_error(s, f"GoldenGate reaction {r}")
    return res if digests else [(c, l) for c, l, _, _ in res]


def GoldenGate(sequences: Sequence[Part], cuttingEnzyme: Enzyme) -> Tuple[List[str], List[str]]:
    """GoldenGate (clone.go:342): (openConstructs, infiniteLoops)."""
    return GoldenGateBatch([sequences], cuttingEnzyme)[0]


def CircularLigateBatch(reactions: Sequence[Sequence[Fragment]], max_bytes: int = 1 << 34, digests: bool = False):
    """CircularLigate for every list of fragments in one call; results as GoldenGateBatch.  A fragment with a
    byte >= 0x80 raises UnsupportedError (seqhash.Hash's strings.ToUpper would re-encode it)."""
    frags = [f for r in reactions for f in r]
    seqs, soff = _ragged([_b(f.Sequence) for f in frags])
    ohs, ooff = _ragged([_b(x) for f in frags for x in (f.ForwardOverhang, f.ReverseOverhang)])
    roff = np.zeros(len(reactions) + 1, np.uint64)
    np.cumsum([len(r) for r in reactions], out=roff[1:])

    def call(L, bcap, ccap, out, coff, kinds, dig, counts, st, nb, nc):
        return L.pg_clone_circular_ligate_batch(_lib.ptr(seqs), _lib.ptr(soff), _lib.ptr(ohs), _lib.ptr(ooff), len(frags), _lib.ptr(roff),
                                                len(reactions), bcap, ccap, out, coff, kinds, dig, counts, nb, nc)

    res, _ = _ligation_outputs(call, len(reactions), max_bytes, per_reaction=False)
    return res if digests else [(c, l) for c, l, _, _ in res]


def CircularLigate(fragments: Sequence[Fragment]) -> Tuple[List[str], List[str]]:
    """CircularLigate (clone.go:326): (outputConstructs, outputInfiniteLoopingConstructs)."""
    return CircularLigateBatch([fragments])[0]
