"""synthesis/fragment on the GPU: cut genes into synthesizable fragments with high-fidelity 4-nt overhangs.

Mirrors poly's synthesis/fragment (fragment.go): `Fragment`, `FragmentWithOverhangs`, `SetEfficiency`,
`NextOverhangs` and `NextOverhang`, with the reference's return shapes and error texts, through
pg_fragment_batch, pg_fragment_set_efficiency_batch and pg_fragment_next_overhangs_batch.  The batch forms
run many genes or sets in one GPU call.  A sequence shorter than 4 bytes makes the reference panic
(`GoPanic`); a byte >= 0x80 is an `UnsupportedError` (DESIGN.md "Fragment").
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib

BytesLike = Union[str, bytes, bytearray]
ITEM_OK, ITEM_PANIC, ITEM_UNSUPPORTED, ITEM_MIN_GT_MAX, ITEM_MIN_LT_12, ITEM_NO_POSITION = 0, 1, 2, 5, 6, 7


class UnsupportedError(ValueError):
    """The sequence holds a byte >= 0x80."""


def _as_bytes(s: BytesLike) -> bytes:
    return s.encode("utf-8") if isinstance(s, str) else bytes(s)


def _ragged(items) -> Tuple[np.ndarray, np.ndarray]:
    raw = [_as_bytes(s) for s in items]
    off = np.zeros(len(raw) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    return np.frombuffer(b"".join(raw) + b"\0", dtype=np.uint8), off


def fragment_arrays(seqs: np.ndarray, offsets: np.ndarray, min_size: int, max_size: int, exclude=(), include=(), ends_cap: Optional[int] = None):
    """(status int32[n], efficiency float64[n], err_min int64[n], err_max int64[n], frag_offsets uint64[n + 1], ends uint64[]) of a
    dense host batch.  ends_cap defaults to a guess, and the call is repeated once with the exact count if it was too small."""
    seqs = np.ascontiguousarray(seqs, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = len(offsets) - 1
    ex, exo = _ragged(exclude)
    inc, inco = _ragged(include)
    st, eff = np.zeros(max(n, 1), dtype=np.int32), np.zeros(max(n, 1))
    emin, emax = np.zeros(max(n, 1), dtype=np.int64), np.zeros(max(n, 1), dtype=np.int64)
    foff = np.zeros(n + 1, dtype=np.uint64)
    if ends_cap is None:
        ends_cap = int(offsets[-1] - offsets[0]) // max(min(int(min_size), int(max_size)) - 4, 8) + 2 * n if n else 0
    for _ in range(2):
        ends = np.zeros(max(ends_cap, 1), dtype=np.uint64)
        total = np.zeros(1, dtype=np.uint64)
        rc = _lib.lib().pg_fragment_batch(seqs.ctypes.data, offsets.ctypes.data, n, int(min_size), int(max_size), ex.ctypes.data, exo.ctypes.data,
                                          len(exclude), inc.ctypes.data, inco.ctypes.data, len(include), st.ctypes.data, eff.ctypes.data,
                                          emin.ctypes.data, emax.ctypes.data, foff.ctypes.data, ends.ctypes.data, ends_cap, total.ctypes.data)
        if rc == _lib.PG_ERR_ARG and int(total[0]) > ends_cap:
            ends_cap = int(total[0])
            continue
        _lib.check(rc, allow=(_lib.PG_ERR_PANIC, _lib.PG_ERR_UNSUPPORTED))
        return st[:n], eff[:n], emin[:n], emax[:n], foff, ends[: int(total[0])]
    raise RuntimeError("pg_fragment_batch: the end count changed between two calls")


def _item_error(status: int, emin: int, emax: int) -> Exception:
    if status == ITEM_MIN_GT_MAX:
        return ValueError(f"minFragmentSize ({emin}) larger than maxFragmentSize ({emax})")
    if status == ITEM_MIN_LT_12:
        return ValueError(f"minFragmentSize must be equal to or greater than 12 . Got size of {emin}")
    if status == ITEM_NO_POSITION:
        return ValueError("bestOverhangPosition failed by equaling zero")
    if status == ITEM_PANIC:
        return _lib.GoPanic("fragment.Fragment panics on a sequence shorter than 4 bytes (slice bounds out of range)")
    return UnsupportedError("a byte >= 0x80 (unsupported)")


def FragmentWithOverhangsBatch(seqs: Sequence[BytesLike], minFragmentSize: int, maxFragmentSize: int, excludeOverhangs: Sequence[BytesLike] = (),
                               includeOverhangs: Sequence[BytesLike] = ()) -> List[Tuple[Optional[List[str]], float, Optional[Exception]]]:
    """FragmentWithOverhangs of every sequence in one GPU call: (fragments, efficiency, error) per item.  The
    reference's errors give ([], 0, error); where it panics the item is (None, 0, GoPanic), and a byte >= 0x80
    gives (None, 0, UnsupportedError)."""
    raw = [_as_bytes(s) for s in seqs]
    if not raw:
        return []
    flat, off = _ragged(raw)
    st, eff, emin, emax, foff, ends = fragment_arrays(flat, off, minFragmentSize, maxFragmentSize, list(excludeOverhangs), list(includeOverhangs))
    out = []
    for i, r in enumerate(raw):
        s = int(st[i])
        if s == ITEM_OK:
            up = r.upper().decode("ascii")
            e = [int(x) for x in ends[int(foff[i]): int(foff[i + 1])]]
            out.append(([up[(e[k - 1] - 4 if k else 0): e[k]] for k in range(len(e))], float(eff[i]), None))
        elif s in (ITEM_PANIC, ITEM_UNSUPPORTED):
            out.append((None, 0.0, _item_error(s, 0, 0)))
        else:
            out.append(([], 0.0, _item_error(s, int(emin[i]), int(emax[i]))))
    return out


def FragmentBatch(seqs: Sequence[BytesLike], minFragmentSize: int, maxFragmentSize: int, excludeOverhangs: Sequence[BytesLike] = ()):
    """Fragment of every sequence in one GPU call (FragmentWithOverhangsBatch without includes)."""
    return FragmentWithOverhangsBatch(seqs, minFragmentSize, maxFragmentSize, excludeOverhangs, ())


def _one(res):
    frags, eff, err = res
    if frags is None:
        raise err
    return frags, eff, err


def Fragment(sequence: BytesLike, minFragmentSize: int, maxFragmentSize: int, excludeOverhangs: Sequence[BytesLike] = ()):
    """fragment.Fragment (fragment.go:191): (fragments, efficiency, error).  Raises GoPanic where the reference panics."""
    return _one(FragmentBatch([sequence], minFragmentSize, maxFragmentSize, excludeOverhangs)[0])


def FragmentWithOverhangs(sequence: BytesLike, minFragmentSize: int, maxFragmentSize: int, excludeOverhangs: Sequence[BytesLike] = (),
                          includeOverhangs: Sequence[BytesLike] = ()):
    """fragment.FragmentWithOverhangs (fragment.go:199): (fragments, efficiency, error)."""
    return _one(FragmentWithOverhangsBatch([sequence], minFragmentSize, maxFragmentSize, excludeOverhangs, includeOverhangs)[0])


def _sets(sets):
    flat, off = _ragged([o for s in sets for o in s])
    soff = np.zeros(len(sets) + 1, dtype=np.uint64)
    np.cumsum([len(s) for s in sets], out=soff[1:])
    return flat, off, soff


def SetEfficiencyBatch(sets: Sequence[Sequence[BytesLike]]) -> np.ndarray:
    """SetEfficiency of every set in one GPU call: float64[n]"""
    flat, off, soff = _sets(sets)
    eff = np.zeros(max(len(sets), 1))
    _lib.check(_lib.lib().pg_fragment_set_efficiency_batch(flat.ctypes.data, off.ctypes.data, soff.ctypes.data, len(sets), eff.ctypes.data))
    return eff[: len(sets)]


def SetEfficiency(overhangs: Sequence[BytesLike]) -> float:
    """fragment.SetEfficiency (fragment.go:24)"""
    return float(SetEfficiencyBatch([overhangs])[0])


def next_overhangs_arrays(sets: Sequence[Sequence[BytesLike]]):
    """(cands uint8[n, 256, 4], n_cands uint32[n], efficiency float64[n, 256]) of NextOverhangs over every set"""
    return next_overhangs_flat(*_sets(sets))


def next_overhangs_flat(flat: np.ndarray, off: np.ndarray, soff: np.ndarray):
    """next_overhangs_arrays of sets already flattened: set i is overhangs [soff[i], soff[i + 1]) of the ragged
    list (flat, off)"""
    flat = np.ascontiguousarray(flat, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.uint64)
    soff = np.ascontiguousarray(soff, dtype=np.uint64)
    n = len(soff) - 1
    cands = np.zeros((max(n, 1), 256, 4), dtype=np.uint8)
    nc = np.zeros(max(n, 1), dtype=np.uint32)
    eff = np.zeros((max(n, 1), 256))
    _lib.check(_lib.lib().pg_fragment_next_overhangs_batch(flat.ctypes.data, off.ctypes.data, soff.ctypes.data, n, cands.ctypes.data, nc.ctypes.data,
                                                           eff.ctypes.data))
    return cands[:n], nc[:n], eff[:n]


def NextOverhangsBatch(sets: Sequence[Sequence[BytesLike]]) -> List[Tuple[List[str], List[float]]]:
    """NextOverhangs of every set in one GPU call: (candidates, efficiencies) per set"""
    cands, nc, eff = next_overhangs_arrays(sets)
    return [([cands[i, j].tobytes().decode("ascii") for j in range(int(nc[i]))], [float(x) for x in eff[i, : int(nc[i])]]) for i in range(len(sets))]


def NextOverhangs(currentOverhangs: Sequence[BytesLike]) -> Tuple[List[str], List[float]]:
    """fragment.NextOverhangs (fragment.go:43)"""
    return NextOverhangsBatch([currentOverhangs])[0]


def NextOverhang(currentOverhangs: Sequence[BytesLike]) -> str:
    """fragment.NextOverhang (fragment.go:85): the first strict maximum above 0, or "" """
    cands, effs = NextOverhangs(currentOverhangs)
    best, out = 0.0, ""
    for c, e in zip(cands, effs):
        if e > best:
            best, out = e, c
    return out
