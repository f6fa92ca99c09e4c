"""fold on the GPU: Zuker minimum free energy and dot-bracket structures of DNA and RNA.

Mirrors poly's fold package (fold/fold.go, fold/seqfold.go): `Zuker(seq, temp)` returns a `Result` with
`MinimumFreeEnergy()` and `DotBracket()`, through pg_fold_zuker_batch.  The fold itself runs in the CUDA
kernel (fold.cu); this module only marshals the batch and formats the reference's errors.

A byte >= 0x80 (strings.ToUpper would re-encode it) or a sequence longer than MAX_LEN nt is an
`UnsupportedError`; an input on which the reference panics (empty, 1 nt, a traceback index out of range)
is a `GoPanic` (DESIGN.md "Fold").
"""
from __future__ import annotations

import math
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib

BytesLike = Union[str, bytes, bytearray, np.ndarray]
MAX_LEN = 1024
ITEM_OK, ITEM_PANIC, ITEM_UNSUPPORTED, ITEM_NOT_NUCLEIC, ITEM_INTERNAL = 0, 1, 2, 3, 4


class UnsupportedError(ValueError):
    """The sequence holds a byte >= 0x80, or is longer than MAX_LEN nt."""


class Result:
    """fold.Result: the folded structure's minimum free energy and dot-bracket notation."""

    def __init__(self, mfe: float = math.inf, dot_bracket: str = ""):
        self._mfe = mfe
        self._db = dot_bracket

    def MinimumFreeEnergy(self) -> float:
        return self._mfe

    def DotBracket(self) -> str:
        return self._db

    def __repr__(self) -> str:
        return f"Result(mfe={self._mfe!r}, dot_bracket={self._db!r})"


def _as_bytes(seq: BytesLike) -> bytes:
    if isinstance(seq, str):
        return seq.encode("utf-8")
    if isinstance(seq, np.ndarray):
        return seq.astype(np.uint8, copy=False).tobytes()
    return bytes(seq)


def zuker_arrays(seqs: np.ndarray, offsets: np.ndarray, temp: float):
    """(mfe float64[n], dot_bracket uint8 laid out like seqs, db_len uint64[n], status int32[n]) of a dense host batch."""
    seqs = np.ascontiguousarray(seqs, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = len(offsets) - 1
    mfe = np.zeros(max(n, 1), dtype=np.float64)
    db = np.zeros(max(int(offsets[-1] - offsets[0]) if n else 0, 1), dtype=np.uint8)
    dbl = np.zeros(max(n, 1), dtype=np.uint64)
    st = np.zeros(max(n, 1), dtype=np.int32)
    rc = _lib.lib().pg_fold_zuker_batch(seqs.ctypes.data, offsets.ctypes.data, n, float(temp), mfe.ctypes.data, db.ctypes.data, dbl.ctypes.data,
                                        st.ctypes.data)
    _lib.check(rc, allow=(_lib.PG_ERR_PANIC, _lib.PG_ERR_UNSUPPORTED))
    return mfe[:n], db, dbl[:n], st[:n]


def _item_error(status: int, raw: bytes) -> Exception:
    if status == ITEM_NOT_NUCLEIC:
        return ValueError("error creating folding context: the sequence " + raw.decode("ascii").upper() + " is not RNA or DNA")
    if status == ITEM_PANIC:
        return _lib.GoPanic("fold.Zuker panics on this sequence (index out of range)")
    if status == ITEM_UNSUPPORTED:
        return UnsupportedError(f"a byte >= 0x80 or more than {MAX_LEN} nt (unsupported)")
    return RuntimeError("fold.Zuker: an internal error of the reference fired on this sequence")


def ZukerBatch(seqs: Sequence[BytesLike], temp: float) -> List[Tuple[Optional[Result], Optional[Exception]]]:
    """Zuker of every sequence in one GPU call: a (Result, error) pair per item.  Where the reference panics
    the pair is (None, GoPanic); unsupported input gives (None, UnsupportedError); the reference's errors give
    (Result(), error)."""
    raw = [_as_bytes(s) for s in seqs]
    if not raw:
        return []
    off = np.zeros(len(raw) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    flat = np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8)
    mfe, db, dbl, st = zuker_arrays(flat, off, temp)
    out = []
    for i, r in enumerate(raw):
        s = int(st[i])
        if s == ITEM_OK:
            b = int(off[i])
            out.append((Result(float(mfe[i]), db[b: b + int(dbl[i])].tobytes().decode("ascii")), None))
        elif s in (ITEM_NOT_NUCLEIC, ITEM_INTERNAL):  # the reference returns (Result{}, err) for its errors
            out.append((Result(), _item_error(s, r)))
        else:
            out.append((None, _item_error(s, r)))
    return out


def Zuker(seq: BytesLike, temp: float) -> Tuple[Result, Optional[Exception]]:
    """fold.Zuker (fold.go:56): (Result, error).  Raises GoPanic where the reference panics."""
    res, err = ZukerBatch([seq], temp)[0]
    if res is None:
        raise err
    return res, err
