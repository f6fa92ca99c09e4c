"""seqhash on the GPU: Seqhash identifiers of DNA, RNA and protein sequences.

Mirrors /root/reference/seqhash/seqhash.go:141-223 (`Hash`) and :127-138 (`RotateSequence`) through
pg_seqhash_batch / pg_least_rotation_batch.  Every digest is computed by the CUDA kernels; this module
only marshals the batch and formats the reference's strings and errors.

Non-ASCII input (a byte >= 0x80 before any letter outside the alphabet) is not guessed at: the item's
result is an `UnsupportedError` (DESIGN.md §7).
"""
from __future__ import annotations

import ctypes as C
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib

BytesLike = Union[str, bytes, bytearray, np.ndarray]

DNA, RNA, PROTEIN = "DNA", "RNA", "PROTEIN"  # seqhash.go:64-68
_TYPES = {DNA: 0, RNA: 1, PROTEIN: 2}
CIRCULAR, DOUBLE_STRANDED = 1, 2


class UnsupportedError(ValueError):
    """The sequence holds a byte >= 0x80 where strings.ToUpper would re-encode it."""


def _as_bytes(seq: BytesLike) -> bytes:
    if isinstance(seq, str):
        return seq.encode("utf-8")
    if isinstance(seq, np.ndarray):
        return seq.astype(np.uint8, copy=False).tobytes()
    return bytes(seq)


def _flatten(seqs: Sequence[BytesLike]) -> Tuple[np.ndarray, np.ndarray, List[bytes]]:
    raw = [_as_bytes(s) for s in seqs]
    off = np.zeros(len(raw) + 1, dtype=np.uint64)
    np.cumsum([len(r) for r in raw], out=off[1:])
    return np.frombuffer(b"".join(raw) or b"\0", dtype=np.uint8), off, raw


def type_error(sequence_type: str) -> ValueError:
    return ValueError("Only sequenceTypes of DNA, RNA, or PROTEIN allowed. Got sequenceType: " + str(sequence_type))


def item_error(code: int, pos: int, seq: bytes, sequence_type: str) -> Optional[Exception]:
    """The reference's error for err_code / err_pos of one item (None for 0)."""
    if code == 0:
        return None
    if code == 1:
        letter = chr(seq[pos]).upper()
        if sequence_type == PROTEIN:
            return ValueError("Only letters ACDEFGHIKLMNPQRSTVWYUO*BXZ are allowed for Proteins. Got letter: " + letter)
        return ValueError("Only letters ATUGCYRSWKMBDHVNZ are allowed for DNA/RNA. Got letter: " + letter)
    if code == 2:
        return ValueError("Proteins cannot be double stranded")
    return UnsupportedError(f"byte 0x{seq[pos]:02x} at {pos} is not ASCII: strings.ToUpper would re-encode it (unsupported)")


def format_hash(digest: bytes, sequence_type: str, circular: bool, double_stranded: bool) -> str:
    """seqhash.go:196-221: "v1_" + metadata + "_" + hex."""
    return "v1_" + sequence_type[0] + ("C" if circular else "L") + ("D" if double_stranded else "S") + "_" + bytes(digest).hex()


def _flags(circular: bool, double_stranded: bool) -> int:
    return (CIRCULAR if circular else 0) | (DOUBLE_STRANDED if double_stranded else 0)


def hash_arrays(seqs: np.ndarray, offsets: np.ndarray, sequence_type: str, circular: bool, double_stranded: bool):
    """(digest uint8[n, 32], err_code int32[n], err_pos uint64[n]) of a dense host batch."""
    if sequence_type not in _TYPES:
        raise type_error(sequence_type)
    seqs = np.ascontiguousarray(seqs, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = len(offsets) - 1
    digest = np.zeros((max(n, 1), 32), dtype=np.uint8)
    code = np.zeros(max(n, 1), dtype=np.int32)
    pos = np.zeros(max(n, 1), dtype=np.uint64)
    _lib.check(_lib.lib().pg_seqhash_batch(seqs.ctypes.data, offsets.ctypes.data, n, _TYPES[sequence_type], _flags(circular, double_stranded),
                                           digest.ctypes.data, code.ctypes.data, pos.ctypes.data))
    return digest[:n], code[:n], pos[:n]


def HashBatch(sequences: Sequence[BytesLike], sequenceType: str, circular: bool, doubleStranded: bool) -> List[Tuple[str, Optional[Exception]]]:
    """Hash of every sequence in one GPU call: a (seqhash, error) pair per item."""
    if sequenceType not in _TYPES:
        return [("", type_error(sequenceType)) for _ in sequences]
    if not len(sequences):
        return []
    flat, off, raw = _flatten(sequences)
    digest, code, pos = hash_arrays(flat, off, sequenceType, circular, doubleStranded)
    out = []
    for i, r in enumerate(raw):
        err = item_error(int(code[i]), int(pos[i]), r, sequenceType)
        out.append(("", err) if err else (format_hash(digest[i], sequenceType, circular, doubleStranded), None))
    return out


def Hash(sequence: BytesLike, sequenceType: str, circular: bool, doubleStranded: bool) -> Tuple[str, Optional[Exception]]:
    """seqhash.Hash (seqhash.go:141): (seqhash, error)."""
    return HashBatch([sequence], sequenceType, circular, doubleStranded)[0]


def least_rotations(sequences: Sequence[BytesLike]) -> np.ndarray:
    """The smallest start of the least rotation of each sequence (raw bytes, no case folding)."""
    flat, off, _ = _flatten(sequences)
    rot = np.zeros(max(len(sequences), 1), dtype=np.uint64)
    _lib.check(_lib.lib().pg_least_rotation_batch(flat.ctypes.data, off.ctypes.data, len(sequences), rot.ctypes.data))
    return rot[: len(sequences)]


def RotateSequence(sequence: BytesLike) -> str:
    """seqhash.RotateSequence (seqhash.go:127)."""
    b = _as_bytes(sequence)
    r = int(least_rotations([b])[0])
    return (b[r:] + b[:r]).decode("latin-1")


def hash_device(d_seqs, d_offsets, n: int, max_len: int, sequenceType: str, circular: bool, doubleStranded: bool, stream=None):
    """pg_seqhash_batch_dev on torch CUDA tensors: (digest uint8[n, 32], err_code int32[n], err_pos int64[n]) on the device."""
    import torch

    if sequenceType not in _TYPES:
        raise type_error(sequenceType)
    dev = d_offsets.device
    digest = torch.empty((max(n, 1), 32), dtype=torch.uint8, device=dev)
    code = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    pos = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    st = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
    _lib.check(_lib.lib().pg_seqhash_batch_dev(d_seqs.data_ptr(), d_offsets.data_ptr(), n, _TYPES[sequenceType], _flags(circular, doubleStranded),
                                               digest.data_ptr(), code.data_ptr(), pos.data_ptr(), max_len, C.c_void_p(st)))
    return digest[:n], code[:n], pos[:n]


def hash_fasta_records(text: bytes, sequenceType: str = PROTEIN, circular: bool = False, doubleStranded: bool = False,
                       max_line_size: int = 2 * 32 * 1024):
    """Parse a FASTA text and Seqhash every record without the sequences leaving the device:
    pg_fasta_ingest_dev -> pg_seqhash_batch_dev.  Returns (digest uint8[n, 32], err_code, err_pos) as
    NumPy arrays and the FASTA error (fasta.FastaError or None) of the records before it."""
    import torch

    from . import fasta

    if sequenceType not in _TYPES:
        raise type_error(sequenceType)
    dev = torch.device("cuda", torch.cuda.current_device())
    d_text = torch.frombuffer(bytearray(text or b"\0"), dtype=torch.uint8).to(dev)
    cap_rec = text.count(b"\n") + 1
    d_bases = torch.empty(max(len(text), 1), dtype=torch.uint8, device=dev)
    d_off = torch.empty(cap_rec + 1, dtype=torch.int64, device=dev)
    n, tot, ntot, ec, el = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_int32(0), C.c_uint64(0)
    st = torch.cuda.current_stream(dev).cuda_stream
    _lib.check(_lib.lib().pg_fasta_ingest_dev(d_text.data_ptr(), len(text), max_line_size, fasta.BUFIO_ALIAS, d_bases.data_ptr(), d_bases.numel(),
                                              d_off.data_ptr(), None, 0, None, cap_rec, C.byref(n), C.byref(tot), C.byref(ntot), C.byref(ec),
                                              C.byref(el), C.c_void_p(st)))
    lens = d_off[1: n.value + 1] - d_off[: n.value]
    max_len = int(lens.max()) if n.value else 0
    digest, code, pos = hash_device(d_bases, d_off, n.value, max_len, sequenceType, circular, doubleStranded, st)
    err = fasta.FastaError(ec.value, el.value) if ec.value else None
    return digest.cpu().numpy(), code.cpu().numpy(), pos.cpu().numpy(), err
