"""Host-side mirror of poly's search/mash package over libpolyb200.so.

Mirrors /root/reference/search/mash/mash.go: `New`, `Mash{KmerSize, SketchSize,
Sketches}`, `(*Mash).Sketch`, `Similarity`, `Distance` keep their names, argument
meaning and failure behaviour (a Go panic surfaces as `GoPanic`, an IndexError).
Batched entry points (`SketchBatch`, `sketch_uniform`, `DistanceMatrix`, ...) are
additions: a single-call API cannot feed a GPU (SURVEY.md 8b).

Every result is computed on the GPU through the C ABI -- there is no host compute
path here beyond marshalling.
"""
from __future__ import annotations

import ctypes as C
import threading
from typing import List, Optional, Sequence, Tuple, Union

import numpy as np

from . import _lib
from ._lib import GoPanic, PolyError

BytesLike = Union[str, bytes, bytearray, np.ndarray]


def _as_bytes(seq: BytesLike) -> np.ndarray:
    if isinstance(seq, str):
        seq = seq.encode("latin-1")  # Go strings are byte strings
    if isinstance(seq, (bytes, bytearray)):
        return np.frombuffer(bytes(seq), dtype=np.uint8)
    return np.ascontiguousarray(seq, dtype=np.uint8)


def flatten(seqs: Sequence[BytesLike]) -> Tuple[np.ndarray, np.ndarray]:
    """[]string -> (bases, offsets) as the C ABI wants them (cgo would do the same)."""
    arrs = [_as_bytes(s) for s in seqs]
    offsets = np.zeros(len(arrs) + 1, dtype=np.uint64)
    if arrs:
        offsets[1:] = np.cumsum([len(a) for a in arrs], dtype=np.uint64)
    bases = np.concatenate(arrs) if arrs else np.zeros(0, dtype=np.uint8)
    return np.ascontiguousarray(bases, dtype=np.uint8), offsets


class Mash:
    """mash.Mash (mash.go:52-56): exported, user-mutable fields."""

    __slots__ = ("KmerSize", "SketchSize", "Sketches")

    def __init__(self, kmer_size: int, sketch_size: int):
        if sketch_size < 0:
            raise GoPanic("makeslice: len out of range")  # mash.go:63
        self.KmerSize = int(kmer_size)
        self.SketchSize = int(sketch_size)
        self.Sketches = np.zeros(self.SketchSize, dtype=np.uint32)  # mash.go:59-65

    def Sketch(self, sequence: BytesLike) -> None:
        """(*Mash).Sketch (mash.go:68-104); mutates the receiver in place."""
        seq = _as_bytes(sequence)
        k, s = self.KmerSize, self.SketchSize
        n = len(seq) - k
        if n <= 0:
            return  # loop body never runs (mash.go:73)
        if k < 0:
            raise GoPanic("slice bounds out of range")  # sequence[i:i+k]
        cnt = min(n, s)
        out = np.zeros(max(cnt, 1), dtype=np.uint32)
        status = np.zeros(1, dtype=np.int32)
        rc = _lib.lib().pg_mash_sketch_uniform(seq.ctypes.data, 1, len(seq), k, s, 0, out.ctypes.data, cnt, status.ctypes.data)
        if rc == _lib.PG_ERR_PANIC or status[0] == _lib.PG_ITEM_PANIC:
            raise GoPanic("index out of range [-1]")  # mash.go:96-98 with sketchSize in {0,1}
        _lib.check(rc)
        # n < s: only the first n slots are overwritten (mash.go:81-84); n >= s: all s
        self.Sketches[:cnt] = out[:cnt]

    def _pair(self, other: "Mash") -> Tuple[int, float, float]:
        a = np.ascontiguousarray(self.Sketches[: self.SketchSize], dtype=np.uint32)
        b = np.ascontiguousarray(other.Sketches[: other.SketchSize], dtype=np.uint32)
        if len(a) < self.SketchSize or len(b) < other.SketchSize:
            raise GoPanic("index out of range")
        sk = np.concatenate([a, b])
        off = np.array([0, len(a), len(a) + len(b)], dtype=np.uint64)
        pa, pb = np.array([0], dtype=np.uint32), np.array([1], dtype=np.uint32)
        same, sim, dist = np.zeros(1, np.int64), np.zeros(1, np.float64), np.zeros(1, np.float64)
        st = np.zeros(1, np.int32)
        rc = _lib.lib().pg_mash_similarity_pairs(sk.ctypes.data, off.ctypes.data, 2, pa.ctypes.data, pb.ctypes.data, 1,
                                                 same.ctypes.data, sim.ctypes.data, dist.ctypes.data, st.ctypes.data)
        if rc == _lib.PG_ERR_PANIC:
            raise GoPanic("index out of range [-1]")  # Sketches[SketchSize-1] with size 0
        _lib.check(rc)
        return int(same[0]), float(sim[0]), float(dist[0])

    def Similarity(self, other: "Mash") -> float:
        """(*Mash).Similarity (mash.go:107-135)."""
        return self._pair(other)[1]

    def Distance(self, other: "Mash") -> float:
        """(*Mash).Distance (mash.go:138-140)."""
        return self._pair(other)[2]


def New(kmer_size: int, sketch_size: int) -> Mash:
    """mash.New (mash.go:59-65)."""
    return Mash(kmer_size, sketch_size)


# ---- batched additions ------------------------------------------------------------
def sketch_arrays(bases: np.ndarray, offsets: np.ndarray, k: int, s: int, pad_zero: bool = False):
    """Sketch every read of a flattened batch.  Returns (out[n, stride], count[n], status[n]);
    row i holds count[i] informative words (the zero tail of a fresh Mash is materialised only
    with pad_zero)."""
    bases = np.ascontiguousarray(bases, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = len(offsets) - 1
    lens = np.diff(offsets.astype(np.int64)) if n else np.zeros(0, np.int64)
    maxn = int(max(int(lens.max()) - k, 0)) if n else 0
    stride = s if pad_zero else min(maxn, s)
    out = np.zeros((n, max(stride, 1)), dtype=np.uint32)
    count = np.zeros(n, dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    rc = _lib.lib().pg_mash_sketch_batch(bases.ctypes.data, offsets.ctypes.data, n, k, s,
                                         _lib.PG_SKETCH_PAD_ZERO if pad_zero else 0, out.ctypes.data, max(stride, 1),
                                         count.ctypes.data, status.ctypes.data)
    _lib.check(rc, allow=(_lib.PG_ERR_PANIC,))
    return out, count, status


def sketch_into(bases: np.ndarray, offsets: np.ndarray, k: int, s: int, sketches: np.ndarray, devices=None):
    """The literal in-place form of (*Mash).Sketch for a batch: `sketches` is the caller's [n, s] uint32 array
    (the Sketches of n Mash values, e.g. one zeroed slab as Go's make gives); row i receives its min(L_i - k, s)
    words and the rest of the row is left as it was (mash.go:73-80 never writes Sketches[n:s]) --
    PG_SKETCH_TAIL_KEEP.  Returns (count, status)."""
    bases = np.ascontiguousarray(bases, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = len(offsets) - 1
    if sketches.dtype != np.uint32 or not sketches.flags.c_contiguous or sketches.shape != (n, s):
        raise ValueError("sketches must be a C-contiguous uint32 array of shape (n, s)")
    count = np.zeros(n, dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    dev, nd = _device_list(devices) if devices is not None else (None, 0)
    if devices is not None:
        rc = _lib.lib().pg_mash_sketch_batch_multi(bases.ctypes.data, offsets.ctypes.data, n, k, s, _lib.PG_SKETCH_TAIL_KEEP,
                                                   sketches.ctypes.data, max(s, 1), count.ctypes.data, status.ctypes.data, _lib.ptr(dev), nd)
    else:
        rc = _lib.lib().pg_mash_sketch_batch(bases.ctypes.data, offsets.ctypes.data, n, k, s, _lib.PG_SKETCH_TAIL_KEEP,
                                             sketches.ctypes.data, max(s, 1), count.ctypes.data, status.ctypes.data)
    _lib.check(rc, allow=(_lib.PG_ERR_PANIC,))
    return count, status


def sketch_uniform(bases: np.ndarray, n_reads: int, read_len: int, k: int, s: int) -> np.ndarray:
    """Fixed-length reads stored back to back -> compact sketches [n, min(max(L-k,0), s)]."""
    bases = np.ascontiguousarray(bases, dtype=np.uint8)
    cnt = min(max(read_len - k, 0), s)
    out = np.zeros((n_reads, max(cnt, 1)), dtype=np.uint32)
    rc = _lib.lib().pg_mash_sketch_uniform(bases.ctypes.data, n_reads, read_len, k, s, 0, out.ctypes.data, max(cnt, 1), None)
    if rc == _lib.PG_ERR_PANIC:
        raise GoPanic("index out of range [-1]")
    _lib.check(rc)
    return out[:, :cnt]


def SketchBatch(sequences: Sequence[BytesLike], kmer_size: int, sketch_size: int) -> List[Mash]:
    """[]string -> []*Mash, each equal to New(k, s) followed by Sketch(seq)."""
    bases, offsets = flatten(sequences)
    out, count, status = sketch_arrays(bases, offsets, kmer_size, sketch_size)
    res = []
    for i in range(len(sequences)):
        if status[i] == _lib.PG_ITEM_PANIC:
            raise GoPanic(f"index out of range [-1] (sequence {i})")
        m = Mash(kmer_size, sketch_size)
        m.Sketches[: count[i]] = out[i, : count[i]]
        res.append(m)
    return res


def _group_args(k: int, s: int, min_copies: int) -> None:
    if not 0 <= k < (1 << 31):
        raise PolyError(_lib.PG_ERR_ARG, f"k-mer size {k}: need 0 <= k < 2^31")
    if not 1 <= s < (1 << 31):
        raise PolyError(_lib.PG_ERR_ARG, f"sketch size {s}: need 1 <= s < 2^31")
    if not 1 <= min_copies < (1 << 32):
        raise PolyError(_lib.PG_ERR_ARG, f"min_copies {min_copies}: need 1 <= min_copies < 2^32")


def sketch_groups(bases, offsets, group_offsets, k: int, s: int, min_copies: int = 1, canonical: bool = False):
    """One sketch per group of records (Mash's `mash sketch` of a multi-FASTA file, or `-r -m min_copies` of a read
    set): group g is records [group_offsets[g], group_offsets[g+1]) of the ragged batch (bases, offsets).  Row g holds
    the smallest min(q_g, s) distinct window hashes of the group that occur at least min_copies times, ascending, then
    zeros; count[g] is how many.  Windows never cross a record.  With canonical=False the windows are positions
    0 .. L - k - 1 of each record, forward strand only; canonical=True (PG_KMER_CANONICAL) takes Mash's k-mer set,
    positions 0 .. L - k, each hashing the smaller of itself and its reverse complement, so contigs of either
    orientation and reads of either strand count as one (k >= 1).  Returns (rows [G, s] uint32, count [G] uint32): NumPy
    arrays for host inputs; for CUDA tensor inputs (uint8 bases, int64 offsets holding uint64 bits) int32 CUDA tensors
    holding the uint32 bits, computed on the current stream (the call waits for it)."""
    k, s, min_copies = int(k), int(s), int(min_copies)
    _group_args(k, s, min_copies)
    if hasattr(bases, "data_ptr"):
        import torch

        G = max(int(group_offsets.numel()) - 1, 0)
        n = max(int(offsets.numel()) - 1, 0)
        for name, t in (("offsets", offsets), ("group_offsets", group_offsets)):
            if t.element_size() != 8 or not t.is_contiguous():
                raise ValueError(f"{name} must be a contiguous 64-bit tensor")
        rows = torch.empty((G, s), dtype=torch.int32, device=bases.device)
        count = torch.empty(G, dtype=torch.int32, device=bases.device)
        st = torch.cuda.current_stream(bases.device).cuda_stream
        _lib.check(_lib.lib().pg_mash_sketch_groups_flags_dev(bases.data_ptr() if bases.numel() else None, offsets.data_ptr() if n or G else None,
                                                              n, group_offsets.data_ptr() if G else None, G, k, s, min_copies, _kmer_flags(canonical),
                                                              rows.data_ptr(), s, count.data_ptr(), st))
        return rows, count
    bases = np.ascontiguousarray(bases, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    group_offsets = np.ascontiguousarray(group_offsets, dtype=np.uint64)
    if offsets.ndim != 1 or group_offsets.ndim != 1 or len(offsets) < 1 or len(group_offsets) < 1:
        raise ValueError("offsets and group_offsets must be 1-d with at least one entry")
    n, G = len(offsets) - 1, len(group_offsets) - 1
    rows = np.zeros((G, s), np.uint32)
    count = np.zeros(G, np.uint32)
    if len(bases) == 0:
        bases = np.zeros(1, np.uint8)
    _lib.check(_lib.lib().pg_mash_sketch_groups_flags(bases.ctypes.data, offsets.ctypes.data, n, group_offsets.ctypes.data, G, k, s, min_copies,
                                                      _kmer_flags(canonical), rows.ctypes.data, s, count.ctypes.data))
    return rows, count


def _kmer_flags(canonical: bool) -> int:
    return _lib.PG_KMER_CANONICAL if canonical else 0


def SketchGroups(groups: Sequence[Sequence[BytesLike]], kmer_size: int, sketch_size: int, min_copies: int = 1,
                 canonical: bool = False) -> List[Mash]:
    """[][]string -> []*Mash: one Mash per group of sequences (an assembly's contigs, a sample's reads), holding the
    smallest sketch_size distinct window hashes of the group seen at least min_copies times, ascending, and a zero
    tail when fewer qualify.  canonical=True hashes canonical k-mers (see sketch_groups).  The result compares with
    Similarity / Distance and feeds every sketch-set call."""
    if isinstance(groups, (str, bytes)) or any(isinstance(g, (str, bytes, bytearray, np.ndarray)) for g in groups):
        raise ValueError("groups must be a list of lists of sequences")
    seqs = [q for g in groups for q in g]
    bases, offsets = flatten(seqs)
    goff = np.zeros(len(groups) + 1, np.uint64)
    if groups:
        goff[1:] = np.cumsum([len(g) for g in groups], dtype=np.uint64)
    rows, count = sketch_groups(bases, offsets, goff, kmer_size, sketch_size, min_copies, canonical)
    res = []
    for g in range(len(groups)):
        m = Mash(kmer_size, sketch_size)
        m.Sketches[:] = rows[g]
        res.append(m)
    return res


class Sketcher:
    """Grouped sketches grown in place (pg_mash_sketcher): n_groups sketches fed batch by batch, for read sets larger
    than the device or a host can stage.  Each add counts the windows of its records into their groups; rows() reads
    them at any time.  Per group the sketcher keeps a cap C (2^32 at first, never growing) and every value below it
    with its count saturated at min_copies: after an add the cap is the smallest of the old cap, the s-th value seen
    min_copies times plus one, and the (max_values + 1)-th distinct value.  A row is complete when it holds s values
    or its cap is still 2^32; a complete row equals sketch_groups over every record added to the group, whatever the
    split, and every row is a prefix of that row.  With min_copies = 1 every row is complete.  max_values defaults to
    64 s; an incomplete row asks for a larger one.  canonical=True counts canonical k-mers in every add, as
    sketch_groups(..., canonical=True) does, and complete rows equal that call's.  The sketcher lives on the device
    current at creation."""

    def __init__(self, n_groups: int, k: int, s: int, min_copies: int = 1, max_values: Optional[int] = None, canonical: bool = False):
        n_groups, k, s, min_copies = int(n_groups), int(k), int(s), int(min_copies)
        _group_args(k, s, min_copies)
        max_values = 64 * s if max_values is None else int(max_values)
        if not 0 <= n_groups < (1 << 64) or not 0 <= max_values < (1 << 64):
            raise PolyError(_lib.PG_ERR_ARG, f"n_groups {n_groups} and max_values {max_values} must fit uint64")
        h = C.c_void_p()
        _lib.check(_lib.lib().pg_mash_sketcher_create_flags(n_groups, k, s, min_copies, max_values, _kmer_flags(canonical), C.byref(h)))
        self._h = h
        self._dev_used = None
        self.n_groups, self.k, self.s, self.min_copies, self.max_values = n_groups, k, s, min_copies, max_values
        self.canonical = bool(canonical)

    def _live(self):
        if self._h is None:
            raise ValueError("the sketcher is closed")
        return self._h

    def _sync_dev(self):
        """Host calls run on the library's own stream: wait for device work enqueued on torch's streams."""
        if self._dev_used is not None:
            import torch

            torch.cuda.synchronize(self._dev_used)

    def add(self, bases, offsets, group_offsets, first_group: int = 0) -> None:
        """Adds records [group_offsets[i], group_offsets[i+1]) of the ragged batch (bases, offsets) to group
        first_group + i.  NumPy arrays go through the host add; CUDA tensors (uint8 bases, int64 offsets holding uint64
        bits) through add_dev on the current stream, which the call waits for."""
        h = self._live()
        first_group = int(first_group)
        if not 0 <= first_group < (1 << 64):
            raise PolyError(_lib.PG_ERR_ARG, f"first group {first_group} does not fit uint64")
        if hasattr(bases, "data_ptr"):
            import torch

            for name, t in (("offsets", offsets), ("group_offsets", group_offsets)):
                if t.element_size() != 8 or not t.is_contiguous():
                    raise ValueError(f"{name} must be a contiguous 64-bit tensor")
            n, nb = max(int(offsets.numel()) - 1, 0), max(int(group_offsets.numel()) - 1, 0)
            st = torch.cuda.current_stream(bases.device).cuda_stream
            _lib.check(_lib.lib().pg_mash_sketcher_add_dev(h, bases.data_ptr() if bases.numel() else None, offsets.data_ptr() if n else None, n,
                                                           group_offsets.data_ptr() if nb else None, first_group, nb, st))
            self._dev_used = bases.device
            return
        bases = np.ascontiguousarray(bases, dtype=np.uint8)
        offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
        group_offsets = np.ascontiguousarray(group_offsets, dtype=np.uint64)
        if offsets.ndim != 1 or group_offsets.ndim != 1 or len(offsets) < 1 or len(group_offsets) < 1:
            raise ValueError("offsets and group_offsets must be 1-d with at least one entry")
        if len(bases) == 0:
            bases = np.zeros(1, np.uint8)
        self._sync_dev()
        _lib.check(_lib.lib().pg_mash_sketcher_add(h, bases.ctypes.data, offsets.ctypes.data, len(offsets) - 1, group_offsets.ctypes.data,
                                                   first_group, len(group_offsets) - 1))

    def add_records(self, group: int, seqs: Sequence[BytesLike]) -> None:
        """Adds the sequences seqs (str / bytes / uint8 arrays) to one group."""
        bases, offsets = flatten(seqs)
        self.add(bases, offsets, np.array([0, len(offsets) - 1], np.uint64), group)

    def rows(self, first: int = 0, count: Optional[int] = None):
        """(rows [count, s] uint32, count [count] uint32, complete [count] bool, held [count] uint64) of groups
        [first, first + count) (count defaults to every group from first).  Changes nothing."""
        h = self._live()
        first = int(first)
        count = self.n_groups - first if count is None else int(count)
        if not (0 <= first < (1 << 64) and 0 <= count < (1 << 64)):
            raise PolyError(_lib.PG_ERR_ARG, f"rows [{first}, {first + count}) of a sketcher of {self.n_groups} groups")
        self._sync_dev()
        n = max(count, 0) if first + count <= self.n_groups else 0
        rows = np.zeros((n, self.s), np.uint32)
        cnt = np.zeros(n, np.uint32)
        complete = np.zeros(n, np.uint8)
        held = np.zeros(n, np.uint64)
        _lib.check(_lib.lib().pg_mash_sketcher_rows(h, first, count, rows.ctypes.data, self.s, cnt.ctypes.data, complete.ctypes.data, held.ctypes.data))
        return rows, cnt, complete.astype(bool), held

    def sketches(self) -> List[Mash]:
        """One Mash per group, as SketchGroups returns them."""
        rows = self.rows()[0]
        res = []
        for g in range(self.n_groups):
            m = Mash(self.k, self.s)
            m.Sketches[:] = rows[g]
            res.append(m)
        return res

    def close(self) -> None:
        if self._h is not None:
            self._sync_dev()
            h, self._h = self._h, None
            _lib.check(_lib.lib().pg_mash_sketcher_free(h))

    def __enter__(self) -> "Sketcher":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):
        if getattr(self, "_h", None) is not None:
            try:
                self.close()
            except Exception:
                pass


def _dist_inputs(q_rows, q_count, r_rows, r_count, k: int, q_length, r_length):
    """Shared checks of dist / dist_within: one s (the rows' width) for both sides, k and lengths given together."""
    k = int(k)
    if not 1 <= k < (1 << 31):
        raise PolyError(_lib.PG_ERR_ARG, f"k-mer size {k}: need 1 <= k < 2^31")
    if len(q_rows.shape) != 2 or len(r_rows.shape) != 2 or q_rows.shape[1] != r_rows.shape[1]:
        raise ValueError("q_rows and r_rows must be 2-d with one common width s")
    if tuple(q_count.shape) != (q_rows.shape[0],) or tuple(r_count.shape) != (r_rows.shape[0],):
        raise ValueError("count arrays must hold one entry per row")
    if (q_length is None) != (r_length is None):
        raise ValueError("pass both q_length and r_length, or neither")
    if q_length is not None and (tuple(q_length.shape) != (q_rows.shape[0],) or tuple(r_length.shape) != (r_rows.shape[0],)):
        raise ValueError("length arrays must hold one entry per row")
    s = int(q_rows.shape[1])
    if not 1 <= s < (1 << 31):
        raise PolyError(_lib.PG_ERR_ARG, f"sketch size {s}: need 1 <= s < 2^31")
    return k, s


def _torch_dist_inputs(q_rows, q_count, r_rows, r_count, q_length, r_length):
    for name, t, size in (("q_rows", q_rows, 4), ("q_count", q_count, 4), ("r_rows", r_rows, 4), ("r_count", r_count, 4),
                          ("q_length", q_length, 8), ("r_length", r_length, 8)):
        if t is not None and (not t.is_cuda or t.element_size() != size or not t.is_contiguous()):
            raise ValueError(f"{name} must be a contiguous CUDA tensor of {size}-byte elements")


def dist(q_rows, q_count, r_rows, r_count, k: int, q_length=None, r_length=None):
    """Mash distance of every query row against every reference row (`mash dist`): rows and counts as sketch_groups or
    Sketcher.rows return them, one sketch size s (the rows' width) for both sides.  For a pair, denom = min(s, |A u B|)
    and common = the shared values among the denom smallest values of A u B (Mash's compareSketches); distance =
    -ln(2J / (1 + J)) / k with J = common / denom (0 when common == denom, 1 when common == 0, at most 1); p_value =
    Mash's p-value, P[Binomial(denom, r) >= common] with r from k and the two genome lengths (bases per sketch, >= 1).
    Returns (common, denom, distance, p_value), each [nq, nr] with the query as the row; p_value is None without
    lengths.  NumPy inputs (uint32 rows and counts, uint64 lengths) give NumPy outputs; CUDA tensors (int32 holding the
    uint32 bits, int64 lengths) give CUDA tensors (common and denom int32 holding uint32 bits), computed by the _dev
    form on the current stream without waiting for it."""
    k, s = _dist_inputs(q_rows, q_count, r_rows, r_count, k, q_length, r_length)
    nq, nr = int(q_rows.shape[0]), int(r_rows.shape[0])
    want_p = q_length is not None
    if hasattr(q_rows, "data_ptr"):
        import torch

        _torch_dist_inputs(q_rows, q_count, r_rows, r_count, q_length, r_length)
        dev = q_rows.device
        common = torch.empty((nq, nr), dtype=torch.int32, device=dev)
        denom = torch.empty((nq, nr), dtype=torch.int32, device=dev)
        distance = torch.empty((nq, nr), dtype=torch.float64, device=dev)
        p = torch.empty((nq, nr), dtype=torch.float64, device=dev) if want_p else None
        st = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(_lib.lib().pg_mash_dist_dev(_lib.ptr(q_rows), _lib.ptr(q_count), nq, _lib.ptr(r_rows), _lib.ptr(r_count), nr, s, s, k,
                                               _lib.ptr(q_length), _lib.ptr(r_length), _lib.ptr(common), _lib.ptr(denom), _lib.ptr(distance),
                                               _lib.ptr(p), st))
        return common, denom, distance, p
    q_rows, r_rows = np.ascontiguousarray(q_rows, np.uint32), np.ascontiguousarray(r_rows, np.uint32)
    q_count, r_count = np.ascontiguousarray(q_count, np.uint32), np.ascontiguousarray(r_count, np.uint32)
    if want_p:
        q_length, r_length = np.ascontiguousarray(q_length, np.uint64), np.ascontiguousarray(r_length, np.uint64)
    common, denom = np.zeros((nq, nr), np.uint32), np.zeros((nq, nr), np.uint32)
    distance = np.zeros((nq, nr), np.float64)
    p = np.zeros((nq, nr), np.float64) if want_p else None
    _lib.check(_lib.lib().pg_mash_dist(_lib.ptr(q_rows), _lib.ptr(q_count), nq, _lib.ptr(r_rows), _lib.ptr(r_count), nr, s, s, k, _lib.ptr(q_length),
                                       _lib.ptr(r_length), _lib.ptr(common), _lib.ptr(denom), _lib.ptr(distance), _lib.ptr(p)))
    return common, denom, distance, p


def dist_within(q_rows, q_count, r_rows, r_count, k: int, q_length=None, r_length=None, max_distance: float = 1.0, max_p_value: float = 1.0,
                upper: bool = False):
    """The pairs of dist with distance <= max_distance and p-value <= max_p_value (`mash dist -d D -v P`); upper=True
    keeps only r > q, for a set against itself (`mash triangle`; needs nq == nr).  max_p_value < 1 needs the lengths.
    Returns (pair_q, pair_r, common, denom, distance, p_value) sorted by (q, r); p_value is None without lengths.  NumPy
    inputs give NumPy outputs; CUDA tensors go through the _dev form on the current stream, and the call waits for it to
    read the pair count."""
    k, s = _dist_inputs(q_rows, q_count, r_rows, r_count, k, q_length, r_length)
    nq, nr = int(q_rows.shape[0]), int(r_rows.shape[0])
    want_p = q_length is not None
    flags = _lib.PG_PAIRS_UPPER if upper else 0
    max_distance, max_p_value = float(max_distance), float(max_p_value)
    cap = max(1024, 4 * nq)
    if hasattr(q_rows, "data_ptr"):
        import torch

        _torch_dist_inputs(q_rows, q_count, r_rows, r_count, q_length, r_length)
        dev = q_rows.device
        st = torch.cuda.current_stream(dev).cuda_stream
        d_n = torch.zeros(1, dtype=torch.int64, device=dev)
        while True:
            out = [torch.empty(cap, dtype=dt, device=dev) for dt in (torch.int32, torch.int32, torch.int32, torch.int32, torch.float64)]
            p = torch.empty(cap, dtype=torch.float64, device=dev) if want_p else None
            _lib.check(_lib.lib().pg_mash_dist_within_dev(_lib.ptr(q_rows), _lib.ptr(q_count), nq, _lib.ptr(r_rows), _lib.ptr(r_count), nr, s, s, k,
                                                          _lib.ptr(q_length), _lib.ptr(r_length), max_distance, max_p_value, flags,
                                                          *[_lib.ptr(t) for t in out], _lib.ptr(p), cap, _lib.ptr(d_n), st))
            n = int(d_n.item())
            if n <= cap:
                break
            cap = n
        pq, pr, c, d, dist_ = (t[:n] for t in out)
        order = torch.argsort(pq.to(torch.int64) * max(nr, 1) + pr.to(torch.int64))
        return pq[order], pr[order], c[order], d[order], dist_[order], (p[:n][order] if want_p else None)
    q_rows, r_rows = np.ascontiguousarray(q_rows, np.uint32), np.ascontiguousarray(r_rows, np.uint32)
    q_count, r_count = np.ascontiguousarray(q_count, np.uint32), np.ascontiguousarray(r_count, np.uint32)
    if want_p:
        q_length, r_length = np.ascontiguousarray(q_length, np.uint64), np.ascontiguousarray(r_length, np.uint64)
    while True:
        pq, pr, c, d = (np.zeros(cap, np.uint32) for _ in range(4))
        dist_ = np.zeros(cap, np.float64)
        p = np.zeros(cap, np.float64) if want_p else None
        cnt = C.c_uint64(0)
        rc = _lib.lib().pg_mash_dist_within(_lib.ptr(q_rows), _lib.ptr(q_count), nq, _lib.ptr(r_rows), _lib.ptr(r_count), nr, s, s, k,
                                            _lib.ptr(q_length), _lib.ptr(r_length), max_distance, max_p_value, flags, pq.ctypes.data, pr.ctypes.data,
                                            c.ctypes.data, d.ctypes.data, dist_.ctypes.data, _lib.ptr(p), cap, C.byref(cnt))
        if rc == _lib.PG_ERR_ARG and cnt.value > cap:
            cap = int(cnt.value)
            continue
        _lib.check(rc)
        n = int(cnt.value)
        order = np.lexsort((pr[:n], pq[:n]))
        return pq[:n][order], pr[:n][order], c[:n][order], d[:n][order], dist_[:n][order], (p[:n][order] if want_p else None)


def similarity_pairs(mashes: Sequence[Mash], pairs: np.ndarray):
    """Explicit pair list (receiver, argument) over sketches of mixed sizes -> (same, similarity, distance)."""
    arrs = [np.ascontiguousarray(m.Sketches[: m.SketchSize], dtype=np.uint32) for m in mashes]
    off = np.zeros(len(arrs) + 1, dtype=np.uint64)
    off[1:] = np.cumsum([len(a) for a in arrs], dtype=np.uint64)
    sk = np.concatenate(arrs) if arrs else np.zeros(0, np.uint32)
    pairs = np.ascontiguousarray(pairs, dtype=np.uint32).reshape(-1, 2)
    pa, pb = np.ascontiguousarray(pairs[:, 0]), np.ascontiguousarray(pairs[:, 1])
    n = len(pa)
    same, sim, dist, st = np.zeros(n, np.int64), np.zeros(n, np.float64), np.zeros(n, np.float64), np.zeros(n, np.int32)
    rc = _lib.lib().pg_mash_similarity_pairs(sk.ctypes.data, off.ctypes.data, len(arrs), pa.ctypes.data, pb.ctypes.data, n,
                                             same.ctypes.data, sim.ctypes.data, dist.ctypes.data, st.ctypes.data)
    if rc == _lib.PG_ERR_PANIC:
        raise GoPanic("index out of range [-1]")
    _lib.check(rc)
    return same, sim, dist


def distance_block(sketches: np.ndarray, row_begin: int = 0, row_end: Optional[int] = None, want_distance: bool = True):
    """Rows [row_begin,row_end) x all columns over equal-size sketches [n, s] (full Go arrays).
    Returns (same uint32 [rows, n], distance float64 [rows, n] or None); receiver = row."""
    sketches = np.ascontiguousarray(sketches, dtype=np.uint32)
    n, s = sketches.shape
    row_end = n if row_end is None else row_end
    rows = row_end - row_begin
    same = np.zeros((rows, n), dtype=np.uint32)
    dist = np.zeros((rows, n), dtype=np.float64) if want_distance else None
    rc = _lib.lib().pg_mash_distance_block(sketches.ctypes.data, n, s, row_begin, row_end, same.ctypes.data,
                                           dist.ctypes.data if dist is not None else None)
    if rc == _lib.PG_ERR_PANIC:
        raise GoPanic("index out of range [-1]")
    _lib.check(rc)
    return same, dist


def distance_sparse(sketches: np.ndarray, row_begin: int = 0, row_end: Optional[int] = None, upper: bool = True):
    """The pairs of a row block that share at least one hash, as (i, j, same) arrays sorted by (i, j);
    every pair that is not listed has same == 0 (Distance 1).  upper: only j > i."""
    sketches = np.ascontiguousarray(sketches, dtype=np.uint32)
    n, s = sketches.shape
    row_end = n if row_end is None else row_end
    cap = max(1024, 4 * (row_end - row_begin))
    while True:
        pi, pj, ps = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
        cnt = C.c_uint64(0)
        rc = _lib.lib().pg_mash_distance_sparse(sketches.ctypes.data, n, s, row_begin, row_end, 1 if upper else 0, pi.ctypes.data, pj.ctypes.data,
                                                ps.ctypes.data, cap, C.byref(cnt))
        if rc == _lib.PG_ERR_ARG and cnt.value > cap:
            cap = int(cnt.value)
            continue
        if rc == _lib.PG_ERR_PANIC:
            raise GoPanic("index out of range [-1]")
        _lib.check(rc)
        k = int(cnt.value)
        order = np.lexsort((pj[:k], pi[:k]))
        return pi[:k][order], pj[:k][order], ps[:k][order]


def DistanceMatrix(mashes: Sequence[Mash]) -> np.ndarray:
    """All-pairs Distance for sketches of one common SketchSize: D[i, j] = mashes[i].Distance(mashes[j])."""
    if not mashes:
        return np.zeros((0, 0))
    s = mashes[0].SketchSize
    if any(m.SketchSize != s for m in mashes):
        raise ValueError("DistanceMatrix needs one common SketchSize; use similarity_pairs for mixed sizes")
    sk = np.stack([np.ascontiguousarray(m.Sketches[:s], dtype=np.uint32) for m in mashes])
    return distance_block(sk)[1]


# ---- sketch index: top-k nearest references (pg_mash_index_*) --------------------------------------------
INDEX_MAX_TOP_K = 1024  # PG_INDEX_MAX_TOP_K
NO_REF = 0xFFFFFFFF


def min_same_for_distance(max_distance: float, den: int) -> int:
    """Smallest matching count whose Distance is <= max_distance, evaluating the reference's own f64
    expression 1 - same/den (mash.go:134,139) for every same in [0, den]; den + 1 when none qualifies.
    The expression is non-increasing in same, so filtering by the returned count is exact."""
    same = np.arange(den + 1, dtype=np.float64)
    ok = np.nonzero(1.0 - same / np.float64(max(den, 1)) <= max_distance)[0]
    return int(ok[0]) if len(ok) else den + 1


def _sketch_rows(sketches):
    """[n, s] uint32 array (host) or CUDA tensor (device), or a list of Mash of one SketchSize."""
    if hasattr(sketches, "data_ptr"):
        if sketches.dim() != 2 or sketches.element_size() != 4 or not sketches.is_contiguous():
            raise ValueError("sketch tensors must be contiguous 32-bit [n, s]")
        return sketches
    if isinstance(sketches, (list, tuple)):
        if not sketches:
            return np.zeros((0, 0), dtype=np.uint32)
        s = sketches[0].SketchSize
        if any(m.SketchSize != s for m in sketches):
            raise ValueError("every sketch of a set must have the same SketchSize")
        return np.stack([np.ascontiguousarray(m.Sketches[:s], dtype=np.uint32) for m in sketches]).reshape(len(sketches), s)
    arr = np.ascontiguousarray(sketches, dtype=np.uint32)
    if arr.ndim != 2:
        raise ValueError("sketches must be [n, s]")
    return arr


def _index_rc(rc: int) -> None:
    if rc == _lib.PG_ERR_PANIC:
        raise GoPanic("index out of range [-1]")  # Sketches[SketchSize-1] with SketchSize 0
    _lib.check(rc)


class SketchIndex:
    """A reference sketch set held on the GPU for top-k queries: `nearest` ranks every reference j for
    query q by queries[q].Similarity(refs[j]) (the query is the receiver, mash.go:107-135).

    sketches: [n, s] uint32 (full Go arrays, zero tail included), a CUDA tensor of that shape, or a list of
    Mash of one SketchSize.  The index copies them; it lives on the device current at creation."""

    def __init__(self, sketches):
        rows = _sketch_rows(sketches)
        n, s = int(rows.shape[0]), int(rows.shape[1])
        h = C.c_void_p()
        if hasattr(rows, "data_ptr"):
            import torch

            rc = _lib.lib().pg_mash_index_create_dev(rows.data_ptr(), n, s, torch.cuda.current_stream(rows.device).cuda_stream, C.byref(h))
        else:
            rc = _lib.lib().pg_mash_index_create(rows.ctypes.data, n, s, C.byref(h))
        _index_rc(rc)
        self._h = h
        self._dev_queried = None
        self.n, self.s = n, s

    @classmethod
    def load(cls, path: str) -> "SketchIndex":
        """An index over the sketch set of a PGSKETCH file (rows re-materialised with their zero tails)."""
        from . import sketchfile

        sk, _, _, s = sketchfile.load(path, pad_zero=True)
        return cls(sk[:, :s])

    def add(self, sketches) -> int:
        """Appends reference sketches (what the constructor takes) on the device: the batch's rows become
        references n, n + 1, ..., and every later query answers as an index built over the concatenated set would.
        An empty index takes the batch's sketch size.  Returns the id of the first added reference."""
        if self._h is None:
            raise ValueError("the index is closed")
        rows = _sketch_rows(sketches)
        m, s = int(rows.shape[0]), int(rows.shape[1])
        first = self.n
        if self._dev_queried is not None:  # the add releases buffers that device queries, on any stream, may still read
            import torch

            torch.cuda.synchronize(self._dev_queried)
        if hasattr(rows, "data_ptr"):
            import torch

            rc = _lib.lib().pg_mash_index_add_dev(self._h, rows.data_ptr(), m, s, torch.cuda.current_stream(rows.device).cuda_stream)
        else:
            rc = _lib.lib().pg_mash_index_add(self._h, rows.ctypes.data, m, s)
        _index_rc(rc)
        if m:
            self.n += m
            if first == 0:
                self.s = s
        return first

    def nearest(self, queries, k: int, min_same: Optional[int] = None, max_distance: Optional[float] = None):
        """For each query sketch, the k references with the largest matching counts (same descending, then
        reference index ascending), keeping only same >= min_same (default 1) -- or, alternatively, only
        Distance <= max_distance.  Returns (ref [nq, k] uint32, same [nq, k] uint32, distance [nq, k] float64,
        n_hits [nq] uint32); slots past n_hits[q] hold ref 0xFFFFFFFF, same 0, distance 1.0.  CUDA tensor
        queries give CUDA tensor results (int32 tensors carry the uint32 bits), ordered on the current stream."""
        if self._h is None:
            raise ValueError("the index is closed")
        if min_same is not None and max_distance is not None:
            raise ValueError("give min_same or max_distance, not both")
        rows = _sketch_rows(queries)
        nq, sq = int(rows.shape[0]), int(rows.shape[1])
        if max_distance is not None:
            min_same = min_same_for_distance(max_distance, min(sq, self.s))
        min_same = 1 if min_same is None else int(min_same)
        if not 0 <= min_same <= 0xFFFFFFFF:
            raise ValueError("min_same must fit 32 bits")
        if k < 0 or k > 0xFFFFFFFF:
            raise PolyError(_lib.PG_ERR_ARG, f"top_k {k} outside [1, {INDEX_MAX_TOP_K}]")
        if hasattr(rows, "data_ptr"):
            import torch

            dev = rows.device
            ref = torch.empty((nq, max(k, 1)), dtype=torch.int32, device=dev)
            same = torch.empty((nq, max(k, 1)), dtype=torch.int32, device=dev)
            dist = torch.empty((nq, max(k, 1)), dtype=torch.float64, device=dev)
            nh = torch.empty(nq, dtype=torch.int32, device=dev)
            rc = _lib.lib().pg_mash_index_query_dev(self._h, rows.data_ptr(), nq, sq, k, min_same, ref.data_ptr(), same.data_ptr(),
                                                    dist.data_ptr(), nh.data_ptr(), torch.cuda.current_stream(dev).cuda_stream)
            self._dev_queried = dev
        else:
            ref = np.empty((nq, max(k, 1)), dtype=np.uint32)
            same = np.empty((nq, max(k, 1)), dtype=np.uint32)
            dist = np.empty((nq, max(k, 1)), dtype=np.float64)
            nh = np.empty(nq, dtype=np.uint32)
            rc = _lib.lib().pg_mash_index_query(self._h, rows.ctypes.data, nq, sq, k, min_same, ref.ctypes.data, same.ctypes.data,
                                                dist.ctypes.data, nh.ctypes.data)
        _index_rc(rc)
        return ref[:, :k], same[:, :k], dist[:, :k], nh

    def within(self, queries, min_same: Optional[int] = None, max_distance: Optional[float] = None):
        """For each query sketch, every reference with at least min_same matching hashes (default 1) -- or,
        alternatively, with Distance <= max_distance -- however many there are, in reference order.  Returns CSR
        lists (offsets [nq + 1] uint64, ref [m] uint32, same [m] uint32, distance [m] float64): query q's hits are
        entries [offsets[q], offsets[q + 1]).  A max_distance that every pair meets (>= 1) is a ValueError.

        CUDA tensor queries give CUDA tensors (int64 offsets, int32 tensors carrying the uint32 bits).  The total
        sizes the outputs, so this call waits for the device to count it, as torch.nonzero does."""
        if self._h is None:
            raise ValueError("the index is closed")
        if min_same is not None and max_distance is not None:
            raise ValueError("give min_same or max_distance, not both")
        rows = _sketch_rows(queries)
        nq, sq = int(rows.shape[0]), int(rows.shape[1])
        if max_distance is not None:
            min_same = min_same_for_distance(max_distance, min(sq, self.s))
            if min_same == 0:
                raise ValueError(f"max_distance {max_distance!r} lists every pair: every Distance is <= it")
        min_same = 1 if min_same is None else int(min_same)
        if not 0 <= min_same <= 0xFFFFFFFF:
            raise ValueError("min_same must fit 32 bits")
        cap = min(nq * self.n, max(1024, 64 * nq))  # first guess; one retry with the exact total when it is short
        on_device = hasattr(rows, "data_ptr")
        if on_device:
            import torch

            dev = rows.device
            st = torch.cuda.current_stream(dev).cuda_stream
            off = torch.empty(nq + 1, dtype=torch.int64, device=dev)
            total = torch.zeros((), dtype=torch.int64, device=dev)
            while True:
                ref = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
                same = torch.empty(max(cap, 1), dtype=torch.int32, device=dev)
                dist = torch.empty(max(cap, 1), dtype=torch.float64, device=dev)
                _index_rc(_lib.lib().pg_mash_index_query_within_dev(self._h, rows.data_ptr(), nq, sq, min_same, off.data_ptr(), ref.data_ptr(),
                                                                    same.data_ptr(), dist.data_ptr(), cap, total.data_ptr(), st))
                self._dev_queried = dev
                m = int(total.item())
                if m <= cap:
                    return off, ref[:m], same[:m], dist[:m]
                cap = m
        off = np.empty(nq + 1, dtype=np.uint64)
        cnt = C.c_uint64(0)
        while True:
            ref = np.empty(max(cap, 1), dtype=np.uint32)
            same = np.empty(max(cap, 1), dtype=np.uint32)
            dist = np.empty(max(cap, 1), dtype=np.float64)
            rc = _lib.lib().pg_mash_index_query_within(self._h, rows.ctypes.data, nq, sq, min_same, off.ctypes.data, ref.ctypes.data,
                                                       same.ctypes.data, dist.ctypes.data, cap, C.byref(cnt))
            if rc == _lib.PG_ERR_ARG and cnt.value > cap:
                cap = int(cnt.value)
                continue
            _index_rc(rc)
            m = int(cnt.value)
            return off, ref[:m], same[:m], dist[:m]

    def close(self) -> None:
        if self._h is not None:
            if self._dev_queried is not None:  # results of device queries may still be in flight on torch's streams
                import torch

                torch.cuda.synchronize(self._dev_queried)
            h, self._h = self._h, None
            _lib.check(_lib.lib().pg_mash_index_free(h))

    def __enter__(self) -> "SketchIndex":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):
        if getattr(self, "_h", None) is not None:
            try:
                self.close()
            except Exception:
                pass


def _link_rows(sketches, min_same: Optional[int], max_distance: Optional[float]):
    """(rows, n, s, min_same) of a cluster or dereplicate call; min_same is None when no matching count reaches
    max_distance, so that nothing links and the caller returns its trivial result without a launch."""
    if (min_same is None) == (max_distance is None):
        raise ValueError("give exactly one of min_same and max_distance")
    rows = _sketch_rows(sketches)
    n, s = int(rows.shape[0]), int(rows.shape[1])
    if max_distance is not None and s > 0:  # s == 0: the library reports the reference's panic
        min_same = min_same_for_distance(max_distance, s)
        if min_same == 0:
            raise ValueError(f"max_distance {max_distance!r} links every pair: every Distance is <= it")
        if min_same == s + 1:
            return rows, n, s, None
    min_same = 1 if min_same is None else int(min_same)
    if not 0 <= min_same <= 0xFFFFFFFF:
        raise ValueError("min_same must fit 32 bits")
    return rows, n, s, min_same


# ---- cluster: single-linkage groups of a sketch set (pg_mash_cluster) -------------------------------------
def cluster(sketches, min_same: Optional[int] = None, max_distance: Optional[float] = None):
    """Groups of a sketch set: sketches i < j are linked when sketches[i].Similarity(sketches[j]) counts at
    least min_same matching hashes (the lower index is the receiver) -- or, alternatively, when their Distance
    is <= max_distance -- and the groups are the connected components (single linkage).

    sketches: what SketchIndex takes.  Returns (labels [n] uint32, n_groups, n_links): labels[i] is the smallest
    index in i's group, so labels[i] == i marks one representative per group; n_links counts the linked pairs.
    CUDA tensor sketches give a CUDA int32 label tensor (carrying the uint32 bits) and 0-dim int64 count
    tensors, ordered on the current stream.  The pairs themselves are never materialised."""
    rows, n, s, min_same = _link_rows(sketches, min_same, max_distance)
    on_device = hasattr(rows, "data_ptr")
    if on_device:
        import torch
    if min_same is None:  # every sketch is its own group
        if on_device:
            return torch.arange(n, dtype=torch.int32, device=rows.device), torch.tensor(n, device=rows.device), torch.tensor(0, device=rows.device)
        return np.arange(n, dtype=np.uint32), n, 0
    if on_device:
        dev = rows.device
        labels = torch.empty(n, dtype=torch.int32, device=dev)
        counts = torch.zeros(2, dtype=torch.int64, device=dev)
        rc = _lib.lib().pg_mash_cluster_dev(rows.data_ptr(), n, s, min_same, labels.data_ptr(), counts.data_ptr(),
                                            counts.data_ptr() + 8, torch.cuda.current_stream(dev).cuda_stream)
        _index_rc(rc)
        return labels, counts[0], counts[1]
    labels = np.empty(n, dtype=np.uint32)
    ng, nl = C.c_uint64(0), C.c_uint64(0)
    _index_rc(_lib.lib().pg_mash_cluster(rows.ctypes.data, n, s, min_same, labels.ctypes.data, C.byref(ng), C.byref(nl)))
    return labels, int(ng.value), int(nl.value)


# ---- dereplicate: greedy representatives of a sketch set (pg_mash_dereplicate) ---------------------------
PG_DEREP_NEAREST = 1


def dereplicate(sketches, min_same: Optional[int] = None, max_distance: Optional[float] = None, nearest: bool = False):
    """Representatives of a sketch set: sketches r < i are linked as in cluster (sketches[r].Similarity(sketches[i])
    counts at least min_same matching hashes, or their Distance is <= max_distance).  In index order, i is a
    representative iff no representative r < i is linked to i.  Every other sketch is assigned the smallest linked
    representative, or with nearest=True the linked one with the largest count (smallest Distance), ties to the
    smaller index.  Permute the set first for another priority.

    sketches: what cluster takes.  Returns (rep [n] uint32, n_reps): rep[i] == i marks a representative.  CUDA
    tensor sketches give a CUDA int32 tensor (carrying the uint32 bits) and a 0-dim int64 count tensor, ordered on
    the current stream.  The pairs themselves are never materialised."""
    rows, n, s, min_same = _link_rows(sketches, min_same, max_distance)
    on_device = hasattr(rows, "data_ptr")
    if on_device:
        import torch
    if min_same is None:  # every sketch represents itself
        if on_device:
            return torch.arange(n, dtype=torch.int32, device=rows.device), torch.tensor(n, device=rows.device)
        return np.arange(n, dtype=np.uint32), n
    flags = PG_DEREP_NEAREST if nearest else 0
    if on_device:
        dev = rows.device
        rep = torch.empty(n, dtype=torch.int32, device=dev)
        count = torch.zeros((), dtype=torch.int64, device=dev)
        rc = _lib.lib().pg_mash_dereplicate_dev(rows.data_ptr(), n, s, min_same, flags, rep.data_ptr(), count.data_ptr(),
                                                torch.cuda.current_stream(dev).cuda_stream)
        _index_rc(rc)
        return rep, count
    rep = np.empty(n, dtype=np.uint32)
    nr = C.c_uint64(0)
    _index_rc(_lib.lib().pg_mash_dereplicate(rows.ctypes.data, n, s, min_same, flags, rep.ctypes.data, C.byref(nr)))
    return rep, int(nr.value)


class _RepresentativeIndex(SketchIndex):
    """An index a growing grouping (Dereplicator, Clusterer) owns, borrowed for queries: it is grown only by its
    owner's adds and released with it."""

    def __init__(self, h, s: int, owner: str = "Dereplicator"):
        self._h = h
        self._dev_queried = None
        self.n, self.s = 0, s
        self._owner = owner

    def add(self, sketches) -> int:
        raise ValueError(f"this index grows only through {self._owner}.add")

    def close(self) -> None:
        if self._h is not None and self._dev_queried is not None:
            import torch

            torch.cuda.synchronize(self._dev_queried)
        self._h = None


class Dereplicator:
    """A dereplication that grows: each add assigns a new batch of sketches against the representatives kept so
    far, on the device, without dereplicating the earlier sketches again.  Sketches are numbered in the order they
    are added.  After any sequence of adds, the concatenated assignments equal dereplicate() of the concatenated
    batches, with the same min_same / max_distance and nearest.

    s: the sketch size of every batch.  A max_distance under which every pair links, or none can, is a ValueError.
    The representatives are kept in a SketchIndex over them: nearest and within query it and give sketch ids."""

    def __init__(self, s: int, min_same: Optional[int] = None, max_distance: Optional[float] = None, nearest: bool = False):
        if (min_same is None) == (max_distance is None):
            raise ValueError("give exactly one of min_same and max_distance")
        s = int(s)
        if max_distance is not None and s > 0:  # s <= 0: the library reports the reference's panic
            min_same = min_same_for_distance(max_distance, s)
            if min_same == 0:
                raise ValueError(f"max_distance {max_distance!r} links every pair: every Distance is <= it")
            if min_same == s + 1:
                raise ValueError(f"max_distance {max_distance!r} links no pair: no Distance is <= it")
        min_same = 1 if min_same is None else int(min_same)
        if not 0 <= min_same <= 0xFFFFFFFF:
            raise ValueError("min_same must fit 32 bits")
        h = C.c_void_p()
        _index_rc(_lib.lib().pg_mash_dereplicator_create(s, min_same, PG_DEREP_NEAREST if nearest else 0, C.byref(h)))
        self._h = h
        self._ix = _RepresentativeIndex(C.c_void_p(_lib.lib().pg_mash_dereplicator_index(h)), s)
        self._lock = threading.Lock()
        self.s, self.min_same, self.nearest_mode = s, min_same, bool(nearest)
        self.n = 0

    def add(self, sketches):
        """Assigns a batch (what dereplicate takes): returns (rep [m] uint32, n_new_reps), rep holding global ids, so
        row i of the batch is sketch first + i.  CUDA tensors give a CUDA int32 tensor (carrying the uint32 bits),
        ordered on the current stream; the call itself synchronises."""
        if self._h is None:
            raise ValueError("the dereplicator is closed")
        rows = _sketch_rows(sketches)
        m, s = int(rows.shape[0]), int(rows.shape[1])
        first, n_new = C.c_uint64(0), C.c_uint64(0)
        if self._ix._dev_queried is not None:  # the add releases buffers that device queries, on any stream, may still read
            import torch

            torch.cuda.synchronize(self._ix._dev_queried)
        if hasattr(rows, "data_ptr"):
            import torch

            rep = torch.empty(m, dtype=torch.int32, device=rows.device)
            rc = _lib.lib().pg_mash_dereplicator_add_dev(self._h, rows.data_ptr(), m, s, rep.data_ptr(), C.byref(first), C.byref(n_new),
                                                         torch.cuda.current_stream(rows.device).cuda_stream)
        else:
            rep = np.empty(m, dtype=np.uint32)
            rc = _lib.lib().pg_mash_dereplicator_add(self._h, rows.ctypes.data, m, s, rep.ctypes.data, C.byref(first), C.byref(n_new))
        _index_rc(rc)
        with self._lock:
            self.n = max(self.n, int(first.value) + m)
            self._ix.n += int(n_new.value)
        return rep, int(n_new.value)

    def representatives(self) -> np.ndarray:
        """The ids of the representatives kept so far, ascending: position p of the representative index is
        sketch representatives()[p]."""
        if self._h is None:
            raise ValueError("the dereplicator is closed")
        cnt = C.c_uint64(0)
        cap = self._ix.n
        while True:
            ids = np.empty(max(cap, 1), dtype=np.uint32)
            rc = _lib.lib().pg_mash_dereplicator_reps(self._h, ids.ctypes.data, cap, C.byref(cnt))
            if rc == _lib.PG_ERR_ARG and cnt.value > cap:  # an add on another thread kept more
                cap = int(cnt.value)
                continue
            _lib.check(rc)
            return ids[: int(cnt.value)]

    def _ids_of(self, ref, ids):
        """Positions of the representative index -> sketch ids; the NO_REF slots stay as they are."""
        if len(ids) == 0:  # no representative: every slot is NO_REF
            return ref
        if hasattr(ref, "data_ptr"):
            import torch

            t = torch.from_numpy(ids.view(np.int32)).to(ref.device)
            return torch.where(ref == -1, ref, t[ref.clamp(min=0).long()])
        return np.where(ref == NO_REF, ref, ids[np.where(ref == NO_REF, 0, ref)]).astype(np.uint32)

    def nearest(self, queries, k: int, min_same: Optional[int] = None, max_distance: Optional[float] = None):
        """SketchIndex.nearest over the representatives, with every hit given as its sketch id."""
        ref, same, dist, nh = self._ix.nearest(queries, k, min_same=min_same, max_distance=max_distance)
        return self._ids_of(ref, self.representatives()), same, dist, nh

    def within(self, queries, min_same: Optional[int] = None, max_distance: Optional[float] = None):
        """SketchIndex.within over the representatives, with every hit given as its sketch id."""
        off, ref, same, dist = self._ix.within(queries, min_same=min_same, max_distance=max_distance)
        return off, self._ids_of(ref, self.representatives()), same, dist

    def close(self) -> None:
        if self._h is not None:
            self._ix.close()
            h, self._h = self._h, None
            _lib.check(_lib.lib().pg_mash_dereplicator_free(h))

    def __enter__(self) -> "Dereplicator":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):
        if getattr(self, "_h", None) is not None:
            try:
                self.close()
            except Exception:
                pass


class Clusterer:
    """A clustering that grows: each add merges a new batch of sketches into the single-linkage groups of the
    sketches added so far, on the device, without clustering the earlier sketches again.  Sketches are numbered in
    the order they are added.  After every add, labels() equals cluster() of the concatenated batches, with the same
    min_same / max_distance; earlier labels can change when a batch joins two earlier groups (n_merged > 0).

    s: the sketch size of every batch.  A max_distance under which every pair links, or none can, is a ValueError.
    Every sketch is kept in a SketchIndex (`index`, read-only, reference p is sketch p), so "which group would this
    sketch join" is a nearest or within query followed by labels()."""

    def __init__(self, s: int, min_same: Optional[int] = None, max_distance: Optional[float] = None):
        if (min_same is None) == (max_distance is None):
            raise ValueError("give exactly one of min_same and max_distance")
        s = int(s)
        if max_distance is not None and s > 0:  # s <= 0: the library reports the reference's panic
            min_same = min_same_for_distance(max_distance, s)
            if min_same == 0:
                raise ValueError(f"max_distance {max_distance!r} links every pair: every Distance is <= it")
            if min_same == s + 1:
                raise ValueError(f"max_distance {max_distance!r} links no pair: no Distance is <= it")
        min_same = 1 if min_same is None else int(min_same)
        if not 0 <= min_same <= 0xFFFFFFFF:
            raise ValueError("min_same must fit 32 bits")
        h = C.c_void_p()
        _index_rc(_lib.lib().pg_mash_clusterer_create(s, min_same, C.byref(h)))
        self._h = h
        self.index = _RepresentativeIndex(C.c_void_p(_lib.lib().pg_mash_clusterer_index(h)), s, "Clusterer")
        self._lock = threading.Lock()
        self.s, self.min_same = s, min_same
        self.n = self.n_groups = self.n_links = 0

    def add(self, sketches):
        """Merges a batch (what cluster takes): returns (labels [m], n_groups, n_links, n_merged).  labels are the
        global labels of the batch's rows (row i is sketch first + i) after this add; n_groups counts every group
        after it, n_links the links this add found and n_merged the earlier groups it absorbed into another.  CUDA
        tensors give a CUDA int32 tensor (carrying the uint32 bits), ordered on the current stream; the call itself
        synchronises."""
        if self._h is None:
            raise ValueError("the clusterer is closed")
        rows = _sketch_rows(sketches)
        m, s = int(rows.shape[0]), int(rows.shape[1])
        first, ng, nl, nm = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
        if self.index._dev_queried is not None:  # the add releases buffers that device queries, on any stream, may still read
            import torch

            torch.cuda.synchronize(self.index._dev_queried)
        if hasattr(rows, "data_ptr"):
            import torch

            labels = torch.empty(m, dtype=torch.int32, device=rows.device)
            rc = _lib.lib().pg_mash_clusterer_add_dev(self._h, rows.data_ptr(), m, s, labels.data_ptr(), C.byref(first), C.byref(ng),
                                                      C.byref(nl), C.byref(nm), torch.cuda.current_stream(rows.device).cuda_stream)
        else:
            labels = np.empty(m, dtype=np.uint32)
            rc = _lib.lib().pg_mash_clusterer_add(self._h, rows.ctypes.data, m, s, labels.ctypes.data, C.byref(first), C.byref(ng),
                                                  C.byref(nl), C.byref(nm))
        _index_rc(rc)
        with self._lock:
            if int(first.value) + m >= self.n:  # the latest add of any thread
                self.n, self.n_groups = int(first.value) + m, int(ng.value)
            self.n_links += int(nl.value)
            self.index.n = self.n
        return labels, int(ng.value), int(nl.value), int(nm.value)

    def labels(self, begin: int = 0, end: Optional[int] = None):
        """The current labels of sketches [begin, end) (end defaults to every sketch added), uint32."""
        if self._h is None:
            raise ValueError("the clusterer is closed")
        end = self.n if end is None else int(end)
        begin = int(begin)
        out = np.empty(max(end - begin, 0), dtype=np.uint32)
        _lib.check(_lib.lib().pg_mash_clusterer_labels(self._h, begin, end, out.ctypes.data if len(out) else None))
        return out

    def close(self) -> None:
        if self._h is not None:
            self.index.close()
            h, self._h = self._h, None
            _lib.check(_lib.lib().pg_mash_clusterer_free(h))

    def __enter__(self) -> "Clusterer":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):
        if getattr(self, "_h", None) is not None:
            try:
                self.close()
            except Exception:
                pass


class Screen:
    """Mash Screen (Ondov et al., Genome Biol 20:232, 2019) on the GPU: which references of a sketch set a pool of
    reads contains.  Every k-mer window a (*Mash).Sketch would hash (positions 0 .. L - k - 1 of each read, forward
    strand, raw bytes) is counted into the pool; results() then gives, for each reference r, shared[r] = the sum
    over hashes v of min(c_r(v), c_pool(v)), containment[r] = shared[r] / s, and multiplicity[r] = the lower median
    of c_pool(v) over the shared hashes, each counted min(c_r(v), c_pool(v)) times (0 when nothing is shared).

    sketches: [n, s] uint32 (full Go arrays, zero tail included), a CUDA tensor of that shape, or a list of Mash of
    one SketchSize; k: the k-mer size they were sketched with (not checked, as in the reference).  The pool grows with
    each add, in any split, and reset() empties it.  With canonical=False reverse-complement windows are not counted:
    the references hash the forward strand only.  canonical=True counts canonical k-mers (positions 0 .. L - k, each the
    smaller of itself and its reverse complement), so reads of both strands count; pass sketches made the same way,
    e.g. by sketch_groups(..., canonical=True) (the mode, like k, is not checked).  The screen copies the sketches; it
    lives on the device current at creation.

    samples: the number of pools the screen holds over the one reference index (a multiplexed run's barcodes).  Each
    read of an add goes to one sample; row q of results_samples / winners_samples is exactly what a one-sample
    screen fed only sample q's reads would answer.  With the default samples=1 and sample=0 everything is the
    single-pool screen."""

    def __init__(self, sketches, k: int, samples: int = 1, canonical: bool = False):
        rows = _sketch_rows(sketches)
        n, s = int(rows.shape[0]), int(rows.shape[1])
        if not -(1 << 31) <= k < (1 << 31):
            raise PolyError(_lib.PG_ERR_ARG, f"k-mer size {k} does not fit 32 bits")
        samples = int(samples)
        if not 0 <= samples < (1 << 32):
            raise PolyError(_lib.PG_ERR_ARG, f"{samples} samples do not fit 32 bits")
        h = C.c_void_p()
        if hasattr(rows, "data_ptr"):
            import torch

            rc = _lib.lib().pg_mash_screen_create_flags_dev(rows.data_ptr(), n, s, k, samples, _kmer_flags(canonical),
                                                            torch.cuda.current_stream(rows.device).cuda_stream, C.byref(h))
        else:
            rc = _lib.lib().pg_mash_screen_create_flags(rows.ctypes.data, n, s, k, samples, _kmer_flags(canonical), C.byref(h))
        _index_rc(rc)
        self._h = h
        self._dev_used = None
        self.n, self.s, self.k, self.samples = n, s, int(k), samples
        self.canonical = bool(canonical)

    def _live(self):
        if self._h is None:
            raise ValueError("the screen is closed")
        return self._h

    def _sync_dev(self):
        """Host calls run on the library's own stream: wait for device adds enqueued on torch's streams."""
        if self._dev_used is not None:
            import torch

            torch.cuda.synchronize(self._dev_used)

    def add(self, reads, sample=0) -> None:
        """Adds host reads to the pool: a list of str / bytes / uint8 arrays, or (bases, offsets) as flatten returns.
        sample: the sample every read goes to (an int), or one sample id per read (a uint32 array)."""
        h = self._live()
        if isinstance(reads, tuple) and len(reads) == 2 and isinstance(reads[0], np.ndarray):
            bases, offsets = np.ascontiguousarray(reads[0], np.uint8), np.ascontiguousarray(reads[1], np.uint64)
        else:
            bases, offsets = flatten(reads)
        n_reads = max(len(offsets) - 1, 0)
        ids = self._sample_ids(sample, n_reads)
        if n_reads == 0:
            return
        if len(bases) == 0:
            bases = np.zeros(1, np.uint8)
        self._sync_dev()
        if ids is None:
            _lib.check(_lib.lib().pg_mash_screen_add(h, bases.ctypes.data, offsets.ctypes.data, n_reads))
        else:
            _lib.check(_lib.lib().pg_mash_screen_add_samples(h, bases.ctypes.data, offsets.ctypes.data, ids.ctypes.data, n_reads))

    def _sample_ids(self, sample, n_reads):
        """None for sample 0 (the single-sample add), else the uint32 id of every read."""
        if np.ndim(sample) == 0:
            q = int(sample)
            if not 0 <= q < self.samples:
                raise PolyError(_lib.PG_ERR_ARG, f"sample {q} of a screen of {self.samples} samples")
            return None if q == 0 else np.full(n_reads, q, np.uint32)
        ids = np.asarray(sample)
        if ids.dtype.kind not in "iu":
            raise ValueError("sample ids must be integers")
        if ids.shape != (n_reads,):
            raise ValueError(f"{ids.shape[0] if ids.ndim == 1 else ids.shape} sample ids for {n_reads} reads")
        if len(ids) and (ids.min() < 0 or ids.max() > 0xFFFFFFFF):
            raise ValueError("sample ids must fit uint32")
        return np.ascontiguousarray(ids, np.uint32)

    def add_dev(self, d_bases, d_offsets, stream=None, d_samples=None) -> None:
        """Adds reads already on the device: uint8 bases and int64 (uint64 bits) offsets tensors, read i being
        d_bases[d_offsets[i] : d_offsets[i + 1]].  d_samples: None (every read is sample 0) or an int32 / uint32
        tensor of one sample id per read, trusted as the offsets are: a read whose id is not a sample counts
        nowhere.  Only enqueues, on `stream` (default: the current stream)."""
        h = self._live()
        import torch

        n_reads = max(int(d_offsets.numel()) - 1, 0)
        if d_samples is not None:
            if d_samples.element_size() != 4 or d_samples.numel() != n_reads or not d_samples.is_contiguous():
                raise ValueError("d_samples must be a contiguous 32-bit tensor of one id per read")
        if n_reads == 0:
            return
        st = (stream if stream is not None else torch.cuda.current_stream(d_bases.device)).cuda_stream
        if d_samples is None:
            _lib.check(_lib.lib().pg_mash_screen_add_dev(h, d_bases.data_ptr(), d_offsets.data_ptr(), n_reads, st))
        else:
            _lib.check(_lib.lib().pg_mash_screen_add_samples_dev(h, d_bases.data_ptr(), d_offsets.data_ptr(), d_samples.data_ptr(), n_reads, st))
        self._dev_used = d_bases.device

    def reset(self) -> None:
        """Empties the pool: the screen then answers as a freshly created one."""
        h = self._live()
        self._sync_dev()
        _lib.check(_lib.lib().pg_mash_screen_reset(h))

    def _table(self, fn, first, count):
        h = self._live()
        first = int(first)
        count = self.samples - first if count is None else int(count)
        if not (0 <= first < (1 << 32) and 0 <= count < (1 << 32)):
            raise PolyError(_lib.PG_ERR_ARG, f"rows [{first}, {first + count}) of a screen of {self.samples} samples")
        self._sync_dev()
        shared = np.zeros((max(count, 0), self.n), np.uint32)
        cont = np.zeros(shared.shape, np.float64)
        mult = np.zeros(shared.shape, np.uint64)
        _lib.check(fn(h, first, count, shared.ctypes.data, cont.ctypes.data, mult.ctypes.data))
        return shared, cont, mult

    def results(self, sample: int = 0):
        """(shared [n] uint32, containment [n] float64, multiplicity [n] uint64) of the pool (of sample `sample`) so far."""
        return tuple(x[0] for x in self._table(_lib.lib().pg_mash_screen_results_samples, sample, 1))

    def results_samples(self, first: int = 0, count: Optional[int] = None):
        """results() of samples [first, first + count) (count defaults to every sample from first) from one call:
        (shared, containment, multiplicity), each [count, n]."""
        return self._table(_lib.lib().pg_mash_screen_results_samples, first, count)

    def winners(self, sample: int = 0):
        """Mash Screen's winner-take-all (mash screen -w): each pool hash goes to the reference that holds it with
        the largest first-pass shared (ties to the smallest index), and the (shared, containment, multiplicity) of
        results() are recomputed over the hashes each reference won.  A strain's siblings then stop reporting the
        hashes it explains better.  Each sample votes alone.  The screen is left as it was."""
        return tuple(x[0] for x in self._table(_lib.lib().pg_mash_screen_winners_samples, sample, 1))

    def winners_samples(self, first: int = 0, count: Optional[int] = None):
        """winners() of samples [first, first + count) from one call: (shared, containment, multiplicity), each [count, n]."""
        return self._table(_lib.lib().pg_mash_screen_winners_samples, first, count)

    def identity(self, sample: int = 0) -> np.ndarray:
        """Mash Screen's identity estimate containment ** (1 / k), computed on the host from results(sample)."""
        if self.k <= 0:
            raise ValueError("identity needs k > 0")
        return self.results(sample)[1] ** (1.0 / self.k)

    def close(self) -> None:
        if self._h is not None:
            self._sync_dev()
            h, self._h = self._h, None
            _lib.check(_lib.lib().pg_mash_screen_free(h))

    def __enter__(self) -> "Screen":
        return self

    def __exit__(self, *exc) -> None:
        self.close()

    def __del__(self):
        if getattr(self, "_h", None) is not None:
            try:
                self.close()
            except Exception:
                pass


# ---- single-process multi-GPU additions (pg_*_multi; SURVEY.md 8b / 8e) ----------------------------
def _device_list(devices):
    if devices is None:
        return None, 0
    arr = np.ascontiguousarray(devices, dtype=np.int32)
    return arr, len(arr)


def sketch_uniform_multi(bases: np.ndarray, n_reads: int, read_len: int, k: int, s: int, devices=None, out: Optional[np.ndarray] = None) -> np.ndarray:
    """sketch_uniform with the batch sharded over several GPUs of this process (all visible ones
    by default): one call, no data-path collective."""
    bases = np.ascontiguousarray(bases, dtype=np.uint8) if not hasattr(bases, "data_ptr") else bases
    cnt = min(max(read_len - k, 0), s)
    if out is None:
        out = np.zeros((n_reads, max(cnt, 1)), dtype=np.uint32)
    dev, nd = _device_list(devices)
    rc = _lib.lib().pg_mash_sketch_uniform_multi(_lib.ptr(bases), n_reads, read_len, k, s, 0, _lib.ptr(out), max(cnt, 1), None,
                                                 _lib.ptr(dev), nd)
    if rc == _lib.PG_ERR_PANIC:
        raise GoPanic("index out of range [-1]")
    _lib.check(rc)
    return out[:, :cnt] if isinstance(out, np.ndarray) else out


def sketch_arrays_multi(bases: np.ndarray, offsets: np.ndarray, k: int, s: int, pad_zero: bool = False, devices=None):
    """sketch_arrays (ragged reads) sharded over several GPUs of this process."""
    bases = np.ascontiguousarray(bases, dtype=np.uint8)
    offsets = np.ascontiguousarray(offsets, dtype=np.uint64)
    n = len(offsets) - 1
    lens = np.diff(offsets.astype(np.int64)) if n else np.zeros(0, np.int64)
    maxn = int(max(int(lens.max()) - k, 0)) if n else 0
    stride = s if pad_zero else min(maxn, s)
    out = np.zeros((n, max(stride, 1)), dtype=np.uint32)
    count = np.zeros(n, dtype=np.uint32)
    status = np.zeros(n, dtype=np.int32)
    dev, nd = _device_list(devices)
    rc = _lib.lib().pg_mash_sketch_batch_multi(bases.ctypes.data, offsets.ctypes.data, n, k, s, _lib.PG_SKETCH_PAD_ZERO if pad_zero else 0,
                                               out.ctypes.data, max(stride, 1), count.ctypes.data, status.ctypes.data, _lib.ptr(dev), nd)
    _lib.check(rc, allow=(_lib.PG_ERR_PANIC,))
    return out, count, status


def sketch_distance_multi(bases: np.ndarray, n_reads: int, read_len: int, k: int, s: int, devices=None, want_sketches: bool = True,
                          want_same: bool = True, want_distance: bool = False):
    """Sketch every read and compute the all-pairs matrix on several GPUs of this process: the sketch
    kernels store their results into every device's gathered buffer (fused all-gather over peer
    memory), device r then computes row block r.  Returns (sketches [n, s], same [n, n], distance [n, n])."""
    bases = np.ascontiguousarray(bases, dtype=np.uint8)
    sk = np.zeros((n_reads, s), dtype=np.uint32) if want_sketches else None
    same = np.zeros((n_reads, n_reads), dtype=np.uint32) if want_same else None
    dist = np.zeros((n_reads, n_reads), dtype=np.float64) if want_distance else None
    dev, nd = _device_list(devices)
    rc = _lib.lib().pg_mash_sketch_distance_multi(bases.ctypes.data, n_reads, read_len, k, s, _lib.ptr(dev), nd, _lib.ptr(sk), _lib.ptr(same),
                                                  _lib.ptr(dist))
    if rc == _lib.PG_ERR_PANIC:
        raise GoPanic("index out of range [-1]")
    _lib.check(rc)
    return sk, same, dist
