"""Host-side mirror of poly's search/align (Smith-Waterman SCORE), alphabet and
search/align/matrix packages over libpolyb200.so.

Mirrors /root/reference/alphabet/alphabet.go:25-61 (`NewAlphabet`, `Encode`, `Error`),
search/align/matrix/matrix.go:13-38 (`NewSubstitutionMatrix`, `Score`, `Default`),
search/align/matrix/matrices.go:33-40 (`NUC_4`) and search/align/align.go:73-95,171-203
(`Scoring`, `NewScoring`, `SmithWaterman`).  `SmithWaterman` returns the score (raising the
reference's `alphabet.Error`); `SmithWatermanAlign` additionally returns the two aligned strings
of the reference's traceback (align.go:205-231; queries of <= 64 symbols); `NeedlemanWunsch`
returns the global score.  All DP cells and the traceback are computed on the GPU.
"""
from __future__ import annotations

from typing import List, Optional, Sequence, Tuple

import ctypes as C

import numpy as np

from . import _lib
from .mash import BytesLike, _as_bytes, flatten


class AlphabetError(Exception):
    """alphabet.Error (alphabet.go:14-22)."""


class Alphabet:
    """alphabet.Alphabet (alphabet.go:9-12): symbols are strings; a sequence byte b is
    looked up as Go's string(b), i.e. the UTF-8 encoding of code point b (align.go:90)."""

    def __init__(self, symbols: Sequence[str]):
        self.symbols = list(symbols)
        self.encoding = {}
        for i, sym in enumerate(self.symbols):  # alphabet.go:27-30 (later duplicates win)
            self.encoding[sym] = i

    def Encode(self, symbol: str) -> int:
        if symbol not in self.encoding:
            raise AlphabetError(f"Symbol {symbol} not in alphabet")  # alphabet.go:38
        return self.encoding[symbol]

    def Symbols(self) -> List[str]:
        return self.symbols

    def byte_lut(self) -> np.ndarray:
        lut = np.full(256, -1, dtype=np.int16)
        for b in range(256):
            lut[b] = self.encoding.get(chr(b), -1)
        return lut


def NewAlphabet(symbols: Sequence[str]) -> Alphabet:
    return Alphabet(symbols)


class SubstitutionMatrix:
    """matrix.SubstitutionMatrix (matrix.go:13-17)."""

    def __init__(self, first: Alphabet, second: Alphabet, scores):
        scores = np.asarray(scores, dtype=np.int64)
        if scores.ndim != 2 or len(first.Symbols()) != scores.shape[0] or len(second.Symbols()) != scores.shape[1]:
            raise ValueError("invalid dimensions of substitution matrix")  # matrix.go:21-23
        self.FirstAlphabet, self.SecondAlphabet, self.scores = first, second, scores

    def Score(self, a: str, b: str) -> int:  # matrix.go:28-38
        return int(self.scores[self.FirstAlphabet.Encode(a), self.SecondAlphabet.Encode(b)])


def NewSubstitutionMatrix(first: Alphabet, second: Alphabet, scores) -> SubstitutionMatrix:
    return SubstitutionMatrix(first, second, scores)


_LETTERS = [chr(ord("A") + i) for i in range(26)]
Default = SubstitutionMatrix(Alphabet(_LETTERS), Alphabet(_LETTERS), 2 * np.eye(26, dtype=np.int64) - 1)  # matrix.go:41-74
NUC_4 = [[0, 0, 0, 0, 0], [0, 5, -4, -4, -4], [0, -4, 5, -4, -4], [0, -4, -4, 5, -4], [0, -4, -4, -4, 5]]  # matrices.go:33-40


class Scoring:
    """align.Scoring (align.go:73-76)."""

    def __init__(self, substitution_matrix: Optional[SubstitutionMatrix], gap_penalty: int):
        self.SubstitutionMatrix = substitution_matrix if substitution_matrix is not None else Default  # align.go:80-82
        self.GapPenalty = int(gap_penalty)


def NewScoring(substitution_matrix: Optional[SubstitutionMatrix], gap_penalty: int) -> Scoring:
    return Scoring(substitution_matrix, gap_penalty)


def sw_scores_arrays(q_bases: np.ndarray, q_offsets: np.ndarray, template: BytesLike, scoring: Scoring,
                     query_is_a: bool = True, global_alignment: bool = False) -> Tuple[np.ndarray, np.ndarray, np.ndarray]:
    """(score, err_code, err_pos) for every query against one template (Smith-Waterman, or the
    Needleman-Wunsch score with global_alignment=True)."""
    m = scoring.SubstitutionMatrix
    lut_a, lut_b = m.FirstAlphabet.byte_lut(), m.SecondAlphabet.byte_lut()
    table = np.ascontiguousarray(m.scores, dtype=np.int64)
    t = _as_bytes(template)
    q_bases = np.ascontiguousarray(q_bases, dtype=np.uint8)
    q_offsets = np.ascontiguousarray(q_offsets, dtype=np.uint64)
    n = len(q_offsets) - 1
    score, ec, ep = np.zeros(n, np.int64), np.zeros(n, np.int32), np.zeros(n, np.int64)
    fn = _lib.lib().pg_nw_score_batch if global_alignment else _lib.lib().pg_sw_score_batch
    rc = fn(q_bases.ctypes.data, q_offsets.ctypes.data, n, t.ctypes.data, len(t), int(query_is_a),
                                      lut_a.ctypes.data, lut_b.ctypes.data, table.ctypes.data, table.shape[0], table.shape[1],
                                      scoring.GapPenalty, score.ctypes.data, ec.ctypes.data, ep.ctypes.data)
    _lib.check(rc)
    return score, ec, ep


def _error_for(ec: int, ep: int, a: np.ndarray, b: np.ndarray) -> AlphabetError:
    byte = int(a[ep]) if ec == 1 else int(b[ep])
    return AlphabetError(f"Symbol {chr(byte)} not in alphabet")  # alphabet.go:38 via align.go:189-191


def SmithWatermanScores(queries: Sequence[BytesLike], template: BytesLike, scoring: Scoring,
                        query_is_a: bool = True, global_alignment: bool = False) -> Tuple[List[int], List[Optional[AlphabetError]]]:
    """Batched addition: score (and error) of SmithWaterman(query, template) per query
    (or SmithWaterman(template, query) with query_is_a=False)."""
    bases, offsets = flatten(queries)
    score, ec, ep = sw_scores_arrays(bases, offsets, template, scoring, query_is_a, global_alignment)
    t = _as_bytes(template)
    errs: List[Optional[AlphabetError]] = []
    for i in range(len(queries)):
        if ec[i]:
            q = bases[int(offsets[i]): int(offsets[i + 1])]
            errs.append(_error_for(int(ec[i]), int(ep[i]), q if query_is_a else t, t if query_is_a else q))
        else:
            errs.append(None)
    return [int(x) for x in score], errs


def SmithWatermanScore(stringA: BytesLike, stringB: BytesLike, scoring: Scoring) -> int:
    """Score of align.SmithWaterman(stringA, stringB, scoring) (align.go:171-203), score kernel only.
    Raises AlphabetError where the reference returns (0, "", "", err)."""
    scores, errs = SmithWatermanScores([stringA], stringB, scoring, query_is_a=True)
    if errs[0] is not None:
        raise errs[0]
    return scores[0]


def NeedlemanWunschScores(queries: Sequence[BytesLike], template: BytesLike, scoring: Scoring, query_is_a: bool = True):
    """Batched score of align.NeedlemanWunsch(query, template) (align.go:100-134,166)."""
    return SmithWatermanScores(queries, template, scoring, query_is_a, global_alignment=True)


def NeedlemanWunschScore(stringA: BytesLike, stringB: BytesLike, scoring: Scoring) -> int:
    """Score of align.NeedlemanWunsch(stringA, stringB, scoring); the aligned strings are not built."""
    scores, errs = NeedlemanWunschScores([stringA], stringB, scoring)
    if errs[0] is not None:
        raise errs[0]
    return scores[0]


def SmithWatermanAligns(queries: Sequence[BytesLike], template: BytesLike, scoring: Scoring, query_is_a: bool = True,
                        global_alignment: bool = False):
    """Batched full align.SmithWaterman (or NeedlemanWunsch with global_alignment=True):
    [(score, alignA, alignB, err)] per query (stringA = query when query_is_a, else the template)."""
    m = scoring.SubstitutionMatrix
    lut_a, lut_b = m.FirstAlphabet.byte_lut(), m.SecondAlphabet.byte_lut()
    table = np.ascontiguousarray(m.scores, dtype=np.int64)
    t = _as_bytes(template)
    bases, offsets = flatten(queries)
    n = len(queries)
    maxq = max((len(_as_bytes(q)) for q in queries), default=0)
    stride = max(2 * maxq + 64, 64) if not global_alignment else maxq + len(t) + 8
    fn = _lib.lib().pg_nw_align_batch if global_alignment else _lib.lib().pg_sw_align_batch
    while True:
        score, ec, ep = np.zeros(n, np.int64), np.zeros(n, np.int32), np.zeros(n, np.int64)
        oa, ob = np.zeros((n, stride), np.uint8), np.zeros((n, stride), np.uint8)
        ln, st = np.zeros(n, np.uint32), np.zeros(n, np.int32)
        rc = fn(bases.ctypes.data, offsets.ctypes.data, n, t.ctypes.data, len(t), int(query_is_a),
                                          lut_a.ctypes.data, lut_b.ctypes.data, table.ctypes.data, table.shape[0], table.shape[1],
                                          scoring.GapPenalty, score.ctypes.data, ec.ctypes.data, ep.ctypes.data, oa.ctypes.data,
                                          ob.ctypes.data, stride, ln.ctypes.data, st.ctypes.data)
        _lib.check(rc)
        if (st == _lib.PG_ITEM_UNSUPPORTED).any():  # an alignment longer than the row: grow and retry
            stride = int(ln.max()) + 8
            continue
        break
    res = []
    for i in range(n):
        if ec[i]:
            q = bases[int(offsets[i]): int(offsets[i + 1])]
            res.append((0, "", "", _error_for(int(ec[i]), int(ep[i]), q if query_is_a else t, t if query_is_a else q)))
        else:
            res.append((int(score[i]), bytes(oa[i, : ln[i]]).decode("latin-1"), bytes(ob[i, : ln[i]]).decode("latin-1"), None))
    return res


def SmithWatermanAlign(stringA: BytesLike, stringB: BytesLike, scoring: Scoring) -> Tuple[int, str, str]:
    """align.SmithWaterman(stringA, stringB, scoring) -> (score, alignA, alignB); raises
    AlphabetError where the reference returns (0, "", "", err).  A string of <= 64 symbols rides in
    registers; when both are longer the whole matrix is kept in HBM, as the reference keeps it on the heap."""
    a, b = _as_bytes(stringA), _as_bytes(stringB)
    if len(a) <= 64:
        score, sa, sb, err = SmithWatermanAligns([a], b, scoring, query_is_a=True)[0]
    else:
        score, sa, sb, err = SmithWatermanAligns([b], a, scoring, query_is_a=False)[0]
    if err is not None:
        raise err
    return score, sa, sb


def NeedlemanWunschAlign(stringA: BytesLike, stringB: BytesLike, scoring: Scoring) -> Tuple[int, str, str]:
    """align.NeedlemanWunsch(stringA, stringB, scoring) -> (score, alignA, alignB) (align.go:100-166),
    including the reference's loop condition (the traceback stops when one string is exhausted)."""
    a, b = _as_bytes(stringA), _as_bytes(stringB)
    if len(a) <= 64:
        score, sa, sb, err = SmithWatermanAligns([a], b, scoring, query_is_a=True, global_alignment=True)[0]
    else:
        score, sa, sb, err = SmithWatermanAligns([b], a, scoring, query_is_a=False, global_alignment=True)[0]
    if err is not None:
        raise err
    return score, sa, sb


def SmithWaterman(stringA: BytesLike, stringB: BytesLike, scoring: Scoring):
    """align.SmithWaterman (align.go:171-232) with the reference's own return shape:
    (score, alignA, alignB, err) -- err is None or the AlphabetError, and (0, "", "", err) on error."""
    try:
        return SmithWatermanAlign(stringA, stringB, scoring) + (None,)
    except AlphabetError as e:
        return 0, "", "", e


def NeedlemanWunsch(stringA: BytesLike, stringB: BytesLike, scoring: Scoring):
    """align.NeedlemanWunsch (align.go:100-166) with the reference's own return shape:
    (score, alignA, alignB, err)."""
    try:
        return NeedlemanWunschAlign(stringA, stringB, scoring) + (None,)
    except AlphabetError as e:
        return 0, "", "", e


# ---- pair lists: pair p aligns stringA = seqs_a[pairs[p, 0]] against stringB = seqs_b[pairs[p, 1]] ----

def _pair_inputs(seqs_a, seqs_b, pairs, scoring: Scoring):
    """Flattened sets, the two index columns of the (n, 2) pair array, LUTs and table."""
    m = scoring.SubstitutionMatrix
    lut_a, lut_b = m.FirstAlphabet.byte_lut(), m.SecondAlphabet.byte_lut()
    table = np.ascontiguousarray(m.scores, dtype=np.int64)
    ba, oa = seqs_a if isinstance(seqs_a, tuple) else flatten(seqs_a)
    bb, ob = seqs_b if isinstance(seqs_b, tuple) else flatten(seqs_b)
    pairs = np.asarray(pairs)
    if pairs.size == 0:
        pairs = pairs.reshape(0, 2)
    if pairs.ndim != 2 or pairs.shape[1] != 2:
        raise ValueError(f"pairs must be an (n, 2) array, got shape {pairs.shape}")
    if pairs.size and (pairs.min() < 0 or pairs.max() > 0xFFFFFFFF):
        raise ValueError("pair indices must lie in [0, 2^32)")
    pa = np.ascontiguousarray(pairs[:, 0], dtype=np.uint32)
    pb = np.ascontiguousarray(pairs[:, 1], dtype=np.uint32)
    return (np.ascontiguousarray(ba, np.uint8), np.ascontiguousarray(oa, np.uint64), np.ascontiguousarray(bb, np.uint8),
            np.ascontiguousarray(ob, np.uint64), pa, pb, lut_a, lut_b, table)


def pair_scores_arrays(seqs_a, seqs_b, pairs, scoring: Scoring, global_alignment: bool = False):
    """(score, err_code, err_pos) NumPy arrays for every pair (pg_sw_score_pairs / pg_nw_score_pairs).
    seqs_a / seqs_b: lists of sequences or (bases, offsets) arrays; pairs: (n, 2) integer array."""
    ba, oa, bb, ob, pa, pb, lut_a, lut_b, table = _pair_inputs(seqs_a, seqs_b, pairs, scoring)
    n = len(pa)
    score, ec, ep = np.zeros(n, np.int64), np.zeros(n, np.int32), np.zeros(n, np.int64)
    fn = _lib.lib().pg_nw_score_pairs if global_alignment else _lib.lib().pg_sw_score_pairs
    _lib.check(fn(ba.ctypes.data, oa.ctypes.data, len(oa) - 1, bb.ctypes.data, ob.ctypes.data, len(ob) - 1, pa.ctypes.data, pb.ctypes.data, n,
                  lut_a.ctypes.data, lut_b.ctypes.data, table.ctypes.data, table.shape[0], table.shape[1], scoring.GapPenalty,
                  score.ctypes.data, ec.ctypes.data, ep.ctypes.data))
    return score, ec, ep


def _pair_errors(ec, ep, ba, oa, bb, ob, pa, pb) -> List[Optional[AlphabetError]]:
    errs: List[Optional[AlphabetError]] = []
    for k in range(len(ec)):
        if ec[k]:
            i, j = int(pa[k]), int(pb[k])
            errs.append(_error_for(int(ec[k]), int(ep[k]), ba[int(oa[i]): int(oa[i + 1])], bb[int(ob[j]): int(ob[j + 1])]))
        else:
            errs.append(None)
    return errs


def SmithWatermanPairScores(seqs_a, seqs_b, pairs, scoring: Scoring, global_alignment: bool = False):
    """Batched align.SmithWaterman(seqs_a[i], seqs_b[j], scoring) score for every (i, j) row of `pairs`:
    (scores, errors) as SmithWatermanScores returns them."""
    ba, oa, bb, ob, pa, pb, _, _, _ = _pair_inputs(seqs_a, seqs_b, pairs, scoring)
    score, ec, ep = pair_scores_arrays((ba, oa), (bb, ob), np.stack([pa, pb], 1), scoring, global_alignment)
    return [int(x) for x in score], _pair_errors(ec, ep, ba, oa, bb, ob, pa, pb)


def NeedlemanWunschPairScores(seqs_a, seqs_b, pairs, scoring: Scoring):
    """Batched align.NeedlemanWunsch(seqs_a[i], seqs_b[j], scoring) score for every (i, j) row of `pairs`."""
    return SmithWatermanPairScores(seqs_a, seqs_b, pairs, scoring, global_alignment=True)


def SmithWatermanPairAligns(seqs_a, seqs_b, pairs, scoring: Scoring, global_alignment: bool = False):
    """Full align.SmithWaterman (NeedlemanWunsch with global_alignment=True) for every (i, j) row of
    `pairs`: [(score, alignA, alignB, err)], as SmithWatermanAligns returns them."""
    ba, oa, bb, ob, pa, pb, lut_a, lut_b, table = _pair_inputs(seqs_a, seqs_b, pairs, scoring)
    n = len(pa)
    la, lb = np.diff(oa.astype(np.int64)), np.diff(ob.astype(np.int64))
    longest = int((la[pa] + lb[pb]).max()) if n else 0
    stride = max(longest, 1)  # an alignment never has more columns than len(a) + len(b)
    fn = _lib.lib().pg_nw_align_pairs if global_alignment else _lib.lib().pg_sw_align_pairs
    score, ec, ep = np.zeros(n, np.int64), np.zeros(n, np.int32), np.zeros(n, np.int64)
    out_a, out_b = np.zeros((max(n, 1), stride), np.uint8), np.zeros((max(n, 1), stride), np.uint8)
    ln, st = np.zeros(n, np.uint32), np.zeros(n, np.int32)
    _lib.check(fn(ba.ctypes.data, oa.ctypes.data, len(oa) - 1, bb.ctypes.data, ob.ctypes.data, len(ob) - 1, pa.ctypes.data, pb.ctypes.data, n,
                  lut_a.ctypes.data, lut_b.ctypes.data, table.ctypes.data, table.shape[0], table.shape[1], scoring.GapPenalty,
                  score.ctypes.data, ec.ctypes.data, ep.ctypes.data, out_a.ctypes.data, out_b.ctypes.data, stride, ln.ctypes.data,
                  st.ctypes.data))
    errs = _pair_errors(ec, ep, ba, oa, bb, ob, pa, pb)
    return [(0, "", "", errs[k]) if errs[k] is not None else
            (int(score[k]), bytes(out_a[k, : ln[k]]).decode("latin-1"), bytes(out_b[k, : ln[k]]).decode("latin-1"), None)
            for k in range(n)]


def NeedlemanWunschPairAligns(seqs_a, seqs_b, pairs, scoring: Scoring):
    """Full align.NeedlemanWunsch for every (i, j) row of `pairs`: [(score, alignA, alignB, err)]."""
    return SmithWatermanPairAligns(seqs_a, seqs_b, pairs, scoring, global_alignment=True)


def pair_scores_device(d_seqs_a, d_offsets_a, max_len_a: int, d_seqs_b, d_offsets_b, max_len_b: int, d_pairs, scoring: Scoring,
                       global_alignment: bool = False, stream=None):
    """pg_sw_score_pairs_dev / pg_nw_score_pairs_dev on torch CUDA tensors: d_offsets_* int64 [n + 1], d_pairs an
    integer [n, 2] tensor (int32 is taken as the uint32 bits of the index; wider indices outside [0, 2^32) are
    flagged, never truncated to a valid one).  Returns (score int64[n],
    err_code int32[n], err_pos int64[n]) on the device; err_code PG_PAIR_OUT_OF_RANGE (3) marks a pair
    whose index or length is out of range.  Only enqueues work on the stream."""
    import torch

    m = scoring.SubstitutionMatrix
    lut_a, lut_b = m.FirstAlphabet.byte_lut(), m.SecondAlphabet.byte_lut()
    table = np.ascontiguousarray(m.scores, dtype=np.int64)
    dev = d_offsets_a.device
    if d_pairs.dim() != 2 or d_pairs.shape[1] != 2:
        raise ValueError(f"d_pairs must be an (n, 2) tensor, got shape {tuple(d_pairs.shape)}")

    def column(x):  # uint32 bits; an index outside [0, 2^32) becomes 2^32 - 1, which the kernel flags (no host sync)
        if x.dtype == torch.int32:
            return x.contiguous()
        x = x.to(torch.int64)
        return torch.where((x < 0) | (x > 0xFFFFFFFF), torch.full_like(x, 0xFFFFFFFF), x).to(torch.int32).contiguous()

    pa, pb = column(d_pairs[:, 0]), column(d_pairs[:, 1])
    n = pa.numel()
    score = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    code = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    pos = torch.empty(max(n, 1), dtype=torch.int64, device=dev)
    st = stream if stream is not None else torch.cuda.current_stream(dev).cuda_stream
    fn = _lib.lib().pg_nw_score_pairs_dev if global_alignment else _lib.lib().pg_sw_score_pairs_dev
    _lib.check(fn(d_seqs_a.data_ptr(), d_offsets_a.data_ptr(), d_offsets_a.numel() - 1, max_len_a, d_seqs_b.data_ptr(), d_offsets_b.data_ptr(),
                  d_offsets_b.numel() - 1, max_len_b, pa.data_ptr(), pb.data_ptr(), n, lut_a.ctypes.data, lut_b.ctypes.data,
                  table.ctypes.data, table.shape[0], table.shape[1], scoring.GapPenalty, score.data_ptr(), code.data_ptr(),
                  pos.data_ptr(), C.c_void_p(st)))
    return score[:n], code[:n], pos[:n]
