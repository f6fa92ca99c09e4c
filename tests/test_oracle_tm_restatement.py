"""A second, independent statement of primers.SantaLucia (primers/primers.go:70-105), written in Python, pinned
bit for bit against the oracle's po_santalucia over the sequences and (cp, na, mg) triples that
test_gpu_tm_bits.py sends to the GPU.  It runs without a GPU, so a change to the oracle's statement order or
constants is caught here before it can move the GPU tests' yardstick.

The restatement does the reference's float64 arithmetic in its statement order.  It is vectorised over the
parameter triples with numpy, whose elementwise + * / are the correctly rounded IEEE operations that Python
floats use, and it takes every log from math.log (libm's log, as the oracle's)."""
import math

import numpy as np

import oracle_ffi as o
from pcr_util import revcomp

NN = {  # primers.go:42-59; absent pairs read as the map's zero value {0, 0} (primers.go:98)
    b"AA": (-7.6, -21.3), b"TT": (-7.6, -21.3), b"AT": (-7.2, -20.4), b"TA": (-7.2, -21.3),
    b"CA": (-8.5, -22.7), b"TG": (-8.5, -22.7), b"GT": (-8.4, -22.4), b"AC": (-8.4, -22.4),
    b"CT": (-7.8, -21.0), b"AG": (-7.8, -21.0), b"GA": (-8.2, -22.2), b"TC": (-8.2, -22.2),
    b"CG": (-10.6, -27.2), b"GC": (-9.8, -24.4), b"GG": (-8.0, -19.9), b"CC": (-8.0, -19.9),
}


def tm_sequences():
    """Primers that reach every branch of SantaLucia, plus one empty (PANIC) and one non-ASCII (UNSUPPORTED) item."""
    rng = np.random.default_rng(51)

    def pick(alphabet, n):
        return bytes(rng.choice(list(alphabet), size=int(n)).astype(np.uint8))

    seqs = [pick(b"ACGT", n) for n in rng.integers(1, 61, 60)]
    seqs += [pick(b"ACGTacgtNnRYSWKMBDHVU\x00 ", n) for n in rng.integers(1, 61, 40)]  # lower case, IUPAC, N, NUL, space
    halves = [pick(b"ACGT", n) for n in rng.integers(1, 31, 20)]
    seqs += [h + revcomp(h) for h in halves]                                 # even-length ACGT palindromes: symmetry = 1
    seqs += [(h + revcomp(h)).lower() for h in halves[:4]]
    seqs += [c * n for c in (b"S", b"W", b"N", b"\x00") for n in (1, 2, 7, 20)]  # self-complementary at any length
    seqs += [b"A\x00T", b"GN\x00NC", b"ACGTN"]
    seqs += [pick(b"ACGT", 24) + end for end in (b"A", b"T", b"C", b"G", b"a", b"t", b"N", b" ")]  # 3' end A/T or not
    seqs += [bytes([a]) for a in b"ACGTNa "] + [bytes([a, b]) for a in b"ACGT" for b in b"ACGT"]  # lengths 1 and 2
    seqs += [pick(b"ACGT", n) for n in (1000, 10_000, 100_000)]              # the (len-1) factor and long sums
    seqs += [pick(b"ACGTN", 3000)]
    seqs += [b"", b"AC\xc3\xa9"]
    return seqs


def tm_triples():
    """(cp, na, mg) triples: the reference's two, 2 000 random log-uniform ones, and IEEE special values."""
    rng = np.random.default_rng(52)
    n = 2000
    cp = 10.0 ** rng.uniform(-12, -3, n)
    na = 10.0 ** rng.uniform(-4, math.log10(2), n)
    mg = np.where(rng.random(n) < 0.25, 0.0, 10.0 ** rng.uniform(-5, -1, n))
    inf, nan = math.inf, math.nan
    return ([(500e-9, 50e-3, 0.0), (0.1e-6, 350e-3, 0.0)]                   # MeltingTemp's (primers.go:122-124), primers_test.go's
            + list(zip(cp.tolist(), na.tolist(), mg.tolist()))
            + [(500e-9, 0.0, 0.0), (500e-9, -0.0, 0.0),                      # log(0); at length 1, 0 * -inf
               (0.0, 50e-3, 0.0), (-0.0, 50e-3, 0.0), (5e-324, 50e-3, 0.0),  # cp / 4 underflows to 0
               (1e-310, 50e-3, 0.0), (2.2250738585072014e-308, 50e-3, 0.0),
               (-500e-9, 50e-3, 0.0), (500e-9, -50e-3, 0.0), (500e-9, 50e-3, -1e-3),
               (inf, 50e-3, 0.0), (500e-9, inf, 0.0), (500e-9, 50e-3, inf), (-inf, 50e-3, 0.0),
               (nan, 50e-3, 0.0), (500e-9, nan, 0.0), (500e-9, 50e-3, nan), (1.7976931348623157e308, 1e-300, 0.0)])


def _log(x: float) -> float:
    """math.log, with libm's results where Python raises instead: log(+-0) = -inf, log(x < 0) = nan."""
    if x == 0:
        return -math.inf
    if x < 0:
        return math.nan
    return math.log(x)


def santalucia_py(seq: bytes, triples):
    """primers.go:70-105 for one sequence over every triple: (rc, tm[T], dH, dS[T]), rc as the oracle's."""
    if len(seq) == 0:
        return o.PO_PANIC, None, None, None                                  # primers.go:89
    if any(c >= 0x80 for c in seq):
        return o.PO_UNSUPPORTED, None, None, None                            # strings.ToUpper would re-encode it
    seq = seq.upper()                                                        # primers.go:71
    cp, na, mg = (np.array(v, np.float64) for v in zip(*triples))
    gas_constant = 1.9872                                                    # primers.go:73
    dH, dS = 0.0, 0.0
    dH += 0.2                                                                # primers.go:78-79
    dS += -5.7
    if seq == revcomp(seq):                                                  # primers.go:81-87
        dH += 0.0
        dS += -1.4
        symmetry = 1.0
    else:
        symmetry = 4.0
    if seq[-1] in b"AT":                                                     # primers.go:89-92
        dH += 2.2
        dS += 6.9
    salt_effect = na + (mg * 140)                                            # primers.go:94
    with np.errstate(all="ignore"):
        dS = dS + (0.368 * float(len(seq) - 1) * np.array([_log(x) for x in salt_effect.tolist()]))  # primers.go:95
        for i in range(len(seq) - 1):                                        # primers.go:97-101
            h, s = NN.get(seq[i:i + 2], (0.0, 0.0))
            dH += h
            dS = dS + s
        log_cp = np.array([_log(c / symmetry) for c in cp.tolist()])
        tm = dH * 1000 / (dS + gas_constant * log_cp) - 273.15              # primers.go:103
    return o.PO_OK, tm, dH, dS


def oracle_table(seqs, triples):
    """po_santalucia of every (triple, sequence): rc int32[T, N], tm / dh / ds float64[T, N]."""
    T, N = len(triples), len(seqs)
    rc, tm, dh, ds = np.zeros((T, N), np.int32), np.zeros((T, N)), np.zeros((T, N)), np.zeros((T, N))
    for j, (cp, na, mg) in enumerate(triples):
        for i, s in enumerate(seqs):
            rc[j, i], tm[j, i], dh[j, i], ds[j, i] = o.santalucia(s, cp, na, mg)
    return rc, tm, dh, ds


def same_bits(got, want):
    """Elementwise: the same float64 bit pattern, or NaN on both sides (NaN payloads and signs are not defined
    across x86, CUDA and Go)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    return (got.view(np.uint64) == want.view(np.uint64)) | (np.isnan(got) & np.isnan(want))


def test_cases_reach_every_branch():
    seqs, triples = tm_sequences(), tm_triples()
    ok = [s.upper() for s in seqs if s and max(s) < 0x80]
    assert sum(s == revcomp(s) for s in ok) >= 30 and sum(s != revcomp(s) for s in ok) >= 100
    assert {s[-1:] in (b"A", b"T") for s in ok} == {True, False}
    assert {1, 2, 100_000} <= {len(s) for s in ok}
    assert len({_log(na + (mg * 140)) for _, na, mg in triples}) > 2000


def test_restatement_matches_oracle_bit_for_bit():
    seqs, triples = tm_sequences(), tm_triples()
    rc, tm, dh, ds = oracle_table(seqs, triples)
    for i, s in enumerate(seqs):
        prc, ptm, pdh, pds = santalucia_py(s, triples)
        assert (rc[:, i] == prc).all(), (i, s[:20])
        if prc != o.PO_OK:
            continue
        for name, got, want in (("tm", ptm, tm[:, i]), ("dH", np.full(len(triples), pdh), dh[:, i]), ("dS", pds, ds[:, i])):
            bad = np.flatnonzero(~same_bits(got, want))
            assert bad.size == 0, (f"{name} of sequence {i} (len {len(s)}): {bad.size} of {len(triples)} triples differ, "
                                   f"first {triples[bad[0]]}: {float(got[bad[0]]).hex()} vs {float(want[bad[0]]).hex()}")
    assert np.isnan(tm).any() and (tm == -273.15).any()  # the special triples reach NaN and dH * 1000 / -inf
