"""K5 (tm_kernel) and the two kernels that decide from Tm (design_primers_kernel, minimal_primer_kernel) against
the oracle, bit for bit.

DesignPrimers and SimulateSimple stop at the first candidate with !(Tm < target).  A Tm one ulp away from the
oracle's therefore changes a primer length, and with it the primer strings and PCR fragments, exactly when a
target sits on a candidate's Tm.  So Tm, dH and dS are compared by their float64 bit patterns (NaN equals NaN:
payloads are not defined across x86, CUDA and Go), and the searches are run at targets equal to a candidate's
oracle Tm and at that value's two float64 neighbours."""
import functools
import math

import numpy as np
import pytest

import pcr_util as P
from poly_b200 import _lib, pcr, primers
from poly_b200.mash import flatten
from test_oracle_align_primers import GENE, design_primers
from test_oracle_tm_restatement import oracle_table, same_bits, tm_sequences, tm_triples

pytestmark = pytest.mark.gpu

ITEM = {0: _lib.PG_ITEM_OK, -1: _lib.PG_ITEM_PANIC, -2: _lib.PG_ITEM_UNSUPPORTED}  # oracle rc -> item status


def neighbours(t: float):
    return t, math.nextafter(t, math.inf), math.nextafter(t, -math.inf)


@pytest.fixture(scope="module")
def tm_cases(oracle):
    seqs, triples = tm_sequences(), tm_triples()
    rc, tm, dh, ds = oracle_table(seqs, triples)
    return seqs, triples, (np.vectorize(ITEM.get)(rc).astype(np.int32), tm, dh, ds)


@pytest.fixture(scope="module")
def melting_temp(oracle):
    """oracle.melting_temp, memoised: the searches below ask for the same candidates many times."""
    return functools.lru_cache(maxsize=None)(oracle.melting_temp)


def assert_rows_match(seqs, triples, want, rows):
    """rows[j] = (tm, dh, ds, status) of triple j over seqs; dh, ds and status may be None (not requested).
    Values are compared where the oracle's status is OK, statuses everywhere."""
    w_st, w_tm, w_dh, w_ds = want
    bad = []
    for j, (tm, dh, ds, st) in enumerate(rows):
        ok = w_st[j] == _lib.PG_ITEM_OK
        d_tm = ~same_bits(tm, w_tm[j]) & ok
        d_hs = ((~same_bits(dh, w_dh[j]) | ~same_bits(ds, w_ds[j])) & ok) if dh is not None else np.zeros_like(ok)
        d_st = (st != w_st[j]) if st is not None else np.zeros_like(ok)
        if (d_tm | d_hs | d_st).any():
            bad.append((j, d_tm, d_hs, d_st))
    if bad:
        j, d_tm, d_hs, d_st = bad[0]
        i = int(np.flatnonzero(d_tm | d_hs | d_st)[0])
        tm, dh, ds, st = rows[j]
        pytest.fail(f"{len(bad)} of {len(rows)} parameter triples gave different bits "
                    f"({sum(int(b[1].sum()) for b in bad)} Tm, {sum(int(b[2].sum()) for b in bad)} dH/dS, "
                    f"{sum(int(b[3].sum()) for b in bad)} status items, of {len(seqs)} per triple); first: triple {triples[j]}, "
                    f"sequence {i} (len {len(seqs[i])}): Tm {float(tm[i]).hex()} vs {float(w_tm[j, i]).hex()}"
                    + (f", dH {float(dh[i]).hex()} vs {float(w_dh[j, i]).hex()}, dS {float(ds[i]).hex()} vs {float(w_ds[j, i]).hex()}"
                       if dh is not None else "")
                    + (f", status {st[i]} vs {w_st[j, i]}" if st is not None else ""))


def test_tm_batch_bits(gpu, tm_cases):
    """pg_tm_batch, one call per (cp, na, mg) triple."""
    seqs, triples, want = tm_cases
    bases, off = flatten(seqs)
    rows = [primers.santalucia_arrays(bases, off, cp, na, mg) for cp, na, mg in triples]
    assert_rows_match(seqs, triples, want, rows)


def test_melting_temps_bits(gpu, tm_cases):
    """primers.MeltingTemps (the defaults) over the items the oracle accepts."""
    seqs, triples, (w_st, w_tm, _, _) = tm_cases
    assert triples[0] == (primers.DEFAULT_CP, primers.DEFAULT_NA, primers.DEFAULT_MG)
    ok = np.flatnonzero(w_st[0] == _lib.PG_ITEM_OK)
    got = primers.MeltingTemps([seqs[i] for i in ok])
    assert same_bits(got, w_tm[0, ok]).all()
    assert same_bits([primers.MeltingTemp(seqs[i]) for i in ok[:20]], w_tm[0, ok[:20]]).all()


def test_tm_batch_dev_bits_on_a_stream(gpu, tm_cases):
    """pg_tm_batch_dev on a non-default stream; every other triple passes dh, ds and status as null, and then
    the Tm of a PANIC or UNSUPPORTED item must be left as it was."""
    import torch

    seqs, triples, want = tm_cases
    bases, off = flatten(seqs)
    n = len(seqs)
    stream = torch.cuda.Stream()
    L = _lib.lib()
    sentinel = -1.5e300
    with torch.cuda.stream(stream):
        d_bases = torch.from_numpy(bases).cuda()
        d_off = torch.from_numpy(off.view(np.int64)).cuda()
        tm = torch.empty(n, dtype=torch.float64, device="cuda")
        dh, ds = torch.empty_like(tm), torch.empty_like(tm)
        st = torch.empty(n, dtype=torch.int32, device="cuda")
        rows = []
        for j, (cp, na, mg) in enumerate(triples):
            full = j % 2 == 0
            tm.fill_(sentinel)
            _lib.check(L.pg_tm_batch_dev(d_bases.data_ptr(), d_off.data_ptr(), n, cp, na, mg, tm.data_ptr(),
                                         dh.data_ptr() if full else None, ds.data_ptr() if full else None,
                                         st.data_ptr() if full else None, stream.cuda_stream))
            out = [x.cpu().numpy() for x in (tm, dh, ds, st)] if full else [tm.cpu().numpy(), None, None, None]
            rows.append(tuple(out))
    stream.synchronize()
    assert_rows_match(seqs, triples, want, rows)
    w_st = want[0]
    for j in range(1, len(triples), 2):
        assert (rows[j][0][w_st[j] != _lib.PG_ITEM_OK] == sentinel).all(), triples[j]


# ---- DesignPrimers -----------------------------------------------------------------------------------------
def design_genes():
    rng = np.random.default_rng(53)
    p = [.22, .22, .22, .22, .02, .02, .02, .02, .04]
    genes = [bytes(rng.choice(list(b"ACGTacgtN"), size=int(rng.integers(15, 401)), p=p).astype(np.uint8)) for _ in range(300)]
    acgt = lambda n: bytes(rng.choice(list(b"ACGT"), size=n).astype(np.uint8))
    # exactly one candidate each way; N runs, whose Tm lies below -273.15 (dH > 0, the denominator < 0)
    genes += [acgt(15), b"N" * 40 + acgt(120) + b"n" * 30, b"N" * 15]
    return genes


def check_design(genes, target, melting_temp):
    fwd, rev, st = pcr.design_primer_lengths(genes, target)
    for i, g in enumerate(genes):
        try:
            wf, wr = design_primers(melting_temp, g.decode("latin-1"), target)
        except IndexError:
            assert st[i] == _lib.PG_ITEM_PANIC, (i, target)
            continue
        assert (st[i], fwd[i], rev[i]) == (0, len(wf), len(wr)), (i, g[:40], target.hex())
    return fwd, rev, st


def test_design_primers_at_exact_targets(gpu, oracle, melting_temp):
    """For m = 15 and a few other m per gene, each way: targets at the oracle Tm of seq[:m] or RC(seq[len-m:]) and
    at its two neighbours; a target just above a gene's highest forward Tm runs it out (PANIC)."""
    rng = np.random.default_rng(54)
    genes = design_genes()
    moved = 0
    for g in genes:
        s = g.decode("latin-1").upper()
        n = len(s)
        tf = {m: melting_temp(s[:m]) for m in range(15, n + 1)}
        tr = {m: melting_temp(oracle.reverse_complement(s[n - m:]).decode("latin-1")) for m in range(15, n + 1)}
        for m in sorted({15, *rng.integers(15, n + 1, 2).tolist()}):
            for t in (tf[m], tr[m]):
                at, above, _ = (check_design([g], x, melting_temp) for x in neighbours(t))
                moved += any((a != b).any() for a, b in zip(at, above))
        assert check_design([g], math.nextafter(max(tf.values()), math.inf), melting_temp)[2][0] == _lib.PG_ITEM_PANIC
    assert moved > 1000  # one ulp above a candidate's Tm moves the answer


@pytest.mark.parametrize("target", [math.inf, -math.inf, math.nan, -273.15])
def test_design_primers_special_targets(gpu, melting_temp, target):
    """+inf runs every gene out; -inf and NaN stop at 15 nt (nothing is < NaN); -273.15 is passed only by N runs."""
    fwd, rev, st = check_design(design_genes(), target, melting_temp)
    if target == math.inf:
        assert (st == _lib.PG_ITEM_PANIC).all()
    elif target != -273.15:
        assert (st == 0).all() and (fwd == 15).all() and (rev == 15).all()
    else:
        assert (st == _lib.PG_ITEM_PANIC).sum() == 1 and (fwd > 15).sum() == 1  # N * 15 runs out; N * 40 + ... passes 40 nt


def test_design_primers_with_overhangs_at_an_exact_target(gpu, melting_temp):
    """example_test.go:46's reaction, at the Tm of its own forward primer and one ulp above it."""
    t = melting_temp("AATAATTACACCGAGATAACACATCATGG")
    got = []
    for target in (t, math.nextafter(t, math.inf)):
        got.append(pcr.DesignPrimersWithOverhangs(GENE, "TTATAGGTCTCATACT", "ATGAAGAGACCATATA", target))
        assert got[-1] == design_primers(melting_temp, GENE, target, "TTATAGGTCTCATACT", "ATGAAGAGACCATATA")
    assert got[0][0] == "TTATAGGTCTCATACTAATAATTACACCGAGATAACACATCATGG" and got[1][0] != got[0][0]


# ---- the minimal primer of SimulateSimple --------------------------------------------------------------------
def test_minimal_primer_at_exact_targets(gpu, melting_temp):
    """Targets at the oracle Tm of every suffix of >= 7 nt and at its two neighbours."""
    rng = np.random.default_rng(55)
    prims = [bytes(rng.choice(list(b"ACGTacgtN"), int(rng.integers(7, 61))).tolist()) for _ in range(60)]
    prims += [b"GCGCGCG", b"ACGTACG", b"N" * 9, b"G" * 15 + b"C" * 15]
    moved = 0
    for p in prims:
        u = p.upper()
        for k in range(7, len(u) + 1):
            t = melting_temp(u[len(u) - k:])
            lengths = []
            for target in neighbours(t):
                ml, st = pcr.minimal_primer_lengths([p], target)
                want = P.minimal_length(u, target)
                assert (st[0], ml[0]) == (0, want), (p, k, target.hex())
                lengths.append(want)
            moved += lengths[0] != lengths[1]
    assert moved > 500


def test_simulate_at_an_exact_target(gpu, melting_temp):
    """A reaction whose fragments change when the target moves one ulp: at t = Tm(fwd[-k:]) the minimal forward
    primer is fwd[-(k-1):], which also binds a decoy site; one ulp above t it is longer and binds only the true site."""
    rng = np.random.default_rng(56)
    acgt = lambda n: bytes(rng.choice(list(b"ACGT"), size=n).astype(np.uint8))
    fwd, rev_site = acgt(30), acgt(30)
    tms = {k: melting_temp(fwd[30 - k:]) for k in range(7, 31)}
    k = next(k for k in range(14, 25) if tms[k] > max(tms[j] for j in range(7, k)))  # the loop stops at k, not before
    t, up = tms[k], math.nextafter(tms[k], math.inf)
    short, long_ = P.minimal_length(fwd, t), P.minimal_length(fwd, up)
    assert short == k - 1 < k <= long_ < 30
    decoy = (b"A" if fwd[30 - k] != ord("A") else b"C") + fwd[30 - short:]
    tpl = acgt(60) + fwd + acgt(120) + decoy + acgt(120) + rev_site + acgt(60)
    prims = [fwd, P.revcomp(rev_site)]
    simple = []
    for target in (t, up):
        got = pcr.SimulateSimple([tpl], target, False, list(prims))
        assert got == P.simulate_simple([tpl], target, False, prims)
        simple.append(got)
        fr, err = pcr.Simulate([tpl], target, False, list(prims))
        assert (fr, str(err) if err else None) == P.simulate([tpl], target, False, prims)
        assert fr == got
    assert simple[0] and simple[1] and simple[0] != simple[1]
