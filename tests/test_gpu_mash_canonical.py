"""Canonical k-mers (PG_KMER_CANONICAL) of the grouped sketch, the sketcher and the screen on the device, against the
canonical oracle (canonical_oracle.py): every walk k at its own span and chunk boundaries and generic k, strand
symmetry, flags = 0 against the old entry points, the sketcher's split rules, the screen's results, winners and
samples, and what the mode is for: reads from both strands of a genome screened against its sketch."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import canonical_oracle
import oracle_ffi
import screen_oracle
import sketch_groups_oracle
import test_gpu_walk_k as walk
from poly_b200 import _lib, mash

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
THREADS = len(os.sched_getaffinity(0))
ACGT = np.frombuffer(b"ACGT", np.uint8)
LETTERS = np.frombuffer(b"ABCDGHKMNRSTVWYabcdghkmnrstvwy", np.uint8)
COMP = canonical_oracle.complement_table()
GENERIC_KS = (1, 5, 33)


def revcomp(a: np.ndarray) -> np.ndarray:
    return COMP[np.asarray(a, np.uint8)[::-1]]


def flip_records(bases, off, which):
    """bases with record i replaced by its reverse complement for every i in which"""
    out = bases.copy()
    for i in which:
        a, b = int(off[i]), int(off[i + 1])
        out[a:b] = revcomp(bases[a:b])
    return out


def canon_layout(k, rng):
    """walk.group_layout (group ends on k's span W and chunk 256 W, each -1, 0, +1, empty groups) with some records
    turned into IUPAC letters, lower case or arbitrary bytes, and closing groups of records of length k and k - 1,
    a palindrome and an empty record."""
    bases, off, goff = walk.group_layout(k, rng)
    for i in range(0, len(off) - 1, 7):
        a, b = int(off[i]), int(off[i + 1])
        kind = (i // 7) % 3
        bases[a:b] = (LETTERS[rng.integers(0, len(LETTERS), b - a)] if kind == 0 else rng.integers(0, 256, b - a, dtype=np.uint8)
                      if kind == 1 else bases[a:b] | np.uint8(0x20))  # lower case
    tail = [ACGT[rng.integers(0, 4, k)], ACGT[rng.integers(0, 4, k - 1)] if k > 1 else np.zeros(0, np.uint8),
            np.frombuffer(b"ACGT" * (k // 2 + 2), np.uint8), np.zeros(0, np.uint8), ACGT[rng.integers(0, 4, 3 * k)]]
    n0 = len(off) - 1
    recs_off = list(off.astype(np.int64))
    for t in tail:
        recs_off.append(recs_off[-1] + len(t))
    bases = np.concatenate([bases] + tail)
    goff = np.concatenate([goff, [n0 + 1, n0 + 2, n0 + 2, n0 + 4, n0 + 5]]).astype(np.uint64)
    return bases, np.array(recs_off, np.uint64), goff


def assert_rows(got, want, *ctx):
    assert got[1].tobytes() == want[1].tobytes(), ctx
    assert got[0].tobytes() == want[0].tobytes(), ctx


def oracle_groups(bases, off, goff, k, s, m):
    return canonical_oracle.sketch_groups(bases, off, goff, k, s, m, THREADS)


# ---- grouped sketches -----------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", walk.WALK_KS + GENERIC_KS)
def test_groups_every_k(gpu, k):
    """groups_walk_kernel<K, true> at every walk k, groups_generic_kernel<true> at generic k, against the oracle: one
    pass when s is above every group's windows (m = 1 and 2), and several at s = 16, m = 2."""
    rng = np.random.default_rng(900 + k)
    if k in walk.WALK_KS:
        bases, off, goff = canon_layout(k, rng)
    else:  # generic k: the grouped-sketch chunk is 256 bytes
        lens = [255, 256, 257, 1, k, max(k - 1, 0), 0, 511, 513, 40, 3000]
        bases, off = walk.ragged_of(lens, rng, arbitrary_every=4)
        goff = np.array([0, 2, 2, 5, 7, 7, 10, 11], np.uint64)
    wide = 2 * int(np.diff(off.astype(np.int64)).max()) + 2
    for s, m, one_pass in ((wide, 1, True), (wide, 2, True), (16, 2, False)):
        with walk.Launches() as la:
            got = mash.sketch_groups(bases, off, goff, k, s, m, canonical=True)
        want = oracle_groups(bases, off, goff, k, s, m)
        if one_pass:
            assert (la.count, la.last) == (walk.GS_SETUP_LAUNCHES + walk.GS_PASS_LAUNCHES, "groups_append_kernel"), (k, s, m)
            assert want[1].max() > 0
        assert_rows(got, want, k, s, m)


@pytest.mark.gpu
@pytest.mark.parametrize("k", (11, 16, 21, 31, 32, 5, 33))
def test_groups_strand_symmetry(gpu, k):
    """Reverse-complementing any subset of records (IUPAC letters of both cases) changes no row and no count."""
    rng = np.random.default_rng(50 + k)
    lens = rng.integers(0, 3000, 300)
    lens[:5] = (k - 1, k, k + 1, 0, 20000)
    bases, off = walk.ragged_of(lens, rng)
    bases[: int(off[100])] = LETTERS[rng.integers(0, len(LETTERS), int(off[100]))]
    goff = np.array([0, 3, 50, 50, 120, 299, 300], np.uint64)
    flipped = flip_records(bases, off, np.nonzero(rng.random(300) < 0.5)[0])
    for s, m in ((1000, 1), (200, 2)):
        a = mash.sketch_groups(bases, off, goff, k, s, m, canonical=True)
        b = mash.sketch_groups(flipped, off, goff, k, s, m, canonical=True)
        assert_rows(a, b, k, s, m)
        assert a[1].sum() > 0
    assert_rows(a, oracle_groups(bases, off, goff, k, 200, 2), k)


@pytest.mark.gpu
def test_flags_zero_is_the_old_call(gpu):
    """flags = 0 gives the old entry points' bytes: grouped sketch (host and _dev), sketcher, screen and samples."""
    import torch

    L = _lib.lib()
    rng = np.random.default_rng(3)
    bases, off = walk.ragged_of(rng.integers(0, 2000, 200), rng, arbitrary_every=9)
    goff = np.array([0, 10, 10, 90, 200], np.uint64)
    G, k, s, m, stride = 4, 21, 300, 2, 310
    outs = []
    for fn, args in ((L.pg_mash_sketch_groups, ()), (L.pg_mash_sketch_groups_flags, (0,))):
        o, c = np.full(G * stride, 7, np.uint32), np.zeros(G, np.uint32)
        _lib.check(fn(bases.ctypes.data, off.ctypes.data, 200, goff.ctypes.data, G, k, s, m, *args, o.ctypes.data, stride, c.ctypes.data))
        outs.append(o.tobytes() + c.tobytes())
    d_b, d_off, d_goff = (torch.from_numpy(x.view(np.int64) if x.dtype == np.uint64 else x).cuda() for x in (bases, off, goff))
    for fn, args in ((L.pg_mash_sketch_groups_dev, ()), (L.pg_mash_sketch_groups_flags_dev, (0,))):
        o, c = torch.full((G * stride,), 7, dtype=torch.int32, device="cuda"), torch.zeros(G, dtype=torch.int32, device="cuda")
        _lib.check(fn(d_b.data_ptr(), d_off.data_ptr(), 200, d_goff.data_ptr(), G, k, s, m, *args, o.data_ptr(), stride, c.data_ptr(),
                      torch.cuda.current_stream().cuda_stream))
        outs.append(o.cpu().numpy().tobytes() + c.cpu().numpy().tobytes())
    assert outs[0] == outs[1] == outs[2] == outs[3]

    rows = []
    for create in (lambda h: L.pg_mash_sketcher_create(G, k, s, m, 1000, C.byref(h)),
                   lambda h: L.pg_mash_sketcher_create_flags(G, k, s, m, 1000, 0, C.byref(h))):
        h = C.c_void_p()
        _lib.check(create(h))
        _lib.check(L.pg_mash_sketcher_add(h, bases.ctypes.data, off.ctypes.data, 200, goff.ctypes.data, 0, G))
        o, c, cm, hd = np.zeros(G * s, np.uint32), np.zeros(G, np.uint32), np.zeros(G, np.uint8), np.zeros(G, np.uint64)
        _lib.check(L.pg_mash_sketcher_rows(h, 0, G, o.ctypes.data, s, c.ctypes.data, cm.ctypes.data, hd.ctypes.data))
        _lib.check(L.pg_mash_sketcher_free(h))
        rows.append(o.tobytes() + c.tobytes() + cm.tobytes() + hd.tobytes())
    assert rows[0] == rows[1]

    sk = np.ascontiguousarray(mash.sketch_groups(bases, off, goff, k, s, 1)[0])
    ids = (np.arange(200) % 3).astype(np.uint32)
    res = []
    for create, S in ((lambda h: L.pg_mash_screen_create(sk.ctypes.data, G, s, k, C.byref(h)), 1),
                      (lambda h: L.pg_mash_screen_create_flags(sk.ctypes.data, G, s, k, 1, 0, C.byref(h)), 1),
                      (lambda h: L.pg_mash_screen_create_samples(sk.ctypes.data, G, s, k, 3, C.byref(h)), 3),
                      (lambda h: L.pg_mash_screen_create_flags(sk.ctypes.data, G, s, k, 3, 0, C.byref(h)), 3)):
        h = C.c_void_p()
        _lib.check(create(h))
        if S == 1:
            _lib.check(L.pg_mash_screen_add(h, bases.ctypes.data, off.ctypes.data, 200))
        else:
            _lib.check(L.pg_mash_screen_add_samples(h, bases.ctypes.data, off.ctypes.data, ids.ctypes.data, 200))
        out = b""
        for fn in (L.pg_mash_screen_results_samples, L.pg_mash_screen_winners_samples):
            sh, co, mu = np.zeros(S * G, np.uint32), np.zeros(S * G, np.float64), np.zeros(S * G, np.uint64)
            _lib.check(fn(h, 0, S, sh.ctypes.data, co.ctypes.data, mu.ctypes.data))
            out += sh.tobytes() + co.tobytes() + mu.tobytes()
        _lib.check(L.pg_mash_screen_free(h))
        res.append(out)
    assert res[0] == res[1] and res[2] == res[3]
    assert np.frombuffer(res[0][:G * 4], np.uint32).sum() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("k", (21, 33))
def test_dev_equals_host_and_row_stride(gpu, k):
    import torch

    rng = np.random.default_rng(k)
    bases, off = walk.ragged_of(rng.integers(0, 1500, 120), rng)
    goff = np.array([0, 40, 40, 120], np.uint64)
    G, s, stride = 3, 150, 170
    want = mash.sketch_groups(bases, off, goff, k, s, 2, canonical=True)
    got = mash.sketch_groups(torch.from_numpy(bases).cuda(), torch.from_numpy(off.view(np.int64)).cuda(),
                             torch.from_numpy(goff.view(np.int64)).cuda(), k, s, 2, canonical=True)
    assert got[0].cpu().numpy().view(np.uint32).tobytes() == want[0].tobytes()
    assert got[1].cpu().numpy().view(np.uint32).tobytes() == want[1].tobytes()
    o = torch.full((G * stride,), -1, dtype=torch.int32, device="cuda")
    c = torch.zeros(G, dtype=torch.int32, device="cuda")
    d = [torch.from_numpy(x).cuda() for x in (bases, off.view(np.int64), goff.view(np.int64))]
    _lib.check(_lib.lib().pg_mash_sketch_groups_flags_dev(d[0].data_ptr(), d[1].data_ptr(), 120, d[2].data_ptr(), G, k, s, 2, _lib.PG_KMER_CANONICAL,
                                                          o.data_ptr(), stride, c.data_ptr(), torch.cuda.current_stream().cuda_stream))
    o = o.cpu().numpy().view(np.uint32).reshape(G, stride)
    assert o[:, :s].tobytes() == want[0].tobytes() and not o[:, s:].any()


# ---- the sketcher -----------------------------------------------------------------------------------------------------
def split_adds(rng, n_records, goff):
    """random record cuts, including empty adds and cuts inside groups"""
    cuts = np.unique(np.concatenate([[0, n_records], rng.integers(0, n_records + 1, 6)]))
    for a, b in zip(cuts[:-1], cuts[1:]):
        yield int(a), int(b)


def add_range(sk, bases, off, goff, a, b):
    """records [a, b) of the batch, with the groups they fall in"""
    g0 = int(np.searchsorted(goff, a, "right")) - 1
    g1 = int(np.searchsorted(goff, b, "left"))
    gl = np.clip(goff[g0:g1 + 1].astype(np.int64), a, b) - a
    sub = off[a:b + 1] - off[a]
    sk.add(bases[int(off[a]):int(off[b])], sub, gl.astype(np.uint64), first_group=g0)


def with_reverse_complements(bases, off):
    """each record followed by its reverse complement: with canonical k-mers every window then counts twice"""
    recs = [bases[int(off[i]):int(off[i + 1])] for i in range(len(off) - 1)]
    recs = [r for x in recs for r in (x, revcomp(x))]
    o = np.concatenate([[0], np.cumsum([len(r) for r in recs])]).astype(np.uint64)
    return np.concatenate(recs), o


@pytest.mark.gpu
@pytest.mark.parametrize("k,s,m,B", [(21, 200, 1, None), (21, 200, 2, None), (16, 100, 2, 150), (33, 100, 2, None), (32, 300, 2, 400)])
def test_sketcher_against_one_shot_and_oracle(gpu, k, s, m, B):
    """m = 2 qualifies a value through a record and its reverse complement, which count together."""
    rng = np.random.default_rng(k * 7 + m)
    bases, off = with_reverse_complements(*walk.ragged_of(rng.integers(0, 600, 200), rng))
    goff = np.array([0, 80, 80, 200, 390, 400], np.uint64)
    G = len(goff) - 1
    once = mash.sketch_groups(bases, off, goff, k, s, m, canonical=True)
    sk = mash.Sketcher(G, k, s, m, B, canonical=True)
    ref = canonical_oracle.Sketcher(G, k, s, m, B)
    assert sk.canonical
    for a, b in split_adds(rng, 400, goff):
        add_range(sk, bases, off, goff, a, b)
        g0 = int(np.searchsorted(goff, a, "right")) - 1
        g1 = int(np.searchsorted(goff, b, "left"))
        gl = np.clip(goff[g0:g1 + 1].astype(np.int64), a, b) - a
        ref.add(bases[int(off[a]):int(off[b])], off[a:b + 1] - off[a], gl, first_group=g0, nthreads=THREADS)
        rows, count, complete, held = sk.rows()
        w = ref.rows()
        assert rows.tobytes() == w[0].tobytes() and count.tobytes() == w[1].tobytes()
        assert complete.tobytes() == w[2].tobytes() and held.tobytes() == w[3].tobytes()
    for g in range(G):  # every record added: each row is a prefix of the one-shot row
        assert rows[g, :count[g]].tobytes() == once[0][g, :count[g]].tobytes()
    if m == 1:
        assert complete.all()
    full = complete & (np.diff(goff.astype(np.int64)) > 0)
    assert (count[full] == s).all()  # every group's windows qualify in pairs, far more than s of them
    for g in np.nonzero(complete)[0]:
        assert rows[g].tobytes() == once[0][g].tobytes() and count[g] == once[1][g]
    sk.close()


# ---- the screen --------------------------------------------------------------------------------------------------------
def assert_same(got, want, *ctx):
    for g, w in zip(got, want):
        assert np.asarray(g).tobytes() == np.asarray(w).tobytes(), ctx


@pytest.mark.gpu
@pytest.mark.parametrize("k", walk.WALK_KS + GENERIC_KS)
def test_screen_every_k(gpu, k):
    """screen_walk_kernel<K, *, true> at every walk k (read ends on W and 256 W) and the generic kernel: results and
    winners against the oracle, split invariant, and reverse-complemented reads count the same."""
    rng = np.random.default_rng(300 + k)
    W = walk.span(k) if k in walk.WALK_KS else 256
    CH = 256 * W
    lens = [W - 1, W, W + 1, CH - 1, CH, CH + 1, k, max(k - 1, 0), 0, 2 * CH + 3] + list(rng.integers(0, 400, 60))
    bases, off = walk.ragged_of(lens, rng, arbitrary_every=11)
    n = len(lens)
    genomes = [bases[int(off[i]):int(off[i + 1])] for i in (3, 4, 9)]  # three of the pool's reads
    go = np.concatenate([[0], np.cumsum([len(g) for g in genomes])]).astype(np.uint64)
    sk = mash.sketch_groups(np.concatenate(genomes), go, np.arange(4, dtype=np.uint64), k, 400, 1, canonical=True)[0]
    sk = np.vstack([sk, rng.integers(0, 1 << 32, (2, 400), dtype=np.uint64).astype(np.uint32)])
    want_r = canonical_oracle.mash_screen(sk, (bases, off), k, THREADS)
    want_w = canonical_oracle.mash_screen_winners(sk, (bases, off), k, THREADS)
    flipped = flip_records(bases, off, range(0, n, 2))
    for pool, cuts in (((bases, off), (0, n)), ((bases, off), (0, 3, 3, 10, 41, n)), ((flipped, off), (0, 25, n))):
        sc = mash.Screen(sk, k, canonical=True)
        for a, b in zip(cuts[:-1], cuts[1:]):
            sc.add((pool[0][int(off[a]):int(off[b])], off[a:b + 1] - off[a]))
        assert_same(sc.results(), want_r, k, cuts)
        assert_same(sc.winners(), want_w, k, cuts)
        sc.close()
    assert want_r[0][:3].min() > 0


@pytest.mark.gpu
@pytest.mark.parametrize("k", (21, 13, 33))
def test_screen_samples(gpu, k):
    rng = np.random.default_rng(k + 1)
    bases, off = walk.ragged_of(rng.integers(0, 800, 300), rng)
    ids = rng.integers(0, 4, 300).astype(np.uint32)
    sk = mash.sketch_groups(bases, off, np.array([0, 100, 200, 300], np.uint64), k, 500, 1, canonical=True)[0]
    sc = mash.Screen(sk, k, samples=4, canonical=True)
    flipped = flip_records(bases, off, np.nonzero(ids % 2)[0])
    sc.add((flipped[: int(off[150])], off[:151]), ids[:150])
    sc.add((flipped[int(off[150]):], off[150:] - off[150]), ids[150:])
    res, win = sc.results_samples(), sc.winners_samples()
    for q in range(4):
        reads = [bases[int(off[i]):int(off[i + 1])] for i in np.nonzero(ids == q)[0]]
        assert_same([x[q] for x in res], canonical_oracle.mash_screen(sk, mash.flatten(reads), k, THREADS), k, q)
        assert_same([x[q] for x in win], canonical_oracle.mash_screen_winners(sk, mash.flatten(reads), k, THREADS), k, q)
    sc.close()


# ---- what the mode is for ----------------------------------------------------------------------------------------------
def sample_reads(rng, genome, n, L):
    """n error-free reads of length L from random positions, each from a random strand"""
    starts = rng.integers(0, len(genome) - L + 1, n)
    reads = genome[starts[:, None] + np.arange(L)]
    rev = rng.random(n) < 0.5
    reads[rev] = COMP[reads[rev][:, ::-1]]
    return reads


@pytest.mark.gpu
def test_both_strand_pool_against_genomes(gpu):
    """20 of 200 genomes (20 kbp each) read at 10x from both strands, 150 bp reads: against canonical sketches every
    source is contained (>= 0.99) at its k-mer coverage c (L - k + 1) / L (within 20 %); forward sketches and a forward
    screen see about half that multiplicity."""
    rng = np.random.default_rng(2026)
    k, s, G, glen, L, cov = 21, 1000, 200, 20000, 150, 10
    genomes = ACGT[rng.integers(0, 4, (G, glen))]
    goff = np.arange(G + 1, dtype=np.uint64)
    off = goff * np.uint64(glen)
    can = mash.sketch_groups(genomes.reshape(-1), off, goff, k, s, 1, canonical=True)[0]
    fwd = mash.sketch_groups(genomes.reshape(-1), off, goff, k, s, 1)[0]
    src = rng.choice(G, 20, replace=False)
    n = cov * glen // L
    reads = np.concatenate([sample_reads(rng, genomes[g], n, L) for g in src])
    roff = np.arange(len(reads) + 1, dtype=np.uint64) * np.uint64(L)
    pool = (reads.reshape(-1), roff)
    sc = mash.Screen(can, k, canonical=True)
    sc.add(pool)
    shared, cont, mult = sc.results()
    sf = mash.Screen(fwd, k)
    sf.add(pool)
    _, fcont, fmult = sf.results()
    kcov = cov * (L - k + 1) / L
    others = np.setdiff1d(np.arange(G), src)
    assert cont[src].min() >= 0.99, cont[src]
    assert np.abs(mult[src] / kcov - 1).max() <= 0.2, mult[src]
    assert cont[others].max() < 0.01
    assert np.abs(fmult[src] / (kcov / 2) - 1).max() <= 0.35, fmult[src]  # half the reads are on the other strand
    assert fcont[src].min() >= 0.9
    # the same against the oracle, for a few sources
    sub = np.concatenate([np.arange(i * n, (i + 1) * n) for i in range(2)])
    sub_pool = (reads[sub].reshape(-1), np.arange(len(sub) + 1, dtype=np.uint64) * np.uint64(L))
    sc.reset()
    sc.add(sub_pool)
    assert_same(sc.results(), canonical_oracle.mash_screen(can, sub_pool, k, THREADS))
    sc.close()
    sf.close()


@pytest.mark.gpu
def test_assembly_orientation(gpu):
    """An assembly and the same assembly with every contig reverse-complemented: equal canonical rows, and forward
    rows that share almost nothing."""
    rng = np.random.default_rng(77)
    k, s = 21, 2000
    lens = rng.integers(2000, 60000, 100)
    bases, off = walk.ragged_of(lens, rng)
    flipped = flip_records(bases, off, range(100))
    both = np.concatenate([bases, flipped])
    off2 = np.concatenate([off, off[1:] + off[-1]])
    goff = np.array([0, 100, 200], np.uint64)
    can = mash.sketch_groups(both, off2, goff, k, s, 1, canonical=True)
    fwd = mash.sketch_groups(both, off2, goff, k, s, 1)
    assert can[0][0].tobytes() == can[0][1].tobytes() and can[1].tolist() == [s, s]
    assert len(np.intersect1d(fwd[0][0], fwd[0][1])) < s // 50
    assert_rows(can, oracle_groups(both, off2, goff, k, s, 1))


# ---- the C++ mirror ----------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_cpp_mirror_agrees_with_the_oracle(gpu):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "canonical_tests"])
    rng = np.random.default_rng(21)
    k, s, m = 21, 300, 1
    groups = [[ACGT[rng.integers(0, 4, int(n))] for n in rng.integers(k, 2000, int(c))] for c in rng.integers(1, 12, 8)]
    with tempfile.TemporaryDirectory() as td:
        txt = os.path.join(td, "groups.txt")
        with open(txt, "wb") as f:
            for g, recs in enumerate(groups):
                f.write(b"".join(b"%d " % g + bytes(r) + b"\n" for r in recs))
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "canonical_tests"), txt, str(len(groups)), str(k), str(s), str(m)],
                             capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: canonical tests pass"
    bases, off, goff = sketch_groups_oracle.flatten_groups(groups)
    rows, count = oracle_groups(bases, off, goff, k, s, m)
    assert len(lines) == len(groups) + 2
    for g, line in enumerate(lines[:len(groups)]):
        vals = [int(x) for x in line.split()]
        assert vals[0] == count[g] and vals[1:] == [int(v) for v in rows[g, :count[g]]]
    assert lines[len(groups)] == "shared " + " ".join(str(int(c)) for c in count)
