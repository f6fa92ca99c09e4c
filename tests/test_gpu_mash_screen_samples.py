"""A screen of several samples on the GPU (pg_mash_screen_*_samples): each row of results_samples and winners_samples
against the CPU restatements (tests/screen_oracle.py, tests/screen_winners_oracle.py) applied to that sample's reads,
for walk and generic k; each row against a fresh one-sample screen; split adds across host and _dev with reset; the
single-sample calls on a screen of several samples; a table spanning two sample groups of the tally; the argument
rules; and the C++ mirror."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle_ffi
import screen_oracle
import screen_winners_oracle
from poly_b200 import _lib, mash, sketchfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
THREADS = len(os.sched_getaffinity(0))
S = 200
ACGT = np.frombuffer(b"ACGT", np.uint8)
SAMPLES = 7
EMPTY, EDGES, LONG = 4, 5, 6  # the sample with no reads, the one with only empty, k- and (k+1)-length reads, the 100 kbp one


def pool_reads(k, seed=0, n_short=700):
    """(reads, ids) over SAMPLES samples, interleaved at random: short reads of 20..300 bp drawn from two 100 kbp
    reads with a few substitutions in samples 0..3 and LONG, a repeat-rich read, no read in EMPTY, only empty, k- and
    (k+1)-length reads in EDGES, and one of the 100 kbp reads in LONG."""
    rng = np.random.default_rng(seed)
    long_reads = [ACGT[rng.integers(0, 4, 100_000)] for _ in range(2)]
    reads = [(long_reads[0], LONG), (np.tile(ACGT[rng.integers(0, 4, 7)], 300), 1)]
    for _ in range(3):
        reads += [(np.zeros(0, np.uint8), EDGES), (ACGT[rng.integers(0, 4, k)], EDGES), (ACGT[rng.integers(0, 4, k + 1)], EDGES)]
    for _ in range(n_short):
        src = long_reads[int(rng.integers(0, 2))]
        L = int(rng.integers(20, 301))
        a = int(rng.integers(0, len(src) - L))
        r = src[a:a + L].copy()
        r[rng.random(L) < 0.01] = ACGT[rng.integers(0, 4)]
        reads.append((r, int(rng.choice([0, 1, 2, 3, LONG]))))
    order = rng.permutation(len(reads))
    return [reads[i][0] for i in order], np.array([reads[i][1] for i in order], np.uint32), long_reads


def references(long_reads, reads, k, seed=0):
    """Select-regime sketches of the 100 kbp reads, fill-regime sketches of short reads (unsorted, zero tails),
    sketches of reads not in the pool, and random words."""
    rng = np.random.default_rng(seed + 1)
    shorts = [r for r in reads if 0 < len(r) < 150][:6]
    others = [ACGT[rng.integers(0, 4, 5000)] for _ in range(2)]
    bases, off = mash.flatten(long_reads + shorts + others)
    rc, sk = oracle_ffi.sketch_batch(bases, off, k, S, variant=1, nthreads=THREADS)
    assert rc == 0
    rand = rng.integers(0, 1 << 32, (3, S), dtype=np.uint64).astype(np.uint32)
    return np.ascontiguousarray(np.concatenate([sk, rand]), np.uint32)


def subset(reads, ids, q):
    return [r for r, i in zip(reads, ids) if i == q]


def assert_same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.tobytes() == w.tobytes(), (g, w)


def row(table, q):
    return tuple(x[q] for x in table)


def one_sample(sk, k, reads, winners=False):
    """What a fresh single-sample screen answers after one add of `reads`."""
    with mash.Screen(sk, k) as sc:
        sc.add(reads)
        return sc.winners() if winners else sc.results()


@pytest.mark.parametrize("k", [21, 31, 32, 11, 12, 33, 0])
def test_each_row_equals_the_oracle_on_its_reads(gpu, k):
    reads, ids, long_reads = pool_reads(k)
    sk = references(long_reads, reads, k)
    with mash.Screen(sk, k, samples=SAMPLES) as sc:
        sc.add(reads, sample=ids)
        table = sc.results_samples()
    assert table[0].shape == (SAMPLES, len(sk))
    for q in range(SAMPLES):
        want = screen_oracle.mash_screen(sk, mash.flatten(subset(reads, ids, q)), k, nthreads=THREADS)
        assert_same(row(table, q), want)
    assert all((x[EMPTY] == 0).all() for x in table)
    if k > 0:  # the 100 kbp read's own sketch: every hash is in sample LONG
        assert table[0][LONG, 0] == S and (table[0][:LONG, 0] < S).all()


def strain_pools(seed=0):
    """4 species x 5 strains at 0.2 .. 5 % substitutions (row species * 5 + strain), and (reads, ids) of 3 samples:
    sample 0 drawn from strain 2 of species 0, sample 1 from strain 4 of species 0, sample 2 from strain 0 of
    species 1 and random reads; about 10x of each source with 1 % substitutions, interleaved."""
    rng = np.random.default_rng(seed)
    glen, read = 20_000, 150

    def mutate(seq, rate):
        out = seq.copy()
        hit = rng.random(len(seq)) < rate
        out[hit] = ACGT[(np.searchsorted(ACGT, out[hit]) + rng.integers(1, 4, int(hit.sum()))) % 4]
        return out

    genomes = []
    for _ in range(4):
        root = ACGT[rng.integers(0, 4, glen)]
        genomes += [mutate(root, r) for r in np.linspace(0.002, 0.05, 5)]
    reads = []
    for q, src in enumerate((2, 4, 5)):
        for a in rng.integers(0, glen - read, 10 * glen // read):
            reads.append((mutate(genomes[src][a:a + read], 0.01), q))
    reads += [(ACGT[rng.integers(0, 4, read)], 2) for _ in range(300)]
    order = rng.permutation(len(reads))
    return genomes, [reads[i][0] for i in order], np.array([reads[i][1] for i in order], np.uint32)


@pytest.mark.parametrize("k", [21, 33])
def test_winners_rows_equal_the_restatement_and_samples_vote_alone(gpu, k):
    genomes, reads, ids = strain_pools()
    bases, off = mash.flatten(genomes)
    rc, sk = oracle_ffi.sketch_batch(bases, off, k, S, variant=1, nthreads=THREADS)
    assert rc == 0
    with mash.Screen(sk, k, samples=3) as sc:
        sc.add(reads, sample=ids)
        table = sc.winners_samples()
    for q in range(3):
        want = screen_winners_oracle.mash_screen_winners(sk, mash.flatten(subset(reads, ids, q)), k, nthreads=THREADS)
        assert_same(row(table, q), want)
    # samples 0 and 1 come from two strains of species 0: each elects its own strain
    assert int(np.argmax(table[0][0, :5])) == 2 and int(np.argmax(table[0][1, :5])) == 4


@pytest.mark.parametrize("k", [21, 33])
def test_each_row_equals_a_fresh_single_sample_screen(gpu, k):
    reads, ids, long_reads = pool_reads(k, seed=2, n_short=400)
    sk = references(long_reads, reads, k, seed=2)
    with mash.Screen(sk, k, samples=SAMPLES) as sc:
        sc.add(reads, sample=ids)
        res, win = sc.results_samples(), sc.winners_samples()
    for q in range(SAMPLES):
        mine = subset(reads, ids, q)
        assert_same(row(res, q), one_sample(sk, k, mine))
        assert_same(row(win, q), one_sample(sk, k, mine, winners=True))


def test_random_splits_equal_one_add(gpu):
    import torch

    k = 21
    reads, ids, long_reads = pool_reads(k, seed=5, n_short=500)
    sk = references(long_reads, reads, k, seed=5)
    rng = np.random.default_rng(6)
    stream = torch.cuda.Stream()
    with mash.Screen(sk, k, samples=SAMPLES) as sc:
        sc.add(reads, sample=ids)
        want = sc.results_samples(), sc.winners_samples()
        for trial in range(3):
            sc.reset()
            assert all((x == 0).all() for x in sc.results_samples())
            cuts = np.sort(rng.integers(0, len(reads) + 1, 6))
            cuts = np.concatenate([[0], cuts, [cuts[-1]], [min(cuts[-1] + 1, len(reads))], [len(reads)]])  # an empty and a one-read add
            for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
                if (i + trial) % 2:
                    sc.add(reads[a:b], sample=ids[a:b])
                else:
                    bases, off = mash.flatten(reads[a:b])
                    with torch.cuda.stream(stream):
                        sc.add_dev(torch.from_numpy(bases).cuda(), torch.from_numpy(off.astype(np.int64)).cuda(), stream=stream,
                                   d_samples=torch.from_numpy(ids[a:b].view(np.int32)).cuda())
            assert_same(sc.results_samples(), want[0])
            assert_same(sc.winners_samples(), want[1])


def test_single_sample_calls_on_a_screen_of_several_samples(gpu):
    import torch

    k = 21
    reads, ids, long_reads = pool_reads(k, seed=7, n_short=300)
    sk = references(long_reads, reads, k, seed=7)
    zeros = np.zeros(len(reads), np.uint32)
    with mash.Screen(sk, k, samples=4) as a, mash.Screen(sk, k, samples=4) as b:
        a.add(reads)
        b.add(reads, sample=zeros)
        assert_same(a.results_samples(), b.results_samples())
        assert_same(a.winners_samples(), b.winners_samples())
        assert_same(a.results(), row(a.results_samples(), 0))
        assert_same(a.winners(), row(a.winners_samples(), 0))
        assert all((x[1:] == 0).all() for x in a.results_samples())
        bases, off = mash.flatten(reads)
        a.add_dev(torch.from_numpy(bases).cuda(), torch.from_numpy(off.astype(np.int64)).cuda())  # add_dev: sample 0 too
        a.add(reads, sample=3)  # one int sample for every read
        twice = one_sample(sk, k, reads + reads)
        assert_same(a.results(), twice)
        assert_same(a.results(3), one_sample(sk, k, reads))
        assert np.array_equal(a.identity(3), a.results(3)[1] ** (1.0 / k))
    # an S = 1 screen made by create_samples answers with the bytes of pg_mash_screen_create
    L = _lib.lib()
    bases, off = mash.flatten(reads)
    n = len(sk)
    outs = []
    for create in (lambda h: L.pg_mash_screen_create(sk.ctypes.data, n, S, k, C.byref(h)),
                   lambda h: L.pg_mash_screen_create_samples(sk.ctypes.data, n, S, k, 1, C.byref(h))):
        h = C.c_void_p()
        _lib.check(create(h))
        try:
            _lib.check(L.pg_mash_screen_add(h, bases.ctypes.data, off.ctypes.data, len(reads)))
            got = []
            for fn in (L.pg_mash_screen_results, L.pg_mash_screen_winners):
                x = np.zeros(n, np.uint32), np.zeros(n, np.float64), np.zeros(n, np.uint64)
                _lib.check(fn(h, *(y.ctypes.data for y in x)))
                got.append(x)
            outs.append(got)
        finally:
            _lib.check(L.pg_mash_screen_free(h))
    for x, y in zip(*outs):
        assert_same(x, y)


def test_a_table_spanning_two_sample_groups(gpu):
    """n s = 2^26 words and 8 samples: at 2^28 slots per group, one results_samples call tallies two groups of 4."""
    slots, samples = 1 << 28, 8
    n, s, k = 1 << 16, 1 << 10, 21
    assert (slots // (n * s)) * 2 == samples
    rng = np.random.default_rng(11)
    genomes = [ACGT[rng.integers(0, 4, 20_000)] for _ in range(samples)]
    reads, ids = [], []
    for q, g in enumerate(genomes):  # sample q: 300 reads of genome q and 50 of genome (q + 1) % samples
        for src, m in ((g, 300), (genomes[(q + 1) % samples], 50)):
            for a in rng.integers(0, len(src) - 150, m):
                reads.append(src[a:a + 150])
                ids.append(q)
    order = rng.permutation(len(reads))
    reads, ids = [reads[i] for i in order], np.array([ids[i] for i in order], np.uint32)
    hashes = screen_oracle.pool_hashes(*mash.flatten(reads), k, THREADS)
    sk = rng.integers(0, 1 << 32, (n, s), dtype=np.uint64).astype(np.uint32)
    sk[:, : s // 2] = rng.choice(hashes, (n, s // 2))  # half of every row from the pool, with repeats
    with mash.Screen(sk, k, samples=samples) as sc:
        sc.add(reads, sample=ids)
        res, win = sc.results_samples(), sc.winners_samples()
        sub_res, sub_win = sc.results_samples(3, 4), sc.winners_samples(3, 4)
    for q in range(samples):
        mine = subset(reads, ids, q)
        assert_same(row(res, q), one_sample(sk, k, mine))
        assert_same(row(win, q), one_sample(sk, k, mine, winners=True))
    assert_same(sub_res, tuple(x[3:7] for x in res))
    assert_same(sub_win, tuple(x[3:7] for x in win))
    assert (res[0] > 0).all()


def test_argument_rules(gpu):
    import torch

    k = 21
    reads, ids, long_reads = pool_reads(k, seed=9, n_short=300)
    sk = references(long_reads, reads, k, seed=9)
    L = _lib.lib()
    bases, off = mash.flatten(reads)
    n = len(sk)
    with mash.Screen(sk, k, samples=SAMPLES) as sc:
        sc.add(reads, sample=ids)
        before = sc.results_samples()
        bad = ids.copy()
        bad[len(bad) // 2] = SAMPLES
        assert L.pg_mash_screen_add_samples(sc._h, bases.ctypes.data, off.ctypes.data, bad.ctypes.data, len(reads)) == _lib.PG_ERR_ARG
        assert L.pg_mash_screen_add_samples(sc._h, bases.ctypes.data, off.ctypes.data, None, len(reads)) == _lib.PG_ERR_ARG
        assert L.pg_mash_screen_add_samples_dev(sc._h, bases.ctypes.data, off.ctypes.data, None, len(reads), None) == _lib.PG_ERR_ARG
        assert L.pg_mash_screen_add_samples(sc._h, None, None, None, 0) == _lib.PG_OK
        with pytest.raises(_lib.PolyError):
            sc.add(reads, sample=bad)
        with pytest.raises(_lib.PolyError):
            sc.add(reads, sample=SAMPLES)
        with pytest.raises(ValueError):
            sc.add(reads, sample=ids[:-1])
        assert_same(sc.results_samples(), before)
        out = np.zeros(n * SAMPLES, np.uint32)
        for fn in (L.pg_mash_screen_results_samples, L.pg_mash_screen_winners_samples):
            assert fn(sc._h, 0, SAMPLES + 1, out.ctypes.data, None, None) == _lib.PG_ERR_ARG
            assert fn(sc._h, SAMPLES, 1, out.ctypes.data, None, None) == _lib.PG_ERR_ARG
            assert fn(sc._h, 0xFFFFFFFF, 2, out.ctypes.data, None, None) == _lib.PG_ERR_ARG  # no 32-bit wrap
            assert fn(sc._h, SAMPLES, 0, out.ctypes.data, None, None) == _lib.PG_OK
            assert fn(sc._h, 0, SAMPLES, None, None, None) == _lib.PG_OK
            for mask in ((1, 0, 0), (0, 1, 0), (0, 0, 1)):  # one output at a time
                xs = np.zeros((SAMPLES, n), np.uint32), np.zeros((SAMPLES, n), np.float64), np.zeros((SAMPLES, n), np.uint64)
                _lib.check(fn(sc._h, 0, SAMPLES, *(x.ctypes.data if m else None for x, m in zip(xs, mask))))
                full = sc._table(fn, 0, SAMPLES)
                for x, f, m in zip(xs, full, mask):
                    if m:
                        assert x.tobytes() == f.tobytes()
        with pytest.raises(_lib.PolyError):
            sc.results(SAMPLES)
    # a _dev read whose id is not a sample counts nowhere: the table is that of the reads without it
    drop = np.zeros(len(reads), bool)
    drop[::7] = True
    dev_ids = ids.copy()
    dev_ids[drop] = np.array([SAMPLES, SAMPLES + 1, 0xFFFFFFFF], np.uint32)[np.arange(drop.sum()) % 3]
    kept = [r for r, d in zip(reads, drop) if not d]
    with mash.Screen(sk, k, samples=SAMPLES) as sc, mash.Screen(sk, k, samples=SAMPLES) as ref:
        sc.add_dev(torch.from_numpy(bases).cuda(), torch.from_numpy(off.astype(np.int64)).cuda(), d_samples=torch.from_numpy(dev_ids.view(np.int32)).cuda())
        ref.add(kept, sample=ids[~drop])
        assert_same(sc.results_samples(), ref.results_samples())
        assert_same(sc.winners_samples(), ref.winners_samples())
        want = ref.results_samples(), ref.winners_samples()
    # create_samples_dev + add_samples_dev + results / winners_samples_dev on a side stream equal the host calls
    stream = torch.cuda.Stream()
    d_sk = torch.from_numpy(sk.view(np.int32)).cuda()
    d_bases = torch.from_numpy(bases).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    d_ids = torch.from_numpy(ids.view(np.int32)).cuda()
    stream.wait_stream(torch.cuda.current_stream())
    h = C.c_void_p()
    with torch.cuda.stream(stream):
        _lib.check(L.pg_mash_screen_create_samples_dev(d_sk.data_ptr(), n, S, k, SAMPLES, stream.cuda_stream, C.byref(h)))
        try:
            _lib.check(L.pg_mash_screen_add_samples_dev(h, d_bases.data_ptr(), d_off.data_ptr(), d_ids.data_ptr(), len(reads), stream.cuda_stream))
            got = []
            for fn in (L.pg_mash_screen_results_samples_dev, L.pg_mash_screen_winners_samples_dev):
                d_sh = torch.empty((SAMPLES, n), dtype=torch.int32, device="cuda")
                d_c = torch.empty((SAMPLES, n), dtype=torch.float64, device="cuda")
                d_m = torch.empty((SAMPLES, n), dtype=torch.int64, device="cuda")
                _lib.check(fn(h, 0, SAMPLES, d_sh.data_ptr(), d_c.data_ptr(), d_m.data_ptr(), stream.cuda_stream))
                stream.synchronize()
                got.append((d_sh.cpu().numpy().view(np.uint32), d_c.cpu().numpy(), d_m.cpu().numpy().view(np.uint64)))
        finally:
            _lib.check(L.pg_mash_screen_free(h))
    with mash.Screen(sk, k, samples=SAMPLES) as sc:
        sc.add(reads, sample=ids)
        assert_same(got[0], sc.results_samples())
        assert_same(got[1], sc.winners_samples())
    for q in range(SAMPLES):  # the dropped reads' table is, row by row, the table of the reads kept
        assert_same(row(want[0], q), one_sample(sk, k, subset(kept, ids[~drop], q)))


def test_cpp_mirror_agrees_with_the_oracle(gpu):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "screen_samples_tests"])
    k, samples = 21, 3
    reads, ids, long_reads = pool_reads(k, seed=10, n_short=300)
    reads = [r for r in reads if len(r)]  # one read per line: no empty line
    ids = np.random.default_rng(10).integers(0, samples, len(reads)).astype(np.uint32)
    sk = references(long_reads, reads, k, seed=10)
    with tempfile.TemporaryDirectory() as td:
        refs, txt = os.path.join(td, "refs.pgsketch"), os.path.join(td, "reads.txt")
        sketchfile.save(refs, sk, np.full(len(sk), S, np.uint32), k, S)
        with open(txt, "wb") as f:
            f.write(b"\n".join(b"%d " % q + r.tobytes() for r, q in zip(reads, ids)) + b"\n")
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "screen_samples_tests"), refs, txt, str(k), str(samples)], capture_output=True,
                             text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: screen samples tests pass"
    assert len(lines) == samples * len(sk) + 1
    wants = [screen_oracle.mash_screen(sk, mash.flatten(subset(reads, ids, q)), k, nthreads=THREADS) for q in range(samples)]
    for line in lines[:-1]:
        q, r, shared, bits, mult = line.split()
        q, r = int(q), int(r)
        want = wants[q]
        assert (int(shared), int(bits, 16), int(mult)) == (int(want[0][r]), int(want[1][r:r + 1].view(np.uint64)[0]), int(want[2][r]))
