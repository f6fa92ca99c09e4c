"""Mash Screen's winner-take-all on the GPU (pg_mash_screen_winners / _dev): shared, multiplicity and the bytes of
containment against the CPU restatement (tests/screen_winners_oracle.py) on strain families generated
here, for walk and generic k; duplicated and reordered rows; one value held by 100 000 references (a shared word and
shared zero tails); a poly-A pool past 2^32 windows; split adds, reset, host against _dev paths; results untouched
by winners; no references; references that share nothing; and the C++ mirror."""
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
SPECIES, STRAINS, GLEN, READ = 4, 5, 20_000, 150
SOURCES = ((0, 2), (1, 0))  # (species, strain) the pool is drawn from


def mutate(rng, seq, rate):
    out = seq.copy()
    hit = rng.random(len(seq)) < rate
    out[hit] = ACGT[(np.searchsorted(ACGT, out[hit]) + rng.integers(1, 4, int(hit.sum()))) % 4]  # a different base
    return out


def strain_families(seed=0):
    """SPECIES random genomes, each with STRAINS strains at 0.2 .. 5 % substitutions from it (row species * STRAINS
    + strain), and a pool of 150 bp reads: about 10x of each source strain with 1 % substitutions, and random reads."""
    rng = np.random.default_rng(seed)
    genomes = []
    for _ in range(SPECIES):
        root = ACGT[rng.integers(0, 4, GLEN)]
        genomes += [mutate(rng, root, r) for r in np.linspace(0.002, 0.05, STRAINS)]
    reads = []
    for sp, st in SOURCES:
        g = genomes[sp * STRAINS + st]
        for a in rng.integers(0, GLEN - READ, 10 * GLEN // READ):
            reads.append(mutate(rng, g[a:a + READ], 0.01))
    reads += [ACGT[rng.integers(0, 4, READ)] for _ in range(300)]
    order = rng.permutation(len(reads))
    return genomes, [reads[i] for i in order]


def sketches_of(genomes, k):
    bases, off = mash.flatten(genomes)
    rc, sk = oracle_ffi.sketch_batch(bases, off, k, S, variant=1, nthreads=THREADS)
    assert rc == 0
    return np.ascontiguousarray(sk, np.uint32)


def assert_same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.tobytes() == w.tobytes(), (g, w)


def winners_of(sk, reads, k):
    return screen_winners_oracle.mash_screen_winners(sk, mash.flatten(reads) if isinstance(reads, list) else reads, k, nthreads=THREADS)


def results_of(sk, reads, k):
    return screen_oracle.mash_screen(sk, mash.flatten(reads) if isinstance(reads, list) else reads, k, nthreads=THREADS)


@pytest.mark.parametrize("k", [21, 31, 32, 11, 33, 0])
def test_strain_families_against_the_restatement(gpu, k):
    genomes, reads = strain_families()
    sk = sketches_of(genomes, k)
    with mash.Screen(sk, k) as sc:
        sc.add(reads)
        first = sc.results()
        got = sc.winners()
        assert_same(sc.results(), first)  # winners leaves the screen as it was
    assert_same(first, results_of(sk, reads, k))
    assert_same(got, winners_of(sk, reads, k))
    assert (got[0] <= first[0]).all() and int(got[0].sum()) <= int(first[0].sum())
    if k in (21, 31):  # each source strain tops its species, and its siblings lose what it explains
        for sp, st in SOURCES:
            rows = slice(sp * STRAINS, (sp + 1) * STRAINS)
            assert int(np.argmax(got[1][rows])) == st and got[1][sp * STRAINS + st] > 0.5
        assert int((got[1] >= 0.5).sum()) == len(SOURCES) < int((first[1] >= 0.5).sum())


def test_duplicated_and_reordered_rows(gpu):
    """Ties follow the index: a duplicate row wins nothing its lower copy holds, and a permutation of the rows moves
    every answer with its row, except where it reorders tied rows."""
    k = 21
    genomes, reads = strain_families(seed=1)
    sk = sketches_of(genomes, k)
    rng = np.random.default_rng(2)
    dup = np.concatenate([sk, sk[[2, 7, 2]], sk[:3]])  # copies after the originals
    perm = rng.permutation(len(dup))
    bases, off = mash.flatten(reads)
    for rows in (dup, dup[perm], dup[::-1].copy()):
        with mash.Screen(rows, k) as sc:
            sc.add((bases, off))
            got = sc.winners()
        want = winners_of(rows, (bases, off), k)
        assert_same(got, want)
    with mash.Screen(dup, k) as sc:
        sc.add((bases, off))
        w = sc.winners()
    n = len(sk)
    assert (w[0][n:] == 0).all()  # each duplicate loses every tie to its lower copy, so the originals answer as alone
    assert_same([x[:n] for x in w], winners_of(sk, (bases, off), k))


def test_a_value_held_by_every_reference(gpu):
    """100 000 references of s = 4: every row holds one pool word w and a zero tail (the pool has a window hashing
    to 0), so two values have 100 000 contenders each; the first pass's maximum sits deep in the set, once uniquely
    (w) and once at a tie."""
    k, n, s = 21, 100_000, 4
    rng = np.random.default_rng(11)
    genomes, reads = strain_families(seed=3)
    reads = reads[:400]
    z = screen_winners_oracle.window_hashing_to(0, k, b"ACGTTGCAACGTTGCAACGT")
    reads = reads + [np.frombuffer(z + b"A", np.uint8), np.frombuffer(z + b"C", np.uint8)]  # c_pool(0) = 2
    bases, off = mash.flatten(reads)
    pool = np.unique(screen_oracle.pool_hashes(bases, off, k))
    assert pool[0] == 0
    w = int(pool[1])
    absent = int(np.setdiff1d(np.arange(1, 64, dtype=np.uint32), pool)[0])

    def off_pool(x):  # random words, none of them a pool hash
        x = x.astype(np.uint32)
        x[np.isin(x, pool)] = absent
        return x

    sk = np.zeros((n, s), np.uint32)  # column 3: the zero tail
    sk[:, 0] = w
    sk[:, 1] = np.where(rng.random(n) < 0.5, rng.choice(pool[1:], n), off_pool(rng.integers(1, 1 << 32, n, dtype=np.uint64)))
    sk[:, 2] = off_pool(rng.integers(1, 1 << 32, n, dtype=np.uint64))  # so every row shares 2 or 3
    sk[77_777, 1:] = [pool[5], pool[6], 0]  # w, two pool words and a zero: shared 4, the unique maximum
    sk[88_888, 1:] = [pool[5], pool[6], 0]  # a second copy: ties, loses
    with mash.Screen(sk, k) as sc:
        sc.add((bases, off))
        first = sc.results()
        got = sc.winners()
    assert_same(first, results_of(sk, (bases, off), k))
    want = winners_of(sk, (bases, off), k)
    assert_same(got, want)
    assert got[0][77_777] == 4 and got[0][88_888] == 0 and first[0][88_888] == 4
    assert int(got[0].sum()) < int(first[0].sum())


def test_low_complexity_pool_past_32_bit_counts(gpu):
    import torch

    k, L = 21, (1 << 30) + 64
    h = oracle_ffi.murmur3_32(b"A" * k)
    sk = np.array([[h, h, h, 0], [h, 5, 6, 7], [h, h, h, h], [1, 2, 3, 4]], np.uint32)  # first pass 3, 1, 4, 0
    d_bases = torch.full((L,), ord("A"), dtype=torch.uint8, device="cuda")
    d_off = torch.tensor([0, L], dtype=torch.int64, device="cuda")
    with mash.Screen(sk, k) as sc:
        for _ in range(4):
            sc.add_dev(d_bases, d_off)
        c = 4 * (L - k)
        assert c > 1 << 32
        shared, cont, mult = sc.results()
        assert shared.tolist() == [3, 1, 4, 0] and mult.tolist() == [c, c, c, 0]
        shared, cont, mult = sc.winners()
        assert shared.tolist() == [0, 0, 4, 0] and mult.tolist() == [0, 0, c, 0] and cont.tolist() == [0.0, 0.0, 1.0, 0.0]


def test_random_splits_and_reset_equal_one_add(gpu):
    import torch

    k = 21
    genomes, reads = strain_families(seed=5)
    sk = sketches_of(genomes, k)
    want = winners_of(sk, reads, k)
    rng = np.random.default_rng(6)
    stream = torch.cuda.Stream()
    with mash.Screen(sk, k) as sc:
        for trial in range(3):
            sc.reset()
            assert all((x == 0).all() for x in sc.winners())
            cuts = np.sort(rng.integers(0, len(reads) + 1, 6))
            cuts = np.concatenate([[0], cuts, [cuts[-1]], [min(cuts[-1] + 1, len(reads))], [len(reads)]])  # an empty and a one-read add
            for i, (a, b) in enumerate(zip(cuts[:-1], cuts[1:])):
                part = reads[a:b]
                if (i + trial) % 2:
                    sc.add(part)
                else:
                    bases, off = mash.flatten(part)
                    with torch.cuda.stream(stream):
                        sc.add_dev(torch.from_numpy(bases).cuda(), torch.from_numpy(off.astype(np.int64)).cuda(), stream=stream)
            assert_same(sc.winners(), want)


def test_dev_against_host_on_a_side_stream(gpu):
    """winners_dev and results_dev on a non-default stream against the host calls; any subset of outputs; results
    the same before and after winners."""
    import torch

    k = 31
    genomes, reads = strain_families(seed=8)
    sk = sketches_of(genomes, k)
    bases, off = mash.flatten(reads)
    L = _lib.lib()
    n = sk.shape[0]
    stream = torch.cuda.Stream()
    d_sk = torch.from_numpy(sk.view(np.int32)).cuda()
    d_bases = torch.from_numpy(bases).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    stream.wait_stream(torch.cuda.current_stream())
    h = C.c_void_p()

    def dev(fn):
        d = (torch.full((n,), -1, dtype=torch.int32, device="cuda"), torch.full((n,), -1.0, dtype=torch.float64, device="cuda"),
             torch.full((n,), -1, dtype=torch.int64, device="cuda"))
        _lib.check(fn(h, *(x.data_ptr() for x in d), stream.cuda_stream))
        stream.synchronize()
        return d[0].cpu().numpy().view(np.uint32), d[1].cpu().numpy(), d[2].cpu().numpy().view(np.uint64)

    def host(fn, mask=(1, 1, 1)):
        out = np.zeros(n, np.uint32), np.zeros(n, np.float64), np.zeros(n, np.uint64)
        _lib.check(fn(h, *(x.ctypes.data if m else None for x, m in zip(out, mask))))
        return out

    with torch.cuda.stream(stream):
        _lib.check(L.pg_mash_screen_create_dev(d_sk.data_ptr(), n, S, k, stream.cuda_stream, C.byref(h)))
        try:
            _lib.check(L.pg_mash_screen_add_dev(h, d_bases.data_ptr(), d_off.data_ptr(), len(reads), stream.cuda_stream))
            res_before = dev(L.pg_mash_screen_results_dev)
            w_dev = dev(L.pg_mash_screen_winners_dev)
            res_after = dev(L.pg_mash_screen_results_dev)
            w_host = host(L.pg_mash_screen_winners)
            res_host = host(L.pg_mash_screen_results)
            parts = [host(L.pg_mash_screen_winners, mask)[i] for i, mask in enumerate(((1, 0, 0), (0, 1, 0), (0, 0, 1)))]
            _lib.check(L.pg_mash_screen_winners(h, None, None, None))
            _lib.check(L.pg_mash_screen_winners_dev(h, None, None, None, stream.cuda_stream))
            stream.synchronize()
        finally:
            _lib.check(L.pg_mash_screen_free(h))
    assert_same(w_dev, w_host)
    assert_same(parts, w_host)
    assert_same(res_before, res_after)
    assert_same(res_host, res_after)
    assert_same(w_host, winners_of(sk, reads, k))


def test_no_references(gpu):
    k = 21
    _, reads = strain_families(seed=9)
    with mash.Screen(np.zeros((0, S), np.uint32), k) as sc:
        sc.add(reads[:100])
        assert [len(x) for x in sc.winners()] == [0, 0, 0]
        L = _lib.lib()
        assert L.pg_mash_screen_winners(sc._h, None, None, None) == _lib.PG_OK
        assert L.pg_mash_screen_winners_dev(sc._h, None, None, None, None) == _lib.PG_OK


def test_references_that_share_nothing_keep_their_results(gpu):
    """Unrelated genomes (no value in two sketches) and one strain per species: winners == results."""
    k = 21
    genomes, reads = strain_families(seed=10)
    sk = sketches_of(genomes[::STRAINS], k)  # one strain per species
    vals = [set(r.tolist()) for r in sk]
    assert all(not (vals[i] & vals[j]) for i in range(len(vals)) for j in range(i))
    with mash.Screen(sk, k) as sc:
        sc.add(reads)
        first = sc.results()
        assert_same(sc.winners(), first)
    assert first[0].max() > S // 2
    one = sketches_of(genomes[:1], k)  # n = 1
    with mash.Screen(one, k) as sc:
        sc.add(reads)
        assert_same(sc.winners(), sc.results())


def test_cpp_mirror_agrees_with_the_restatement(gpu):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "screen_winners_tests"])
    k = 21
    genomes, reads = strain_families(seed=12)
    sk = sketches_of(genomes, k)
    want = winners_of(sk, reads, k)
    with tempfile.TemporaryDirectory() as td:
        refs, txt = os.path.join(td, "refs.pgsketch"), os.path.join(td, "reads.txt")
        sketchfile.save(refs, sk, np.full(len(sk), S, np.uint32), k, S)
        with open(txt, "wb") as f:
            f.write(b"\n".join(r.tobytes() for r in reads) + b"\n")
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "screen_winners_tests"), refs, txt, str(k), "4"], capture_output=True,
                             text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: screen winners tests pass"
    assert len(lines) == len(sk) + 1
    for r, line in enumerate(lines[:-1]):
        i, shared, bits, mult = line.split()
        assert (int(i), int(shared), int(bits, 16), int(mult)) == (r, int(want[0][r]), int(want[1][r:r + 1].view(np.uint64)[0]), int(want[2][r]))
