"""Mash Screen on the GPU (pg_mash_screen_*): shared, multiplicity and the bytes of containment against the CPU oracle
(tests/screen_oracle.py) for walk and generic k, ragged pools with empty, k-, k+1- and 100 kbp reads, select- and
fill-regime references, hand-built words at the edges of the value directory, a low-complexity pool, split adds,
reset, host against _dev paths, no references, and the C++ mirror."""
import ctypes as C
import itertools
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle_ffi
import screen_oracle
from poly_b200 import _lib, mash, sketchfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
THREADS = len(os.sched_getaffinity(0))
S = 200


def pool_reads(k, seed=0, n_short=1500):
    """Reads of length 0, k, k + 1, two of 100 kbp (they cross many chunks of the add kernel), a repeat-rich one,
    and short reads of 20..300 bp drawn from the long ones with a few substitutions."""
    rng = np.random.default_rng(seed)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    long_reads = [acgt[rng.integers(0, 4, 100_000)] for _ in range(2)]
    reads = [np.zeros(0, np.uint8), acgt[rng.integers(0, 4, k)], acgt[rng.integers(0, 4, k + 1)], *long_reads,
             np.tile(acgt[rng.integers(0, 4, 7)], 300)]
    for _ in range(n_short):
        src = long_reads[int(rng.integers(0, 2))]
        L = int(rng.integers(20, 301))
        a = int(rng.integers(0, len(src) - L))
        r = src[a:a + L].copy()
        r[rng.random(L) < 0.01] = acgt[rng.integers(0, 4)]
        reads.append(r)
    order = rng.permutation(len(reads))
    return [reads[i] for i in order]


def references(reads, k, seed=0):
    """Select-regime sketches of the 100 kbp reads (every hash in the pool), fill-regime sketches of short reads
    (unsorted, zero tails), sketches of reads not in the pool, and random words."""
    rng = np.random.default_rng(seed + 1)
    longs = [r for r in reads if len(r) >= 100_000]
    shorts = [r for r in reads if 0 < len(r) < 150][:6]
    others = [np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, 5000)] for _ in range(2)]
    bases, off = mash.flatten(longs + shorts + others)
    rc, sk = oracle_ffi.sketch_batch(bases, off, k, S, variant=1, nthreads=THREADS)
    assert rc == 0
    rand = rng.integers(0, 1 << 32, (3, S), dtype=np.uint64).astype(np.uint32)
    return np.ascontiguousarray(np.concatenate([sk, rand]), np.uint32), len(longs)


def oracle_of(sk, reads, k):
    return screen_oracle.mash_screen(sk, mash.flatten(reads), k, nthreads=THREADS)


def assert_same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.tobytes() == w.tobytes(), (g, w)


@pytest.mark.parametrize("k", [21, 31, 32, 11, 12, 33, 0])
def test_pool_against_oracle(gpu, k):
    reads = pool_reads(k)
    sk, n_select = references(reads, k)
    want = oracle_of(sk, reads, k)
    with mash.Screen(sk, k) as sc:
        sc.add(reads)
        got = sc.results()
    assert_same(got, want)
    if k > 0:  # the long reads' own sketches: every hash is in the pool
        assert (got[0][:n_select] == S).all() and (got[1][:n_select] == 1.0).all()
    assert got[0][n_select:].min() < S


def test_directory_edges(gpu):
    """Reference words at 0, at the largest value, at 0xFFFFFFFF and one either side of pool hashes, so that many
    values sit on both sides of bucket boundaries."""
    k = 21
    reads = pool_reads(k, seed=3, n_short=300)
    bases, off = mash.flatten(reads)
    windows = itertools.islice(((r, p) for r in reads for p in range(max(len(r) - k, 0))), 20000)
    hashes = np.unique(np.array([oracle_ffi.murmur3_32(r[p:p + k].tobytes()) for r, p in windows], np.uint64))
    near = np.unique(np.concatenate([hashes - 1, hashes, hashes + 1]))
    near = near[(near >= 0) & (near <= 0xFFFFFFFF)].astype(np.uint32)
    s = 64
    rows = -(-len(near) // s)
    words = np.zeros(rows * s, np.uint32)
    words[: len(near)] = near[np.random.default_rng(4).permutation(len(near))]
    base = words.reshape(rows, s)
    edge = base.copy()
    edge[0, :3] = [0, 0xFFFFFFFF, int(hashes.max())]
    for sk in (base, edge):  # vmax a pool hash + 1 (or so), then 0xFFFFFFFF: every window a candidate
        with mash.Screen(sk, k) as sc:
            sc.add((bases, off))
            assert_same(sc.results(), screen_oracle.mash_screen(sk, (bases, off), k, nthreads=THREADS))


def test_low_complexity_pool_counts_exactly(gpu):
    import torch

    k, n, L = 21, 1_000_000, 32
    h = oracle_ffi.murmur3_32(b"A" * k)
    sk = np.array([[h, h, h, 0], [h, 5, 6, 7], [1, 2, 3, 4]], np.uint32)
    d_bases = torch.full((n * L,), ord("A"), dtype=torch.uint8, device="cuda")
    d_off = torch.arange(n + 1, dtype=torch.int64, device="cuda") * L
    with mash.Screen(sk, k) as sc:
        sc.add_dev(d_bases, d_off)
        shared, cont, mult = sc.results()
        c = n * (L - k)
        assert shared.tolist() == [3, 1, 0] and mult.tolist() == [c, c, 0] and cont.tolist() == [0.75, 0.25, 0.0]
        sc.add_dev(d_bases, d_off)
        assert sc.results()[2].tolist() == [2 * c, 2 * c, 0]


def test_random_splits_equal_one_add(gpu):
    import torch

    k = 21
    reads = pool_reads(k, seed=5, n_short=600)
    sk, _ = references(reads, k, seed=5)
    want = oracle_of(sk, reads, k)
    rng = np.random.default_rng(6)
    stream = torch.cuda.Stream()
    with mash.Screen(sk, k) as sc:
        for trial in range(3):
            sc.reset()
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
            assert_same(sc.results(), want)


def test_reset_answers_as_a_fresh_screen(gpu):
    k = 31
    reads = pool_reads(k, seed=7, n_short=200)
    sk, _ = references(reads, k, seed=7)
    with mash.Screen(sk, k) as sc:
        sc.add(reads[:50])
        sc.reset()
        assert all((x == 0).all() for x in sc.results())
        sc.add(reads)
        got = sc.results()
    with mash.Screen(sk, k) as fresh:
        fresh.add(reads)
        assert_same(got, fresh.results())
    assert_same(got, oracle_of(sk, reads, k))


def test_host_and_dev_paths_identical(gpu):
    """create_dev, add_dev on a non-default stream from an unaligned base with offsets that do not start at 0, and
    results_dev, against the host calls."""
    import torch

    k = 21
    reads = pool_reads(k, seed=8, n_short=400)
    sk, _ = references(reads, k, seed=8)
    bases, off = mash.flatten(reads)
    want = oracle_of(sk, reads, k)
    L = _lib.lib()
    stream = torch.cuda.Stream()
    pad = np.frombuffer(b"GATTACA", np.uint8)  # 7 bytes before the pool: its windows must not count
    d_bases = torch.from_numpy(np.concatenate([pad, bases])).cuda()
    d_off6 = torch.from_numpy((off + len(pad) - 1).astype(np.int64)).cuda()
    d_off7 = torch.from_numpy((off + len(pad)).astype(np.int64)).cuda()
    d_sk = torch.from_numpy(sk.view(np.int32)).cuda()
    stream.wait_stream(torch.cuda.current_stream())
    h = C.c_void_p()
    with torch.cuda.stream(stream):
        _lib.check(L.pg_mash_screen_create_dev(d_sk.data_ptr(), sk.shape[0], sk.shape[1], k, stream.cuda_stream, C.byref(h)))
        try:
            # the pool twice: from a base one byte into the buffer, then from the buffer itself, so the kernel's
            # chunks start at different alignments; counts double
            _lib.check(L.pg_mash_screen_add_dev(h, d_bases.data_ptr() + 1, d_off6.data_ptr(), len(reads), stream.cuda_stream))
            _lib.check(L.pg_mash_screen_add_dev(h, d_bases.data_ptr(), d_off7.data_ptr(), len(reads), stream.cuda_stream))
            n = sk.shape[0]
            d_sh = torch.empty(n, dtype=torch.int32, device="cuda")
            d_c = torch.empty(n, dtype=torch.float64, device="cuda")
            d_m = torch.empty(n, dtype=torch.int64, device="cuda")
            _lib.check(L.pg_mash_screen_results_dev(h, d_sh.data_ptr(), d_c.data_ptr(), d_m.data_ptr(), stream.cuda_stream))
            stream.synchronize()
            got_dev = (d_sh.cpu().numpy().view(np.uint32), d_c.cpu().numpy(), d_m.cpu().numpy().view(np.uint64))
            host = np.zeros(n, np.uint32), np.zeros(n, np.float64), np.zeros(n, np.uint64)
            _lib.check(L.pg_mash_screen_results(h, *(x.ctypes.data for x in host)))
        finally:
            _lib.check(L.pg_mash_screen_free(h))
    assert_same(got_dev, host)
    twice = oracle_of(sk, reads + reads, k)
    assert_same(host, twice)
    with mash.Screen(sk, k) as sc:
        sc.add(reads)
        assert_same(sc.results(), want)


def test_identity_and_no_references(gpu):
    k = 21
    reads = pool_reads(k, seed=9, n_short=100)
    with mash.Screen(np.zeros((0, S), np.uint32), k) as sc:
        sc.add(reads)
        assert [len(x) for x in sc.results()] == [0, 0, 0]
    sk, _ = references(reads, k, seed=9)
    with mash.Screen(sk, k) as sc:
        sc.add(reads)
        assert np.array_equal(sc.identity(), sc.results()[1] ** (1.0 / k))


def test_decreasing_offsets_are_refused_in_a_host_add(gpu):
    sk = np.ones((1, 4), np.uint32)
    with mash.Screen(sk, 21) as sc:
        with pytest.raises(_lib.PolyError) as e:
            sc.add((np.zeros(64, np.uint8), np.array([0, 40, 30, 64], np.uint64)))
        assert e.value.code == _lib.PG_ERR_ARG
        assert sc.results()[0].tolist() == [0]


def test_cpp_mirror_agrees_with_the_oracle(gpu):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "screen_tests"])
    k = 21
    reads = [r for r in pool_reads(k, seed=10, n_short=300)]
    sk, _ = references(reads, k, seed=10)
    want = oracle_of(sk, reads, k)
    with tempfile.TemporaryDirectory() as td:
        refs, txt = os.path.join(td, "refs.pgsketch"), os.path.join(td, "reads.txt")
        sketchfile.save(refs, sk, np.full(len(sk), S, np.uint32), k, S)
        with open(txt, "wb") as f:
            f.write(b"\n".join(r.tobytes() for r in reads) + b"\n")
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "screen_tests"), refs, txt, str(k), "4"], capture_output=True, text=True,
                             timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: screen tests pass"
    for r, line in enumerate(lines[:-1]):
        i, shared, bits, mult = line.split()
        assert (int(i), int(shared), int(bits, 16), int(mult)) == (r, int(want[0][r]), int(want[1][r:r + 1].view(np.uint64)[0]), int(want[2][r]))
