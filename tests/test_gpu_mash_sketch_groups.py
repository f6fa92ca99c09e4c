"""The grouped sketch on the GPU (pg_mash_sketch_groups): rows and counts byte for byte against the restatement in
tests/sketch_groups_oracle.py on random groups for walk and generic k, the per-record sketch of one long record, a
read set filtered at min_copies 2 over several passes, degenerate groups (poly-A, short periods, a table overflow),
invariance under reordering and splitting, the _dev form, assemblies through cluster and screen, and the C++
mirror."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

import oracle_ffi
import sketch_groups_oracle as oracle
from poly_b200 import _lib, mash

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
THREADS = len(os.sched_getaffinity(0))
ACGT = np.frombuffer(b"ACGT", np.uint8)
# one pass of the call is 3 launches (walk, collect, append) after 2 of set-up (window counts, group sizes)
SETUP_LAUNCHES, PASS_LAUNCHES = 2, 3


def rand_seq(rng, n):
    return ACGT[rng.integers(0, 4, n)]


def random_groups(rng, k, n_groups=7):
    """Groups of 1..50 records of 0..5000 bytes cut from a per-group source, so values recur; an empty group, a group
    of records no longer than k, and one with a (k+1)-byte record."""
    groups = []
    for g in range(n_groups):
        src = rand_seq(rng, int(rng.integers(2000, 20000)))
        recs = []
        for _ in range(int(rng.integers(1, 51))):
            L = int(min(rng.integers(0, 5001), len(src)))
            a = int(rng.integers(0, len(src) - L + 1))
            recs.append(src[a:a + L].copy())
        groups.append(recs)
    groups.insert(2, [])
    groups.insert(4, [rand_seq(rng, k), rand_seq(rng, max(k - 1, 0)), np.zeros(0, np.uint8)])
    groups.append([rand_seq(rng, k + 1)])
    return groups


def run(groups, k, s, m):
    bases, off, goff = oracle.flatten_groups(groups)
    return mash.sketch_groups(bases, off, goff, k, s, m), (bases, off, goff)


def assert_rows(got, want):
    assert got[1].tobytes() == want[1].tobytes(), (got[1], want[1])
    assert got[0].tobytes() == want[0].tobytes()


@pytest.mark.parametrize("k", [0, 11, 16, 21, 31, 33])
@pytest.mark.parametrize("s", [1, 2, 100, 1000, 20000])
def test_random_groups_match_the_oracle(gpu, k, s):
    rng = np.random.default_rng(1000 * k + s)
    groups = random_groups(rng, k)
    for m in (1, 2, 3):
        got, (bases, off, goff) = run(groups, k, s, m)
        assert_rows(got, oracle.sketch_groups(bases, off, goff, k, s, m, THREADS))


def test_one_record_equals_the_per_record_sketch(gpu):
    rng = np.random.default_rng(2)
    rec = rand_seq(rng, 200_000)
    k, s = 21, 1000
    rows, count = mash.sketch_groups(rec, np.array([0, len(rec)], np.uint64), np.array([0, 1], np.uint64), k, s)
    out, cnt, status = mash.sketch_arrays(rec, np.array([0, len(rec)], np.uint64), k, s)
    assert status[0] == 0 and cnt[0] == s and count[0] == s
    assert len(np.unique(out[0])) == s  # its bottom-s multiset holds no repeat
    assert rows[0].tobytes() == out[0].tobytes()


def read_set(rng, genome, coverage=30, L=150, err=0.01):
    n = len(genome) * coverage // L
    st = rng.integers(0, len(genome) - L + 1, n)
    reads = genome[st[:, None] + np.arange(L)]
    sub = ACGT[(np.searchsorted(ACGT, reads) + rng.integers(1, 4, reads.shape)) % 4]
    reads = np.where(rng.random(reads.shape) < err, sub, reads)
    return np.ascontiguousarray(reads.reshape(-1)), np.arange(n + 1, dtype=np.uint64) * np.uint64(L)


def distance(a, b, k, s):
    x, y = mash.Mash(k, s), mash.Mash(k, s)
    x.Sketches[:], y.Sketches[:] = a, b
    return x.Distance(y)


def test_read_set_filtered_by_min_copies(gpu):
    rng = np.random.default_rng(3)
    k, s = 21, 1000
    genome = rand_seq(rng, 200_000)
    bases, off = read_set(rng, genome)
    goff = np.array([0, len(off) - 1], np.uint64)
    ref = mash.sketch_groups(genome, np.array([0, len(genome)], np.uint64), np.array([0, 1], np.uint64), k, s)[0][0]
    dist = {}
    for m in (1, 2):
        before = _lib.lib().pg_launch_count()
        got = mash.sketch_groups(bases, off, goff, k, s, m)
        launches = _lib.lib().pg_launch_count() - before
        assert_rows(got, oracle.sketch_groups(bases, off, goff, k, s, m, THREADS))
        if m == 2:
            assert launches > SETUP_LAUNCHES + PASS_LAUNCHES, launches  # more than one pass ran
        dist[m] = distance(got[0][0], ref, k, s)
    # At 1 % substitutions and ~26x window coverage about 8 % of the error k-mers recur, so m = 2 keeps some of them;
    # m = 1 keeps every one and its bottom-s is mostly errors.
    assert dist[2] < 0.2 and dist[1] > 0.7, dist


def test_degenerate_groups(gpu):
    k, s = 21, 100
    rng = np.random.default_rng(4)
    poly_a = np.full(10_000_000, ord("A"), np.uint8)
    period3 = np.tile(np.frombuffer(b"ACG", np.uint8), 5000)
    two = np.tile(np.frombuffer(b"AT", np.uint8), 5000)
    groups = [[poly_a], [period3, two], [two]]
    got, (bases, off, goff) = run(groups, k, s, 1)
    assert_rows(got, oracle.sketch_groups(bases, off, goff, k, s, 1, THREADS))
    rows, count = got
    assert list(count) == [1, 5, 2] and not rows[:, 5:].any()
    got2, _ = run(groups, k, s, 3)
    assert_rows(got2, oracle.sketch_groups(bases, off, goff, k, s, 3, THREADS))


def mm3_word(w):
    """murmur3.Sum32 of 4-byte keys (little-endian words w), seed 0."""
    M = np.uint64(0xFFFFFFFF)
    w = w.astype(np.uint64)
    rotl = lambda x, r: ((x << np.uint64(r)) | (x >> np.uint64(32 - r))) & M
    k1 = rotl((w * np.uint64(0xCC9E2D51)) & M, 15) * np.uint64(0x1B873593) & M
    h = rotl(k1, 13) * np.uint64(5) + np.uint64(0xE6546B64) & M
    h ^= np.uint64(4)
    for sh, c in ((16, 0x85EBCA6B), (13, 0xC2B2AE35)):
        h = (h ^ (h >> np.uint64(sh))) * np.uint64(c) & M
    return (h ^ (h >> np.uint64(16))).astype(np.uint32)


def test_table_overflow_retries(gpu):
    """k = 4, s = 1, m = 2, built so that a table overflows: 10^6 windows of one value (a poly-A record) set the first
    range to [0, T1), T1 = 55 / 10^6 of the hash range, which holds two single windows; the second range is 64 T1 wide
    and its table is sized from those two values per T1 (2 x 128 expected, 512 slots), but it holds 1 000 distinct
    single windows.  The pass is dropped and retried narrower; the row must still be exact."""
    rng = np.random.default_rng(5)
    k, s, m = 4, 1, 2
    words = rng.integers(0, 1 << 32, 1 << 22, dtype=np.uint64).astype(np.uint32)
    h = mm3_word(words)
    W = 1_000_000
    T1 = int(np.ceil((1 + 6 + 48) / W * 2.0 ** 32))
    low = np.unique(words[h < T1])[:2]
    mid = np.unique(words[(h >= T1) & (h < 65 * T1)])[:1000]
    assert len(low) == 2 and len(mid) == 1000
    recs = [np.frombuffer(x.tobytes() + b"C", np.uint8) for x in np.concatenate([low, mid])]  # one window each
    recs.append(np.full(W + k, ord("A"), np.uint8))
    groups = [recs, [np.full(300, ord("A"), np.uint8)]]
    got, (bases, off, goff) = run(groups, k, s, m)
    want = oracle.sketch_groups(bases, off, goff, k, s, m, THREADS)
    assert mm3_word(np.frombuffer(b"AAAA", np.uint32))[0] == want[0][1][0]  # the hash restated here is murmur3
    assert_rows(got, want)


def test_invariance(gpu):
    rng = np.random.default_rng(6)
    k, s, m = 21, 200, 2
    groups = random_groups(rng, k, n_groups=9)
    base, _ = run(groups, k, s, m)
    shuffled = [[g[i] for i in rng.permutation(len(g))] for g in groups]
    assert_rows(run(shuffled, k, s, m)[0], base)
    perm = rng.permutation(len(groups))
    rows, count = run([groups[i] for i in perm], k, s, m)[0]
    assert rows.tobytes() == base[0][perm].tobytes() and count.tobytes() == base[1][perm].tobytes()
    parts = [run(groups[a:b], k, s, m)[0] for a, b in ((0, 3), (3, 7), (7, len(groups)))]
    assert np.concatenate([p[0] for p in parts]).tobytes() == base[0].tobytes()
    assert np.concatenate([p[1] for p in parts]).tobytes() == base[1].tobytes()


def test_dev_equals_host_and_row_stride(gpu):
    import torch

    rng = np.random.default_rng(7)
    k, s, m = 21, 300, 1
    groups = random_groups(rng, k)
    (rows, count), (bases, off, goff) = run(groups, k, s, m)
    dev = torch.device("cuda", 0)
    d_rows, d_count = mash.sketch_groups(torch.from_numpy(bases).to(dev), torch.from_numpy(off.view(np.int64)).to(dev),
                                         torch.from_numpy(goff.view(np.int64)).to(dev), k, s, m)
    assert d_rows.cpu().numpy().view(np.uint32).tobytes() == rows.tobytes()
    assert d_count.cpu().numpy().view(np.uint32).tobytes() == count.tobytes()
    G, stride = len(goff) - 1, s + 37
    out = np.full((G, stride), 0xABCD, np.uint32)
    cnt = np.zeros(G, np.uint32)
    _lib.check(_lib.lib().pg_mash_sketch_groups(bases.ctypes.data, off.ctypes.data, len(off) - 1, goff.ctypes.data, G, k, s, m, out.ctypes.data,
                                                stride, cnt.ctypes.data))
    assert out[:, :s].tobytes() == rows.tobytes() and not out[:, s:].any() and cnt.tobytes() == count.tobytes()


def cut(rng, genome, pieces):
    at = np.sort(rng.choice(np.arange(1, len(genome)), pieces - 1, replace=False))
    return np.split(genome, at)


def test_assemblies_cluster_and_screen(gpu):
    rng = np.random.default_rng(8)
    k, s = 21, 1000
    genomes = [rand_seq(rng, 1_000_000) for _ in range(20)]
    groups = [cut(rng, g, 50) for g in genomes] + [cut(rng, g, 50) for g in genomes]
    rows, count = run(groups, k, s, 1)[0]
    assert (count == s).all()
    labels, n_groups, _ = mash.cluster(rows, max_distance=0.05)
    assert n_groups == 20 and all(labels[i] == labels[i + 20] for i in range(20))
    picked = [1, 4, 9, 13, 17]
    reads = []
    for i in picked:
        st = rng.integers(0, len(genomes[i]) - 150, len(genomes[i]) * 20 // 150)
        reads.append(genomes[i][st[:, None] + np.arange(150)])
    reads = np.ascontiguousarray(np.concatenate(reads).reshape(-1))
    off = np.arange(len(reads) // 150 + 1, dtype=np.uint64) * np.uint64(150)
    with mash.Screen(rows[:20], k) as sc:
        sc.add((reads, off))
        _, cont, _ = sc.results()
    for i in range(20):
        assert (cont[i] >= 0.99) if i in picked else (cont[i] < 0.2), (i, cont[i])


def test_cpp_mirror_agrees_with_the_oracle(gpu):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "sketch_groups_tests"])
    rng = np.random.default_rng(9)
    k, s, m = 21, 500, 2
    groups = [g for g in random_groups(rng, k) if g]
    with tempfile.TemporaryDirectory() as td:
        txt = os.path.join(td, "groups.txt")
        with open(txt, "wb") as f:  # one record per line, "g record"; records with no byte are left out
            for g, recs in enumerate(groups):
                f.write(b"".join(b"%d " % g + bytes(r) + b"\n" for r in recs if len(r)))
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "sketch_groups_tests"), txt, str(len(groups)), str(k), str(s), str(m)],
                             capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: sketch groups tests pass"
    bases, off, goff = oracle.flatten_groups([[r for r in g if len(r)] for g in groups])
    rows, count = oracle.sketch_groups(bases, off, goff, k, s, m, THREADS)
    assert len(lines) == len(groups) + 1
    for g, line in enumerate(lines[:-1]):
        vals = [int(x) for x in line.split()]
        assert vals[0] == count[g] and vals[1:] == [int(v) for v in rows[g, :count[g]]]
