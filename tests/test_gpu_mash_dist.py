"""GPU tier of the Mash distance between grouped sketches (pg_mash_dist, pg_mash_dist_within): the device against the
plain restatement (mash_dist_oracle) on seeded row sets, its symmetry and self-pair rules, the _dev forms, the filtered
list, and end to end from genomes sketched by pg_mash_sketch_groups."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

import mash_dist_oracle as oracle
from poly_b200 import _lib, mash

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U32 = 1 << 32

pytestmark = pytest.mark.gpu


def row_set(rng, n, s, pool):
    """n rows of width s drawn from the sorted value pool: full rows, short rows, empty rows, copies of the row before,
    rows sharing a prefix with the row before, and rows holding 0 and 2^32 - 1."""
    rows, count = np.zeros((n, s), np.uint32), np.zeros(n, np.uint32)
    for i in range(n):
        kind = i % 7
        if kind in (0, 6):
            v = np.sort(rng.choice(pool, size=min(s, len(pool)), replace=False))
        elif kind == 1:
            v = np.sort(rng.choice(pool, size=int(rng.integers(1, s + 1)), replace=False))
        elif kind == 2:
            v = np.zeros(0, np.uint32) if i % 14 == 2 else np.sort(rng.choice(pool, size=int(rng.integers(0, max(s // 10, 1) + 1)), replace=False))
        elif kind == 3 and i:
            v = rows[i - 1, : count[i - 1]].copy()
        elif kind == 4 and i:
            m = int(rng.integers(0, count[i - 1] + 1))
            v = np.union1d(rows[i - 1, :m], rng.choice(pool, size=s, replace=False))[:s]
        else:
            v = np.union1d(np.array([0, U32 - 1], np.uint32), rng.choice(pool, size=s, replace=False))[:s]
        v = np.unique(v.astype(np.uint32))[:s]
        rows[i, : len(v)] = v
        count[i] = len(v)
    return rows, count


def check_against_oracle(got, want):
    (gc, gd, gdist, gp), (wc, wd, wdist, wp) = got, want
    assert np.array_equal(gc, wc) and np.array_equal(gd, wd)
    exact = (wdist == 0.0) | (wdist == 1.0)
    assert np.array_equal(gdist[exact], wdist[exact]) and not np.signbit(gdist[exact]).any()
    assert (np.abs(gdist[~exact] - wdist[~exact]) <= 2 * np.spacing(wdist[~exact])).all()
    if wp is not None:
        big = wp >= 1e-290
        rel = np.abs(gp[big] - wp[big]) / wp[big]
        assert (rel <= 1e-9).all(), float(rel.max())
        assert (gp[~big] <= 1e-280).all()


# s = 3418 is the largest s whose rows are staged in shared memory; 3419 reads them from global memory
@pytest.mark.parametrize("s,nq,nr,k,pool", [(1, 37, 45, 21, 3), (10, 37, 45, 6, 25), (1000, 37, 45, 21, 2500), (1000, 33, 70, 3, 1600),
                                            (3418, 5, 7, 21, 6000), (3419, 5, 7, 6, 6000)])
def test_row_sets_match_the_oracle(gpu, s, nq, nr, k, pool):
    rng = np.random.default_rng(s * 1000 + nq + k)
    vals = np.unique(rng.integers(0, U32, size=pool, dtype=np.uint64)).astype(np.uint32)
    q, qc = row_set(rng, nq, s, vals)
    r, rc = row_set(rng, nr, s, vals)
    r[: nq // 2], rc[: nq // 2] = q[: nq // 2], qc[: nq // 2]  # some references are copies of queries
    ql = rng.integers(1, 10 ** 6, size=nq, dtype=np.uint64)
    rl = rng.integers(1, 10 ** 6, size=nr, dtype=np.uint64)
    got = mash.dist(q, qc, r, rc, k, ql, rl)
    check_against_oracle(got, oracle.dist(q, qc, r, rc, k, ql, rl))
    # swapping the sets with their lengths transposes every output bit for bit
    back = mash.dist(r, rc, q, qc, k, rl, ql)
    for a, b in zip(got, back):
        assert np.array_equal(a.view(np.uint64 if a.dtype == np.float64 else np.uint32), b.T.view(np.uint64 if b.dtype == np.float64 else np.uint32))
    # a row against itself: common = denom = count, distance 0
    c, d, dist, _ = mash.dist(q, qc, q, qc, k)
    assert np.array_equal(np.diag(c), qc) and np.array_equal(np.diag(d), qc) and (np.diag(dist) == 0).all()
    # without lengths no p-value; the other outputs are the same
    assert np.array_equal(dist, mash.dist(q, qc, q, qc, k, ql, ql)[2])


def test_dev_equals_host_and_row_stride(gpu):
    import torch

    rng = np.random.default_rng(5)
    s, k = 300, 15
    vals = np.unique(rng.integers(0, U32, size=700, dtype=np.uint64)).astype(np.uint32)
    q, qc = row_set(rng, 40, s, vals)
    r, rc = row_set(rng, 29, s, vals)
    ql, rl = rng.integers(1, 10 ** 9, size=40, dtype=np.uint64), rng.integers(1, 10 ** 9, size=29, dtype=np.uint64)
    host = mash.dist(q, qc, r, rc, k, ql, rl)
    t = lambda a: torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a.view(np.int64)).cuda()
    dev = mash.dist(t(q), t(qc), t(r), t(rc), k, t(ql), t(rl))
    torch.cuda.synchronize()
    for h, d in zip(host, dev):
        assert np.array_equal(h.view(np.uint8), d.cpu().numpy().view(np.uint8))
    # a row stride wider than s: the words past each count are never read
    stride = s + 13
    wq, wr = np.full((40, stride), 7, np.uint32), np.full((29, stride), 7, np.uint32)
    wq[:, :s], wr[:, :s] = q, r
    for i in range(40):
        wq[i, qc[i]:] = rng.integers(0, U32, size=stride - qc[i], dtype=np.uint64).astype(np.uint32)
    out = [np.zeros((40, 29), np.uint32), np.zeros((40, 29), np.uint32), np.zeros((40, 29)), np.zeros((40, 29))]
    _lib.check(_lib.lib().pg_mash_dist(wq.ctypes.data, qc.ctypes.data, 40, wr.ctypes.data, rc.ctypes.data, 29, stride, s, k, ql.ctypes.data,
                                       rl.ctypes.data, *[o.ctypes.data for o in out]))
    for h, o in zip(host, out):
        assert np.array_equal(h, o)


def test_host_blocks_match_one_block(gpu):
    # the host form cuts the queries into blocks under 1 GiB of outputs; 2 500 x 20 000 pairs of four outputs is 1.2 GB
    rng = np.random.default_rng(9)
    s, k = 8, 9
    vals = np.unique(rng.integers(0, U32, size=40, dtype=np.uint64)).astype(np.uint32)
    q, qc = row_set(rng, 2500, s, vals)
    r, rc = row_set(rng, 20000, s, vals)
    ql, rl = np.full(2500, 5000, np.uint64), np.full(20000, 7000, np.uint64)
    c, d, dist, p = mash.dist(q, qc, r, rc, k, ql, rl)
    for rows in (slice(0, 3), slice(1300, 1303), slice(2497, 2500)):
        part = mash.dist(q[rows], qc[rows], r, rc, k, ql[rows], rl)
        for a, b in zip((c, d, dist, p), part):
            assert np.array_equal(a[rows], b)


def filtered(dense, max_d, max_p, upper):
    c, d, dist, p = dense
    keep = (dist <= max_d) & ((p if p is not None else np.zeros_like(dist)) <= max_p)
    if upper:
        keep &= np.triu(np.ones_like(keep), 1).astype(bool)
    qi, ri = (a.astype(np.uint32) for a in np.nonzero(keep))
    return qi, ri, c[qi, ri], d[qi, ri], dist[qi, ri], (p[qi, ri] if p is not None else None)


@pytest.mark.parametrize("upper", [False, True])
def test_within_equals_the_filtered_block(gpu, upper):
    import torch

    rng = np.random.default_rng(11 + upper)
    s, k = 500, 12
    vals = np.unique(rng.integers(0, U32, size=900, dtype=np.uint64)).astype(np.uint32)
    q, qc = row_set(rng, 90, s, vals)
    ql = rng.integers(1, 10 ** 7, size=90, dtype=np.uint64)
    dense = mash.dist(q, qc, q, qc, k, ql, ql)
    for max_d, max_p in ((1.0, 1.0), (0.08, 1.0), (0.08, 1e-30), (0.0, 1.0)):
        got = mash.dist_within(q, qc, q, qc, k, ql, ql, max_d, max_p, upper)
        want = filtered(dense, max_d, max_p, upper)
        for a, b in zip(got, want):
            assert np.array_equal(a, b)
        t = lambda a: torch.from_numpy(a.view(np.int32) if a.dtype == np.uint32 else a.view(np.int64)).cuda()
        dev = mash.dist_within(t(q), t(qc), t(q), t(qc), k, t(ql), t(ql), max_d, max_p, upper)
        for a, b in zip(dev, want):
            assert np.array_equal(a.cpu().numpy().view(b.dtype), b)
    # without lengths, a distance cut only
    got = mash.dist_within(q, qc, q, qc, k, max_distance=0.08, upper=upper)
    want = filtered((dense[0], dense[1], dense[2], None), 0.08, 1.0, upper)
    assert got[5] is None and all(np.array_equal(a, b) for a, b in zip(got[:5], want[:5]))


def test_within_cap_overflow(gpu):
    import torch

    rng = np.random.default_rng(13)
    s, k = 64, 21
    vals = np.unique(rng.integers(0, U32, size=100, dtype=np.uint64)).astype(np.uint32)
    q, qc = row_set(rng, 50, s, vals)
    want = filtered(mash.dist(q, qc, q, qc, k), 1.0, 1.0, True)
    n_true = len(want[0])
    truth = set(zip(want[0].tolist(), want[1].tolist()))
    cap = n_true // 3
    pq, pr = np.zeros(cap, np.uint32), np.zeros(cap, np.uint32)
    dist = np.zeros(cap)
    cnt = C.c_uint64(0)
    rc = _lib.lib().pg_mash_dist_within(q.ctypes.data, qc.ctypes.data, 50, q.ctypes.data, qc.ctypes.data, 50, s, s, k, None, None, 1.0, 1.0,
                                        _lib.PG_PAIRS_UPPER, pq.ctypes.data, pr.ctypes.data, None, None, dist.ctypes.data, None, cap, C.byref(cnt))
    assert rc == _lib.PG_ERR_ARG and "pairs_cap" in _lib.last_error() and cnt.value == n_true
    stored = set(zip(pq.tolist(), pr.tolist()))
    assert len(stored) == cap and stored <= truth
    # _dev: the device counter holds the true count, the first cap entries are stored, and the call does not fail
    t = lambda a: torch.from_numpy(a.view(np.int32)).cuda()
    dq, dc = t(q), t(qc)
    d_pq, d_pr = torch.zeros(cap, dtype=torch.int32, device="cuda"), torch.zeros(cap, dtype=torch.int32, device="cuda")
    d_n = torch.full((1,), 12345, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(_lib.lib().pg_mash_dist_within_dev(dq.data_ptr(), dc.data_ptr(), 50, dq.data_ptr(), dc.data_ptr(), 50, s, s, k, None, None, 1.0, 1.0,
                                                  _lib.PG_PAIRS_UPPER, d_pq.data_ptr(), d_pr.data_ptr(), None, None, None, None, cap, d_n.data_ptr(), st))
    assert int(d_n.item()) == n_true
    assert set(zip(d_pq.cpu().tolist(), d_pr.cpu().tolist())) <= truth


# ---- end to end from genomes -----------------------------------------------------------------------------------
ACGT = np.frombuffer(b"ACGT", np.uint8)


def mutate(rng, genome, p):
    g = genome.copy()
    sub = rng.random(len(g)) < p
    idx = np.searchsorted(ACGT, g[sub])
    g[sub] = ACGT[(idx + rng.integers(1, 4, size=int(sub.sum()))) % 4]
    return g


def sketch(genomes, k, s, canonical=False):
    bases, off = mash.flatten(genomes)
    goff = np.arange(len(genomes) + 1, dtype=np.uint64)
    rows, count = mash.sketch_groups(bases, off, goff, k, s, canonical=canonical)
    return rows, count, np.array([len(g) for g in genomes], np.uint64)


def test_species_and_strains(gpu):
    rng = np.random.default_rng(17)
    k, s, G, P = 21, 1000, 200_000, 4
    rates = [0.005, 0.01, 0.02, 0.03, 0.05]
    genomes = []
    for _ in range(P):
        root = ACGT[rng.integers(0, 4, size=G)]
        genomes += [root] + [mutate(rng, root, p) for p in rates]
    rows, count, lens = sketch(genomes, k, s)
    assert (count == s).all()
    c, d, dist, p = mash.dist(rows, count, rows, count, k, lens, lens)
    T = len(rates) + 1
    for sp in range(P):
        for t, rate in enumerate(rates):
            a = (1 - rate) ** k
            j = a / (2 - a)  # expected Jaccard of the two k-mer sets; then -ln(2j / (1 + j)) / k = -ln(1 - rate)
            sd_j = math.sqrt(j * (1 - j) / s)
            bound = 5 * sd_j / (k * j * (1 + j))  # five binomial spreads of j, carried through dD/dj
            got = dist[sp * T, sp * T + t + 1]
            assert abs(got + math.log(1 - rate)) <= bound, (rate, got, bound)
            assert p[sp * T, sp * T + t + 1] < 1e-100
    # between species only 32-bit chance collisions: about s * G / 2^32 = 0.05 shared values per pair
    species = np.arange(P * T) // T
    other = species[:, None] != species[None, :]
    assert c[other].max() <= 3 and c[other].mean() < 0.2
    assert (dist[other][c[other] == 0] == 1.0).all()


def test_short_group_against_itself(gpu):
    rng = np.random.default_rng(19)
    k, s = 21, 1000
    phage = ACGT[rng.integers(0, 4, size=600)]
    rows, count, lens = sketch([phage, phage.copy()], k, s)
    assert count[0] < s and count[0] == count[1]
    c, d, dist, p = mash.dist(rows, count, rows, count, k, lens, lens)
    assert (dist == 0).all() and (c == count[0]).all() and (d == count[0]).all()
    # the reference's Distance of the same full rows (zero tail) is 1, itself included
    ref = mash.distance_block(rows)[1]
    assert (ref == 1.0).all()


def test_both_strands_canonical(gpu):
    rng = np.random.default_rng(23)
    k, s = 21, 1000
    comp = np.zeros(256, np.uint8)
    comp[ACGT] = np.frombuffer(b"TGCA", np.uint8)
    contigs = [ACGT[rng.integers(0, 4, size=int(n))] for n in rng.integers(5_000, 40_000, size=12)]
    flipped = [comp[c[::-1]] if i % 2 else c for i, c in enumerate(contigs)]
    bases, off = mash.flatten(contigs + flipped)
    goff = np.array([0, 12, 24], np.uint64)
    lens = np.array([sum(map(len, contigs))] * 2, np.uint64)
    rows, count = mash.sketch_groups(bases, off, goff, k, s, canonical=True)
    c, d, dist, p = mash.dist(rows, count, rows, count, k, lens, lens)
    assert (dist == 0).all() and (c == s).all()
    # forward sketches share about the unflipped half of the k-mers: J near 1/3, D near ln(2) / k = 0.033
    fwd, fcount = mash.sketch_groups(bases, off, goff, k, s)
    fc, _, fdist, _ = mash.dist(fwd, fcount, fwd, fcount, k)
    assert fdist[0, 1] > 0.02 and fc[0, 1] < 0.6 * s


def test_cpp_mirror_agrees_with_the_python_mirror(gpu):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "mash_dist_tests"])
    rng = np.random.default_rng(29)
    k, s = 21, 200
    root = ACGT[rng.integers(0, 4, size=30_000)]
    genomes = [root, mutate(rng, root, 0.01), mutate(rng, root, 0.03), ACGT[rng.integers(0, 4, size=30_000)], root[:900]]
    with tempfile.TemporaryDirectory() as tmp:
        txt = os.path.join(tmp, "groups.txt")
        with open(txt, "w") as f:
            for g, seq in enumerate(genomes):
                for piece in (seq[: len(seq) // 2], seq[len(seq) // 2:]):
                    f.write(f"{g} {piece.tobytes().decode()}\n")
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "mash_dist_tests"), txt, str(len(genomes)), str(k), str(s), "0.05"],
                             capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and out.stdout.strip().endswith("ok: mash dist tests pass"), out.stdout + out.stderr
    bases, off = mash.flatten([p for seq in genomes for p in (seq[: len(seq) // 2], seq[len(seq) // 2:])])
    goff = np.arange(0, 2 * len(genomes) + 1, 2, dtype=np.uint64)
    rows, count = mash.sketch_groups(bases, off, goff, k, s)
    lens = np.array([len(g) for g in genomes], np.uint64)
    c, d, dist, p = mash.dist(rows, count, rows, count, k, lens, lens)
    for line in out.stdout.strip().splitlines()[:-1]:
        q, r, cc, dd, dh, ph = line.split()
        q, r = int(q), int(r)
        assert (int(cc), int(dd)) == (c[q, r], d[q, r])
        assert float.fromhex(dh) == dist[q, r] and float.fromhex(ph) == p[q, r]
