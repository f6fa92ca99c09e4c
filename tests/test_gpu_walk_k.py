"""Every walk instantiation (k in WalkKs, kmer_walk.cuh) of the sketch, screen and grouped-sketch kernels against the
oracles, bit for bit, at each k's own chunk and span boundaries.

The walk kernels are templates on K.  The 14 walk k give seven bodies of code, one per NB = k / 4, and each NB has its
own register ring, tail handling (k % 4) and geometry: the span W of a screen or grouped-sketch thread and its chunk of
256 W windows, and the K2t lane segment SEG, its warp chunk of 32 SEG positions and work item of 8 chunks.  A mistake
in one body, or at one k's boundary, shows only at that k, so every test here runs at every walk k, with rows and read
ends placed on that k's boundaries, and checks which launcher took the batch.

The geometry is restated once below; test_walk_geometry_matches_the_sources (CPU tier) checks it against the headers
and kernel sources, so a k added to WalkKs fails there until it is listed here, and is then tested everywhere."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import oracle_ffi
import screen_oracle
import sketch_groups_oracle
from poly_b200 import _lib, mash

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "poly_b200", "csrc")
THREADS = len(os.sched_getaffinity(0))
ACGT = np.frombuffer(b"ACGT", np.uint8)

# ---- the walk geometry, restated ----------------------------------------------------------------------------------
WALK_KS = (11, 13, 15, 16, 17, 19, 21, 23, 24, 25, 27, 29, 31, 32)
# k: (NB, W = walk_span(NB), K2t SEG = SeltGeom<K>::SEG)
GEOM = {11: (2, 64, 68), 13: (3, 60, 84), 15: (3, 60, 84), 16: (4, 64, 68), 17: (4, 64, 68), 19: (4, 64, 68), 21: (5, 60, 60),
        23: (5, 60, 60), 24: (6, 48, 84), 25: (6, 48, 84), 27: (6, 48, 84), 29: (7, 56, 84), 31: (7, 56, 84), 32: (8, 64, 84)}
SCREEN_THREADS = 256      # mash_screen.cu: threads of screen_walk_kernel, one span each
GS_THREADS = 256          # sketch_groups.cu: threads of groups_walk_kernel
SELT_ITEM_CHUNKS = 8      # sketch_select.cu: warp chunks per K2t work item
SELW_SEG = 20             # sketch_smem.cuh: K2w positions per lane segment, the same for every k
# launches of one grouped-sketch call: 2 of set-up, then walk, collect and append per pass
GS_SETUP_LAUNCHES, GS_PASS_LAUNCHES = 2, 3


def span(k):
    """W: windows per thread of the screen and grouped-sketch walks"""
    return GEOM[k][1]


def walk_chunk(k):
    """bytes of one CTA chunk of the screen / grouped-sketch walk"""
    return SCREEN_THREADS * span(k)


def selt_chunk(k):
    """K2t: positions of one warp chunk, 32 lane segments"""
    return 32 * GEOM[k][2]


def selt_item(k):
    """K2t: positions of one work item"""
    return SELT_ITEM_CHUNKS * selt_chunk(k)


def selt_mu(s):
    """K2t: the expected admissions per row, s + 6 sqrt(s) + 48; RARE when mu x 512 < the longest row's windows"""
    return s + 6 * math.ceil(math.sqrt(s)) + 48


GEOMETRY_PROGRAM = r"""
#include <cstdio>
#include "kmer_walk.cuh"
#include "walk_chunk.cuh"
#include "sketch_smem.cuh"
using namespace pg;

int main() {
    std::printf("ks");
    for (int k = -4; k <= 2048; ++k)
        with_walk_k(k, [&](auto kk) { std::printf(" %d", decltype(kk)::value); });
    std::printf("\n");
    for (int k = 0; k <= 64; ++k)
        with_walk_k(k, [&](auto kk) {
            constexpr int K = decltype(kk)::value;
            std::printf("k %d %u %d %d\n", K, walk_span(K / 4), SeltGeom<K>::SEG, SeltGeom<K>::CHUNK);
        });
    std::printf("selw_seg %d\n", SELW_SEG);
    return 0;
}
"""


def nvcc():
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    pytest.fail("nvcc not found: the walk geometry is checked by compiling its headers")


def test_walk_geometry_matches_the_sources(tmp_path):
    """CPU tier: the restated k list and per-k geometry against the headers (compiled on the host), and the launch
    constants that live in the kernel sources."""
    src = tmp_path / "geometry.cu"
    src.write_text(GEOMETRY_PROGRAM)
    exe = tmp_path / "geometry"
    subprocess.run([nvcc(), "-std=c++17", "-O1", "--expt-relaxed-constexpr", "-gencode", "arch=compute_90a,code=sm_90a", "-I", CSRC, str(src),
                    "-o", str(exe)], check=True, capture_output=True, text=True)
    out = subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines()
    assert tuple(int(x) for x in out[0].split()[1:]) == WALK_KS
    got = {int(f[1]): (int(f[2]), int(f[3]), int(f[4])) for f in (line.split() for line in out if line.startswith("k "))}
    assert got == {k: (span(k), GEOM[k][2], selt_chunk(k)) for k in WALK_KS}
    assert all(GEOM[k][0] == k // 4 for k in WALK_KS)
    assert out[-1] == f"selw_seg {SELW_SEG}"

    def source(name):
        with open(os.path.join(CSRC, name)) as f:
            return f.read()

    assert re.search(r"constexpr int SCREEN_THREADS = (\d+);", source("mash_screen.cu")).group(1) == str(SCREEN_THREADS)
    assert re.search(r"constexpr int GS_THREADS = (\d+);", source("sketch_groups.cu")).group(1) == str(GS_THREADS)
    select = source("sketch_select.cu")
    assert re.search(r"constexpr int SELT_ITEM_CHUNKS = (\d+);", select).group(1) == str(SELT_ITEM_CHUNKS)
    mu = re.search(r"const uint32_t mu = \(uint32_t\)s \+ (\d+)u \* \(uint32_t\)ceil\(sqrt\(\(double\)s\)\) \+ (\d+)u;", select)
    assert mu and (int(mu.group(1)), int(mu.group(2))) == (6, 48)
    assert re.search(r"const bool rare = \(uint64_t\)mu \* (\d+) < nmax;", select).group(1) == "512"


# ---- helpers ------------------------------------------------------------------------------------------------------
def rand_bases(rng, n):
    return ACGT[rng.integers(0, 4, n)]


def ragged_of(lens, rng, arbitrary_every=0):
    """(bases, offsets) of random ACGT rows of the given lengths; every arbitrary_every-th row holds arbitrary bytes"""
    lens = np.asarray(lens, np.int64)
    off = np.zeros(len(lens) + 1, np.uint64)
    off[1:] = np.cumsum(lens)
    bases = rand_bases(rng, int(off[-1]))
    if arbitrary_every:
        for i in range(0, len(lens), arbitrary_every):
            bases[int(off[i]):int(off[i + 1])] = rng.integers(0, 256, int(lens[i]), dtype=np.uint8)
    return bases, off


def sm_count():
    sms = C.c_int(0)
    _lib.check(_lib.lib().pg_device_sm_count(C.byref(sms)))
    return sms.value


class Launches:
    """The kernel launches of the calls made inside the block (pg_launch_count) and the last one's name."""

    def __enter__(self):
        self.before = _lib.lib().pg_launch_count()
        return self

    def __exit__(self, *exc):
        self.count = _lib.lib().pg_launch_count() - self.before
        self.last = _lib.lib().pg_last_kernel().decode()


def sketch_batch_dev(bases, off, k, s, pad_zero=False):
    """One pg_mash_sketch_batch_dev call over the whole batch, into dirty buffers: (out, count, status, launches)."""
    import torch

    dev = torch.device("cuda", 0)
    n = len(off) - 1
    maxlen = int(np.diff(off.astype(np.int64)).max())
    stride = s if pad_zero else max(min(max(maxlen - k, 0), s), 1)
    d_bases = torch.from_numpy(bases if len(bases) else np.zeros(1, np.uint8)).to(dev)
    d_off = torch.from_numpy(off.astype(np.int64)).to(dev)
    d_out = torch.full((n, stride), -1, dtype=torch.int32, device=dev)
    d_count = torch.full((n,), -1, dtype=torch.int32, device=dev)
    d_status = torch.full((n,), -1, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    with Launches() as la:
        rc = _lib.lib().pg_mash_sketch_batch_dev(d_bases.data_ptr(), d_off.data_ptr(), n, maxlen, k, s, _lib.PG_SKETCH_PAD_ZERO if pad_zero else 0,
                                                 d_out.data_ptr(), stride, d_count.data_ptr(), d_status.data_ptr(), st)
    _lib.check(rc)
    torch.cuda.synchronize(dev)
    return d_out.cpu().numpy().view(np.uint32), d_count.cpu().numpy().view(np.uint32), d_status.cpu().numpy(), la


def sketch_uniform_dev(reads, k, s):
    """One pg_mash_sketch_uniform_dev call over the [n, L] reads (select regime), into a dirty buffer: (out, launches)."""
    import torch

    dev = torch.device("cuda", 0)
    n, L = reads.shape
    d_in = torch.from_numpy(np.ascontiguousarray(reads).reshape(-1)).to(dev)
    d_out = torch.full((n, s), -1, dtype=torch.int32, device=dev)
    d_status = torch.full((n,), -1, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    with Launches() as la:
        rc = _lib.lib().pg_mash_sketch_uniform_dev(d_in.data_ptr(), n, L, k, s, 0, d_out.data_ptr(), s, d_status.data_ptr(), st)
    _lib.check(rc)
    torch.cuda.synchronize(dev)
    assert not d_status.cpu().numpy().any()
    return d_out.cpu().numpy().view(np.uint32), la


def oracle_rows(bases, off, k, s):
    rc, want = oracle_ffi.sketch_batch(bases, off, k, s, variant=1, nthreads=THREADS)
    assert rc == oracle_ffi.PO_OK
    return want


def oracle_bottom_s_long(row, k, s, piece=1 << 20):
    """The oracle's bottom-s of one long row, computed in pieces of at least `piece` windows on every host thread:
    the pieces partition the row's windows (each piece holds its windows' bytes, k - 1 of them shared with the next), so
    the row's bottom-s multiset is the bottom-s of the pieces' bottom-s."""
    n = len(row) - k
    cuts = list(range(0, n - piece + 1, piece)) if n >= 2 * piece else [0]
    cuts.append(n)
    parts = [row[a:b + k] for a, b in zip(cuts[:-1], cuts[1:])]
    off = np.zeros(len(parts) + 1, np.uint64)
    off[1:] = np.cumsum([len(p) for p in parts])
    low = oracle_rows(np.concatenate(parts), off, k, s)
    return np.sort(low.reshape(-1))[:s]


# ---- K1r: ragged fill-regime batches ------------------------------------------------------------------------------
def k1r_lens(rng, k, s, widest, tiles, tail):
    """32 x tiles rows for K1r, every edge among them, then `tail` (< 32) rows for the generic kernel."""
    nb = k // 4
    edge = [0, k - 1, k, k + 1, k + 2, k + 3, k + 4, widest + k, widest + k - 1, widest + k - 2, widest + k - 3]
    edge += [4 * nb * j + r + k for j in (1, 2, 5) for r in (-1, 0, 1, 2, 3) if 4 * nb * j + r < widest]
    head = np.concatenate([edge, rng.integers(0, widest + k + 1, 32 * tiles - len(edge))])
    rng.shuffle(head)
    return np.concatenate([head, rng.integers(0, widest + k + 1, tail)])


@pytest.mark.gpu
@pytest.mark.parametrize("k", WALK_KS)
def test_k1r_ragged_fill_every_k(gpu, k):
    """K1r (sketch_fill_ragged_kernel): compact rows at s = 1000 up to the widest row K1r stages (768 windows: its
    output tile is at most 96 KiB), and PG_SKETCH_PAD_ZERO rows at s = 256 up to s + k - 1 bytes, the widest fill
    row.  Each batch runs twice: its whole tiles alone (K1r only), then with a last tile of fewer than 32 reads, which
    the generic fill kernel takes."""
    rng = np.random.default_rng(k)
    for s, widest, pad in ((1000, 768, False), (256, 255, True)):
        lens = k1r_lens(rng, k, s, widest, tiles=20, tail=13)
        bases, off = ragged_of(lens, rng, arbitrary_every=7)
        want = oracle_rows(bases, off, k, s)
        for n, kernels, last in ((32 * 20, 1, "sketch_fill_ragged_kernel"), (len(lens), 2, "sketch_fill_generic_kernel")):
            sub = off[:n + 1]
            out, count, status, la = sketch_batch_dev(bases[:int(sub[-1])], sub, k, s, pad_zero=pad)
            assert (la.count, la.last) == (kernels, last), (k, s, n)
            assert out.shape[1] == (s if pad else widest)
            assert not status.any()
            assert np.array_equal(count, np.minimum(np.maximum(lens[:n] - k, 0), s))
            bad = np.nonzero((out != want[:n, :out.shape[1]]).any(axis=1))[0]
            assert not len(bad), (k, s, pad, n, bad[:5], lens[bad[:5]])


# ---- K2t: the threshold walk --------------------------------------------------------------------------------------
def k2t_windows(k, s, rare):
    """Window counts n = L - k on k's K2t boundaries: every window a candidate (n = s + 1, T = 2^32), n ~ 1.3 s, the
    last partial chunk (n at one and two chunks, -1 .. +3), one item +- 1, several items; RARE: one row past mu x 512."""
    ch, item = selt_chunk(k), selt_item(k)
    ns = [s + 1, (13 * s + 9) // 10] + [j * ch + d for j in (1, 2) for d in (-1, 0, 1, 3)] + [item - 1, item, item + 1, 3 * item + 5]
    if rare:
        ns.append(max(4 * item + 1, selt_mu(s) * 512 + 1))
    return ns


def with_retry_rows(rng, lens, k):
    """The rows of `lens` (random ACGT), and two rows K2t hands to K2w through its retry list: a homopolymer (one
    distinct window) and a period-3 row (three)."""
    rows = [rand_bases(rng, L) for L in lens]
    rows.insert(1, np.full(5000 + k, ord("A"), np.uint8))
    rows.insert(4, np.frombuffer((b"ACG" * 3000)[:7000 + k], np.uint8).copy())
    return rows


@pytest.mark.gpu
@pytest.mark.parametrize("k", WALK_KS)
def test_k2t_ragged_every_k(gpu, k, monkeypatch):
    """K2t (sketch_thresh_walk_kernel<K, RARE>) on ragged select-regime batches, in launch groups of 3 rows: s = 1000
    without RARE, and s = 16 (mu = 88) with a row long enough for RARE.  Fill-regime and empty rows between."""
    monkeypatch.setenv("PG_K2T_GROUP_ROWS", "3")
    rng = np.random.default_rng(100 + k)
    for s, rare in ((1000, False), (16, True)):
        ns = k2t_windows(k, s, rare)
        assert (selt_mu(s) * 512 < max(ns)) == rare
        rows = with_retry_rows(rng, [n + k for n in ns], k) + [np.zeros(0, np.uint8), rand_bases(rng, k), rand_bases(rng, k + s // 2)]
        rng.shuffle(rows)
        bases, off = mash.flatten(rows)
        out, count, status, la = sketch_batch_dev(bases, off, k, s)
        # the fill kernel, then walk + select per group of 3 rows, then K2w over the retry list
        assert (la.count, la.last) == (1 + 2 * -(-len(rows) // 3) + 1, "sketch_select_walk_kernel"), (k, s)
        want = oracle_rows(bases, off, k, s)
        lens = np.array([len(r) for r in rows])
        assert not status.any() and np.array_equal(count, np.minimum(np.maximum(lens - k, 0), s))
        bad = np.nonzero((out != want).any(axis=1))[0]
        assert not len(bad), (k, s, lens[bad] - k)


@pytest.mark.gpu
@pytest.mark.parametrize("k", WALK_KS)
def test_k2t_uniform_every_k(gpu, k, monkeypatch):
    """K2t on fixed-length batches (the threshold computed once on the host), 5 rows each with a homopolymer and a
    period-3 row, in launch groups of 3 rows: at n = s + 1, one chunk - 1, one item + 1 (s = 1000), and RARE (s = 16)."""
    monkeypatch.setenv("PG_K2T_GROUP_ROWS", "3")
    rng = np.random.default_rng(200 + k)
    item = selt_item(k)
    for s, n in ((1000, 1001), (1000, selt_chunk(k) - 1), (1000, item + 1), (16, 4 * item + 1)):
        L = n + k
        reads = rand_bases(rng, 5 * L).reshape(5, L)
        reads[1] = ord("A")
        reads[2] = np.frombuffer((b"ACG" * (L // 3 + 1))[:L], np.uint8)
        out, la = sketch_uniform_dev(reads, k, s)
        assert (la.count, la.last) == (2 * 2 + 1, "sketch_select_walk_kernel"), (k, s, n)
        want = oracle_rows(reads.reshape(-1), np.arange(6, dtype=np.uint64) * np.uint64(L), k, s)
        bad = np.nonzero((out != want).any(axis=1))[0]
        assert not len(bad), (k, s, n, bad)


# ---- K2w: the streaming select walk -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", WALK_KS)
def test_k2w_direct_every_k(gpu, k):
    """K2w (sketch_select_walk_kernel) as the main path on random content: a ragged batch K2t declines (rows x work
    items of its longest row > 4 Mi) with too many rows to slice (> 4 x 3 x SMs), so every select-regime row goes to
    K2w directly: 20 000 fill-regime or empty rows, 30 select-regime rows and one row of just enough items."""
    rng = np.random.default_rng(300 + k)
    s = 1000
    n_rows = 20_031
    items = (4 << 20) // n_rows + 1
    lens = np.concatenate([rng.integers(0, s + k, n_rows - 31), rng.integers(2_000, 20_000, 30), [(items - 1) * selt_item(k) + 5 + k]])
    rng.shuffle(lens)
    assert n_rows > 4 * 3 * sm_count() and n_rows * items > 4 << 20
    bases, off = ragged_of(lens, rng)
    out, count, status, la = sketch_batch_dev(bases, off, k, s)
    assert (la.count, la.last) == (2, "sketch_select_walk_kernel")  # the fill kernel, then K2w
    assert not status.any() and np.array_equal(count, np.minimum(np.maximum(lens - k, 0), s))
    want = oracle_rows(bases, off, k, s)
    bad = np.nonzero((out != want).any(axis=1))[0]
    assert not len(bad), (k, lens[bad[:5]])


@pytest.mark.gpu
@pytest.mark.parametrize("k", WALK_KS)
def test_k2w_sketch_size_one_every_k(gpu, k):
    """s = 1 always goes to K2w: Sketches[0] is the first window's hash, and the reference panics (status
    PG_ITEM_PANIC) when a later window hashes below it.  Rows of 1 .. 6 windows panic or not about evenly."""
    rng = np.random.default_rng(400 + k)
    lens = np.concatenate([rng.integers(k - 2, k + 7, 300), rng.integers(200, 3_000, 20)])
    rng.shuffle(lens)
    bases, off = ragged_of(lens, rng)
    out, count, status, la = sketch_batch_dev(bases, off, k, 1)
    assert (la.count, la.last) == (2, "sketch_select_walk_kernel")
    seen = set()
    for i, L in enumerate(lens):
        o = oracle_ffi.OracleMash(k, 1)
        rc = o.Sketch(bases[int(off[i]):int(off[i + 1])].tobytes(), faithful=False)
        panic = rc != oracle_ffi.PO_OK
        seen.add(panic)
        assert status[i] == (_lib.PG_ITEM_PANIC if panic else _lib.PG_ITEM_OK), (k, i, int(L))
        if not panic:
            assert count[i] == min(max(int(L) - k, 0), 1) and out[i, 0] == o.Sketches[0], (k, i, int(L))
    assert seen == {False, True}


@pytest.mark.gpu
@pytest.mark.parametrize("k", WALK_KS)
def test_k2w_sliced_every_k(gpu, k):
    """K2w on slices of one long row, merged by select_merge_kernel: 4 x 3 x SMs - 1 rows, fewer than 3 x SMs of them
    in the select regime, and one row of just enough K2t items to be declined (about 41 to 57 Mbp with 132 SMs)."""
    rng = np.random.default_rng(500 + k)
    s = 1000
    sms = sm_count()
    n_rows = 4 * 3 * sms - 1
    items = (4 << 20) // n_rows + 1
    long_len = (items - 1) * selt_item(k) + 1 + k
    lens = np.concatenate([[long_len], rng.integers(2_000, 60_000, 10), rng.integers(0, s + k, n_rows - 11)])
    rng.shuffle(lens)
    assert (lens - k >= s).sum() < 3 * sms
    bases, off = ragged_of(lens, rng)
    out, count, status, la = sketch_batch_dev(bases, off, k, s)
    assert (la.count, la.last) == (3, "select_merge_kernel")  # the fill kernel, K2w over the slices, the merge
    assert not status.any() and np.array_equal(count, np.minimum(np.maximum(lens - k, 0), s))
    at = int(np.nonzero(lens == long_len)[0][0])
    short = np.delete(np.arange(n_rows), at)
    keep = np.concatenate([bases[int(off[i]):int(off[i + 1])] for i in short])
    koff = np.zeros(len(short) + 1, np.uint64)
    koff[1:] = np.cumsum(lens[short])
    want = oracle_rows(keep, koff, k, s)
    assert np.array_equal(out[short], want)
    assert np.array_equal(out[at], oracle_bottom_s_long(bases[int(off[at]):int(off[at + 1])], k, s))


# ---- the screen's add ---------------------------------------------------------------------------------------------
def screen_pool(k, rng):
    """(bases, offsets) of a pool whose read ends, counted from its first byte, sit at multiples of W and of the chunk
    256 W, each -1, 0, +1, k - 1, k, k + 1; then reads of length k, 0 and k + 1 and a last one of 500 bytes."""
    W, CH = span(k), walk_chunk(k)
    marks = [m * W for m in (1, 2, 3, 7, 31, 64, 127, 200, 255)] + [c * CH for c in (1, 2, 3)] + \
            [CH + m * W for m in (1, 100, 254)] + [2 * CH + 128 * W, 3 * CH + 40 * W]
    ends = sorted({b + d for b in marks for d in (-1, 0, 1, k - 1, k, k + 1)})
    t = ends[-1]
    ends += [t + k, t + k, t + 2 * k + 1, t + 2 * k + 501]
    off = np.array([0] + ends, np.uint64)
    return rand_bases(rng, int(off[-1])), off


def witness_and_refs(bases, k, rng):
    """Reference rows of one width: the witness (every window hash of the pool's bytes taken as one record, windows
    across read ends included), the bottom-200 sketch of that record and 200 random words, both padded with zeros."""
    whole = np.array([0, len(bases)], np.uint64)
    wit = screen_oracle.pool_hashes(bases, whole, k)
    rows = np.zeros((3, len(wit)), np.uint32)
    rows[0] = wit
    rows[1, :200] = oracle_rows(bases, whole, k, 200)[0]
    rows[2, :200] = rng.integers(0, 1 << 32, 200, dtype=np.uint64).astype(np.uint32)
    return rows


def assert_same(got, want):
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.tobytes() == w.tobytes(), (g, w)


@pytest.mark.gpu
@pytest.mark.parametrize("k", WALK_KS)
def test_screen_add_every_k(gpu, k):
    """screen_walk_kernel<K, false> (one sample, host add, then add_dev from a base 1 .. 15 bytes past a 16-byte
    boundary: every chunk head) and <K, true> (3 samples, per-read ids), against screen_oracle.  The witness row's
    vmax is near 2^32, so every window reaches the lookup, and its shared is exactly the pool's window count: a dropped
    window lowers it, a window counted across a read end (or Mash's excluded last window) raises it."""
    import torch

    rng = np.random.default_rng(600 + k)
    bases, off = screen_pool(k, rng)
    lens = np.diff(off.astype(np.int64))
    assert {0, k, k + 1} <= set(lens.tolist())
    sk = witness_and_refs(bases, k, rng)
    want = screen_oracle.mash_screen(sk, (bases, off), k, nthreads=THREADS)
    assert want[0][0] == np.maximum(lens - k, 0).sum()
    with mash.Screen(sk, k) as sc:
        with Launches() as la:
            sc.add((bases, off))
        assert (la.count, la.last) == (1, "screen_walk_kernel")
        assert_same(sc.results(), want)
        dev = torch.device("cuda", 0)
        buf = torch.zeros(16 + len(bases), dtype=torch.uint8, device=dev)
        for head in range(1, 16):
            sc.reset()
            buf[head:head + len(bases)] = torch.from_numpy(bases).to(dev)
            d_off = torch.from_numpy(off.astype(np.int64) + head).to(dev)
            assert (buf.data_ptr() + head) % 16 == head
            with Launches() as la:
                sc.add_dev(buf, d_off)
            assert (la.count, la.last) == (1, "screen_walk_kernel")
            assert_same(sc.results(), want)
    ids = rng.integers(0, 3, len(lens)).astype(np.uint32)
    with mash.Screen(sk, k, samples=3) as sc:
        with Launches() as la:
            sc.add((bases, off), sample=ids)
        assert (la.count, la.last) == (1, "screen_walk_kernel")
        table = sc.results_samples()
    for q in range(3):
        reads = [bases[int(off[i]):int(off[i + 1])] for i in np.nonzero(ids == q)[0]]
        w = screen_oracle.mash_screen(sk, mash.flatten(reads), k, nthreads=THREADS)
        assert w[0][0] == np.maximum(lens[ids == q] - k, 0).sum()
        assert_same([x[q] for x in table], w)


# ---- the grouped sketch -------------------------------------------------------------------------------------------
def group_layout(k, rng):
    """(bases, record offsets, group offsets): group byte boundaries at multiples of W and of 256 W, each -1, 0, +1, so
    that threads see one group (an exact range compare) or several (the forward cursor); an empty group after every
    fifth; groups longer than 2k + 2 bytes are two records, the second opening with a copy of part of the first."""
    W, CH = span(k), walk_chunk(k)
    marks = [m * W for m in (1, 2, 5, 9, 30, 64, 65, 130, 255)] + [c * CH for c in (1, 2, 3)] + [CH + 77 * W, 2 * CH + 200 * W, 3 * CH + 90 * W]
    bounds = [0] + sorted({b + d for b in marks for d in (-1, 0, 1)})
    bases = rand_bases(rng, bounds[-1])
    rec, goff = [0], [0]
    for g, (a, b) in enumerate(zip(bounds[:-1], bounds[1:])):
        if g % 5 == 4:
            goff.append(goff[-1])  # an empty group
        if b - a > 2 * k + 2:
            cut = a + (b - a) // 2
            dup = (cut - a) // 3
            bases[cut:cut + dup] = bases[a:a + dup]
            rec.append(cut)
        rec.append(b)
        goff.append(len(rec) - 1)
    return bases, np.array(rec, np.uint64), np.array(goff, np.uint64)


@pytest.mark.gpu
@pytest.mark.parametrize("k", WALK_KS)
def test_sketch_groups_every_k(gpu, k):
    """groups_walk_kernel<K> against sketch_groups_oracle.  With s above every group's window count each row is all of
    the group's distinct window hashes (m = 1), or all that occur twice (m = 2), in one pass, so any window error shows;
    s = 16 at m = 2 needs later passes, which walk only the spans of the groups still open."""
    rng = np.random.default_rng(700 + k)
    bases, off, goff = group_layout(k, rng)
    wide = 2 * int(np.diff(off.astype(np.int64)).max())  # above every group's window count
    for s, m, one_pass in ((wide, 1, True), (wide, 2, True), (16, 2, False)):
        with Launches() as la:
            got = mash.sketch_groups(bases, off, goff, k, s, m)
        want = sketch_groups_oracle.sketch_groups(bases, off, goff, k, s, m, THREADS)
        if one_pass:
            assert (la.count, la.last) == (GS_SETUP_LAUNCHES + GS_PASS_LAUNCHES, "groups_append_kernel"), (k, s, m)
            assert want[1].max() > 0
        else:
            assert la.count > GS_SETUP_LAUNCHES + GS_PASS_LAUNCHES, (k, la.count)
        assert got[1].tobytes() == want[1].tobytes(), (k, s, m, got[1], want[1])
        assert got[0].tobytes() == want[0].tobytes(), (k, s, m)
