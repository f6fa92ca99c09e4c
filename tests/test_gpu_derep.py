"""pg_mash_dereplicate on the GPU against the dereplication oracle: assignments element for element in both
modes, and the representative count."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import derep_oracle
import oracle_ffi
from poly_b200 import _lib, mash, sketchfile, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def sketches_of(reads, n, L, k, s):
    rc, sk = oracle_ffi.sketch_batch(reads, synth.uniform_offsets(n, L), k, s, variant=1, nthreads=len(os.sched_getaffinity(0)))
    assert rc == 0
    return sk


def check_against_oracle(sk, min_same):
    """Both modes against the oracle; returns the two assignments."""
    out = []
    links = derep_oracle.links_of(sk, min_same)  # one scan of the pairs for both modes
    for nearest in (False, True):
        want = derep_oracle.dereplicate_pairs(*links, len(sk), min_same, nearest)
        rep, n_reps = mash.dereplicate(sk, min_same=min_same, nearest=nearest)
        assert rep.dtype == np.uint32 and np.array_equal(rep, want[0]), (min_same, nearest)
        assert n_reps == want[1]
        out.append(rep)
    assert np.array_equal(out[0] == np.arange(len(sk)), out[1] == np.arange(len(sk)))  # the same representatives
    return out


@pytest.fixture(scope="module")
def family(gpu):
    """2 048 family reads of 2 kbp, 16 per family, k = 21, s = 400: members share 137..273 hashes."""
    n, L, k, s = 2048, 2000, 21, 400
    return sketches_of(synth.family_reads(n, L, family=16), n, L, k, s)


def test_family_reads_at_several_cuts(family):
    differ = 0
    for min_same in (1, 100, 200, 400):
        first, near = check_against_oracle(family, min_same)
        differ += not np.array_equal(first, near)
    first, _ = check_against_oracle(family, 100)  # below every in-family count: the first member represents
    assert np.array_equal(first, np.arange(len(family)) // 16 * 16)
    assert differ > 0


def test_identical_sketches(family):
    sk = family[:512].copy()
    sk[[7, 100, 511]] = sk[3]
    sk[300] = sk[20]
    for min_same in (400, 150):
        check_against_oracle(sk, min_same)
    for nearest in (False, True):
        rep, n_reps = mash.dereplicate(sk, min_same=400, nearest=nearest)
        want = np.arange(512, dtype=np.uint32)
        want[[7, 100, 511]] = 3
        want[300] = 20
        assert np.array_equal(rep, want) and n_reps == 508


def test_unsorted_regime_every_sketch_represents_itself(gpu):
    """150 bp reads, k = 21, s = 1000: the literal Similarity walk counts 0 for every pair."""
    n, L, k, s = 512, 150, 21, 1000
    sk = sketches_of(synth.independent_reads(n, L), n, L, k, s)
    for rep in check_against_oracle(sk, 1):
        assert np.array_equal(rep, np.arange(n))


def test_row_length_not_a_multiple_of_four(family):
    for n in (2045, 2046, 2047, 5, 1):
        check_against_oracle(family[:n], 150)


def test_chain_in_two_row_tiles(gpu):
    """49 152 sketches, sketch i = 8 i ... 8 i + 15 (s = 16): neighbours share 8 values and nothing else links, so
    the even indices are the representatives.  The dense pass runs in two row tiles, and every sub-block boundary
    and the tile cut sit inside a link."""
    n = 49152
    rows_per = ((2 << 30) // n) & ~7  # distance_tile_rows
    assert 0 < rows_per < n
    sk = (np.arange(n, dtype=np.uint32)[:, None] * 8 + np.arange(16, dtype=np.uint32)).astype(np.uint32)
    want = np.arange(n, dtype=np.uint32)
    want -= want % 2
    for nearest in (False, True):
        rep, n_reps = mash.dereplicate(sk, min_same=8, nearest=nearest)
        assert np.array_equal(rep, want) and n_reps == n // 2
    check_against_oracle(sk, 8)


def test_families_across_the_tile_cut(gpu):
    n, L, k, s, min_same = 49152, 80, 21, 16, 4
    rows_per = ((2 << 30) // n) & ~7
    assert rows_per % 16 != 0  # a family straddles the cut
    sk = sketches_of(synth.family_reads(n, L, family=16), n, L, k, s)
    first, _ = check_against_oracle(sk, min_same)
    fam = rows_per // 16 * 16
    assert (first[rows_per: fam + 16] < rows_per).any()  # members after the cut assigned to one before it


def test_device_path_equals_host_path(family):
    import torch

    d_sk = torch.from_numpy(family.view(np.int32)).cuda()
    st = torch.cuda.current_stream().cuda_stream
    for min_same in (100, 200, 400):
        for nearest in (False, True):
            want = mash.dereplicate(family, min_same=min_same, nearest=nearest)
            rep, n_reps = mash.dereplicate(d_sk, min_same=min_same, nearest=nearest)
            assert rep.is_cuda and rep.dtype == torch.int32 and n_reps.dim() == 0
            assert np.array_equal(rep.cpu().numpy().view(np.uint32), want[0]) and int(n_reps) == want[1]
    # the count is optional on both paths
    for flags in (0, mash.PG_DEREP_NEAREST):
        want = mash.dereplicate(family, min_same=150, nearest=bool(flags))[0]
        rep = torch.empty(len(family), dtype=torch.int32, device="cuda")
        _lib.check(_lib.lib().pg_mash_dereplicate_dev(d_sk.data_ptr(), len(family), 400, 150, flags, rep.data_ptr(), None, st))
        assert np.array_equal(rep.cpu().numpy().view(np.uint32), want)
        host = np.zeros(len(family), np.uint32)
        _lib.check(_lib.lib().pg_mash_dereplicate(family.ctypes.data, len(family), 400, 150, flags, host.ctypes.data, None))
        assert np.array_equal(host, want)
    rep, n_reps = mash.dereplicate(d_sk, max_distance=-1.0)  # nothing can link: no launch
    assert rep.is_cuda and rep.cpu().tolist() == list(range(len(family))) and int(n_reps) == len(family)


def test_empty_set_and_argument_errors(family):
    L = _lib.lib()
    for nearest in (False, True):
        rep, n_reps = mash.dereplicate(np.zeros((0, 400), np.uint32), min_same=1, nearest=nearest)
        assert (len(rep), n_reps) == (0, 0)
    sk = family[:32]
    rep = np.zeros(32, np.uint32)
    nr = C.c_uint64(9)
    assert L.pg_mash_dereplicate(None, 0, 400, 1, 0, None, C.byref(nr)) == _lib.PG_OK and nr.value == 0
    # an unknown flag bit comes first: before the count limit, the empty set, the sketch size and min_same
    for n, s, min_same in ((32, 400, 100), (1 << 32, 400, 1), (0, 400, 1), (32, 0, 1), (32, 400, 0)):
        nr.value = 9
        assert L.pg_mash_dereplicate(sk.ctypes.data, n, s, min_same, 2, rep.ctypes.data, C.byref(nr)) == _lib.PG_ERR_ARG
        assert "flags" in _lib.last_error() and nr.value == 0
    assert L.pg_mash_dereplicate(None, 1 << 32, 0, 0, 1, None, None) == _lib.PG_ERR_ARG  # count limit before s
    assert L.pg_mash_dereplicate(sk.ctypes.data, 32, 0, 0, 1, rep.ctypes.data, None) == _lib.PG_ERR_PANIC  # s before min_same
    for flags in (0, 1):
        for bad in (0, 401):
            nr.value = 9
            assert L.pg_mash_dereplicate(sk.ctypes.data, 32, 400, bad, flags, rep.ctypes.data, C.byref(nr)) == _lib.PG_ERR_ARG
            assert "min_same" in _lib.last_error() and nr.value == 0
            with pytest.raises(_lib.PolyError) as e:
                mash.dereplicate(sk, min_same=bad, nearest=bool(flags))
            assert e.value.code == _lib.PG_ERR_ARG
    with pytest.raises(_lib.GoPanic):
        mash.dereplicate(np.zeros((3, 0), np.uint32), min_same=1)
    with pytest.raises(_lib.GoPanic):
        mash.dereplicate(np.zeros((3, 0), np.uint32), max_distance=0.5, nearest=True)
    # the device entry point applies the same order and clears its counter
    import torch

    d_cnt = torch.full((), 9, dtype=torch.int64, device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    assert L.pg_mash_dereplicate_dev(None, 0, 400, 1, 2, None, d_cnt.data_ptr(), st) == _lib.PG_ERR_ARG
    assert L.pg_mash_dereplicate_dev(None, 0, 400, 1, 1, None, d_cnt.data_ptr(), st) == _lib.PG_OK and int(d_cnt) == 0


@pytest.mark.parametrize("mode", ["first", "nearest"])
def test_cpp_mirror_agrees_with_the_oracle(family, mode):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "hostcpp"), "-s", "CXX=g++", "derep_tests"])
    sk = family[:512]
    with tempfile.TemporaryDirectory() as td:
        path = os.path.join(td, "set.pgsketch")
        sketchfile.save(path, sk, np.full(len(sk), 400, np.uint32), 21, 400)
        out = subprocess.run([os.path.join(ROOT, "hostcpp", "derep_tests"), path, "200", mode], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = out.stdout.splitlines()
    assert lines[-1] == "ok: derep tests pass"
    rep, n_reps = derep_oracle.dereplicate(sk, 200, mode == "nearest")
    assert lines[0] == f"{n_reps}" and lines[1] == " ".join(str(int(x)) for x in rep)
