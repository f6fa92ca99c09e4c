"""CPU tier: the oracle is one library, oracle/liboracle.so, built by one recipe (oracle/Makefile, run by
oracle_ffi.build()) and loaded through one handle.  What it exports, what oracle/poly_oracle.h declares and
what the Python bindings bind are the same set of functions."""
import ctypes as C
import os
import re
import subprocess
import sys

import numpy as np

import oracle_ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TESTS = os.path.join(ROOT, "tests")
PREFIXES = r"(?:po|co|fo|fr)_"


def declared_symbols():
    text = open(os.path.join(oracle_ffi.ORACLE_DIR, "poly_oracle.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return set(re.findall(rf"\b({PREFIXES}[a-z0-9_]+)\s*\(", text))


def exported_symbols():
    out = subprocess.run(["nm", "-D", "--defined-only", oracle_ffi.build()], check=True, capture_output=True, text=True).stdout
    return {line.split()[-1] for line in out.splitlines()}


def test_declared_bound_and_exported_symbols_agree():
    tables = [__import__(m).SIGS for m in oracle_ffi.BINDINGS]
    bound = set().union(*tables)
    assert sum(len(t) for t in tables) == len(bound), "a function is bound by two modules"
    declared, exported = declared_symbols(), exported_symbols()
    assert len(declared) >= 40
    assert declared == bound, declared ^ bound
    assert exported == declared, exported ^ declared
    assert set(oracle_ffi.signatures()) == bound


def test_one_build_path():
    c_files = [os.path.join(dp, f) for dp, _, fs in os.walk(TESTS) for f in fs if f.endswith(".c")]
    assert not c_files, c_files
    for m in oracle_ffi.BINDINGS:
        src = open(os.path.join(TESTS, m + ".py")).read()
        assert "tempfile" not in src and "mkdtemp" not in src and "gcc" not in src, m
        if m != "oracle_ffi":  # oracle_ffi.build() runs oracle/Makefile
            assert "subprocess" not in src, m


def test_fresh_library_is_not_rebuilt():
    """A cold process that loads every binding finds the library up to date and leaves it alone."""
    so = oracle_ffi.build()
    before = os.stat(so).st_mtime_ns
    code = "import importlib, oracle_ffi\nfor m in oracle_ffi.BINDINGS:\n    importlib.import_module(m).lib()\n"
    subprocess.run([sys.executable, "-c", code], check=True, cwd=TESTS)
    assert os.stat(so).st_mtime_ns == before


def test_worker_pool_result_does_not_depend_on_thread_count():
    """The pooled drivers give the one-thread result on any thread count, more threads than items and an
    empty batch included, with one item per claim (seqhash) and with blocks of items (the pair list)."""
    import pair_oracle
    import seqhash_oracle

    rng = np.random.default_rng(3)
    seqs = [bytes(rng.choice(list(b"ACGTacgtN"), int(rng.integers(0, 300)))) for _ in range(2000)]
    flat, off = oracle_ffi.ragged(seqs)
    lut = np.full(256, -1, np.int16)
    lut[list(b"-ACGT")] = np.arange(5)
    mat = np.array([[0] * 5] + [[0] + [3 if i == j else -3 for j in range(4)] for i in range(4)], np.int64)
    pairs = rng.integers(0, len(seqs), (2000, 2))
    for n in (0, 5, 2000):
        want_h = seqhash_oracle.seqhash_batch(flat, off[: n + 1], "DNA", True, True, 1)
        want_p = pair_oracle.scores(seqs, seqs, pairs[:n], lut, lut, mat, -2, False, 1)
        for threads in (0, 3, 64):
            got_h = seqhash_oracle.seqhash_batch(flat, off[: n + 1], "DNA", True, True, threads)
            got_p = pair_oracle.scores(seqs, seqs, pairs[:n], lut, lut, mat, -2, False, threads)
            assert all(np.array_equal(a, b) for a, b in zip(want_h + want_p, got_h + got_p)), (n, threads)
