"""GPU tier for seqhash: every digest, error code and error position of pg_seqhash_batch(_dev) and every
start of pg_least_rotation_batch compared bit-exact with the C restatement (oracle/seqhash_oracle.c)
or with tests/golden/seqhash_goldens.json."""
import gzip
import json
import os
import random

import numpy as np
import pytest

import oracle_ffi
import seqhash_oracle
from poly_b200 import _lib, seqhash

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDENS = json.load(open(os.path.join(HERE, "golden", "seqhash_goldens.json")))
PUC19 = open(os.path.join(HERE, "golden", "seqhash", "puc19.txt")).read().strip().encode()
FLAGS = [(c, d) for c in (False, True) for d in (False, True)]
COMP = dict(zip(b"ABCDGHKMNRSTVWY", b"TVGHCDMKNYSABWR"))


def rc(s: bytes) -> bytes:
    return bytes(COMP.get(c, 0) for c in reversed(s.upper()))


def check(seqs, t, circular, ds, threads=8):
    """GPU batch == oracle on every item; returns the digests."""
    flat, off, raw = seqhash._flatten(seqs)
    dig, code, pos = seqhash.hash_arrays(flat, off, t, circular, ds)
    want_dig, want_code, want_pos = seqhash_oracle.seqhash_batch(flat, off, t, circular, ds, threads)
    bad = [i for i in range(len(raw)) if code[i] != want_code[i] or pos[i] != want_pos[i] or not np.array_equal(dig[i], want_dig[i])]
    assert not bad, [(i, len(raw[i]), raw[i][:40], int(code[i]), int(want_code[i]), int(pos[i]), int(want_pos[i])) for i in bad[:5]]
    return dig


def test_reference_pins_and_errors(gpu):
    for seq, t, circular, ds, want in GOLDENS["pins"]:
        assert seqhash.Hash(seq, t, circular, ds) == (want, None)
        assert seqhash.HashBatch([seq, seq.lower()], t, circular, ds) == [(want, None)] * 2
    for seq, t, circular, ds, msg in GOLDENS["errors"]:
        h, err = seqhash.Hash(seq, t, circular, ds)
        assert h == "" and str(err) == msg


def test_device_entry_point_pins(gpu):
    import torch

    for seq, t, circular, ds, want in GOLDENS["pins"]:
        d_seq = torch.tensor(list(seq.encode()), dtype=torch.uint8, device="cuda")
        d_off = torch.tensor([0, len(seq)], dtype=torch.int64, device="cuda")
        dig, code, pos = seqhash.hash_device(d_seq, d_off, 1, len(seq), t, circular, ds)
        assert int(code[0]) == 0 and seqhash.format_hash(dig[0].cpu().numpy().tobytes(), t, circular, ds) == want


def test_random_goldens(gpu):
    groups = {}
    for seq, t, circular, ds, want in GOLDENS["random"]:
        groups.setdefault((t, circular, ds), []).append((seq, want))
    assert len(groups) == 10
    for (t, circular, ds), items in groups.items():
        got = seqhash.HashBatch([s for s, _ in items], t, circular, ds)
        assert [h for h, _ in got] == [w for _, w in items], (t, circular, ds)


def _random_batch(rng, letters, n, max_len):
    return ["".join(rng.choice(letters) for _ in range(rng.choice([0, 1, 2, rng.randint(3, max_len)]))) for _ in range(n)]


@pytest.mark.parametrize("t", ["DNA", "RNA", "PROTEIN"])
@pytest.mark.parametrize("circular,ds", FLAGS)
def test_types_and_flags(gpu, t, circular, ds):
    rng = random.Random(f"{t}{circular}{ds}")
    letters = "ACDEFGHIKLMNPQRSTVWYUO*BXZacdefgh" if t == "PROTEIN" else "ACGTTGCAUZNRYacgtu"
    seqs = _random_batch(rng, letters, 300, 3000)
    seqs += ["ACGT" * 300 + "J", "acgt\x00", "AC" * 700 + "\xc5\xbf"]  # bad letters, NUL, non-ASCII
    check([s.encode("latin-1") for s in seqs], t, circular, ds)


def test_chunk_and_tree_boundaries(gpu):
    rng = np.random.default_rng(5)
    lengths = [0, 1, 2, 3, 63, 64, 65, 1023, 1024, 1025]
    for k in range(1, 11):
        lengths += [(1 << k) * 1024 - 1, (1 << k) * 1024, (1 << k) * 1024 + 1]
    seqs = [bytes(rng.choice(np.frombuffer(b"ACGT", np.uint8), size=n)) for n in lengths]
    rng.shuffle(seqs)
    for circular, ds in FLAGS:
        check(seqs, "DNA", circular, ds)


def test_64mi_sequence_mixed_with_tiny_ones(gpu):
    """65,537 chunks: a tree of depth 17, next to single-chunk sequences in the same call."""
    rng = np.random.default_rng(11)
    big = rng.choice(np.frombuffer(b"ACGT", np.uint8), size=(64 << 20) + 1).tobytes()
    seqs = [b"A", big, b"", b"GATTACA" * 200]
    for circular, ds in [(False, False), (False, True)]:
        check(seqs, "DNA", circular, ds, threads=4)


def test_adversarial_rotations(gpu):
    mb = 1 << 20
    half = b"GAATTCAGGCTTA" * 23
    pal = half + rc(half)  # a reverse-complement palindrome
    assert rc(pal) == pal
    seqs = [
        b"A" * mb, b"AC" * (mb // 2), b"ACG" * (mb // 3 + 1), b"AAB"[:2] * 1000 + b"C",
        pal, pal[100:] + pal[:100],  # rc(s) is a rotation of s
        b"ATAT" * 5000, b"GC" * 3, b"AUZ" * 40, b"ZZZZ", b"uuacgZ", b"acgtnnRYkm" * 30, b"T", b"",
    ]
    for circular, ds in FLAGS:
        check(seqs, "DNA", circular, ds, threads=4)
    check([b"ACGU" * 100, b"uuuu", b"UACG" * 333], "RNA", True, True)
    check([b"MGC*" * 50, b"*M*G", b"mkv*" * 1000, b"*"], "PROTEIN", True, False)


def test_error_ordering(gpu):
    seqs = [b"ACGTJACGT", b"ACGT\xc5\xbfJ", b"ACGTJ\xc5\xbf", b"acgT", b"\xff", b"MGCS*", b"MGCJ*", b"MGCS*\x80"]
    for t, (circular, ds) in [("DNA", (True, True)), ("PROTEIN", (False, True)), ("PROTEIN", (True, False))]:
        check(seqs, t, circular, ds)
    dig, code, pos = seqhash.hash_arrays(*seqhash._flatten(seqs)[:2], "PROTEIN", False, True)
    assert code.tolist() == [1, 3, 1, 2, 3, 2, 1, 3] and pos.tolist() == [4, 4, 4, 0, 0, 0, 3, 5]
    assert not dig.any()
    got = seqhash.HashBatch([b"ACGT", b"ACGTX", b"ACGT"], "DNA", False, False)
    assert got[0] == got[2] and got[0][1] is None and str(got[1][1]).endswith("Got letter: X")
    assert isinstance(seqhash.Hash("acſt", "DNA", False, False)[1], seqhash.UnsupportedError)


def test_puc19_rotations_one_batch(gpu):
    n = len(PUC19)
    rots = [PUC19[r:] + PUC19[:r] for r in range(n)]
    got = seqhash.HashBatch(rots, "DNA", True, True)
    want = GOLDENS["puc19_circular_double_stranded"]
    assert want == seqhash_oracle.seqhash_string(PUC19, "DNA", True, True)
    assert all(g == (want, None) for g in got)
    assert {seqhash.RotateSequence(r) for r in rots} == {seqhash_oracle.rotate_sequence(PUC19).decode()}


def test_least_rotation_against_booth(gpu):
    rng = random.Random(3)
    seqs = []
    for alphabet in ("A", "AB", "AAB", "ABC", "ACGT"):
        seqs += ["".join(rng.choice(alphabet) for _ in range(rng.randint(1, 24))).encode() for _ in range(400)]
    seqs += [b"", b"AB" * 50000, b"ABC" * 40000 + b"AB", b"A" * 300000, b"BA" * 3 + b"A", PUC19, PUC19.upper(),
             bytes(np.random.default_rng(1).integers(0, 256, 100000, dtype=np.uint8)),
             b"AAB" * 30 + b"AAAB" + b"AAB" * 30]
    got = seqhash.least_rotations(seqs)
    want = [seqhash_oracle.booth_least_rotation(s) for s in seqs]
    assert got.tolist() == want


def test_device_path_equals_host(gpu):
    import torch

    rng = random.Random(9)
    seqs = [s.encode() for s in _random_batch(rng, "ACGTacgtUZN", 500, 5000)]
    flat, off, _ = seqhash._flatten(seqs)
    for circular, ds in FLAGS:
        dig, code, pos = seqhash.hash_arrays(flat, off, "DNA", circular, ds)
        d_dig, d_code, d_pos = seqhash.hash_device(torch.from_numpy(flat.copy()).cuda(), torch.from_numpy(off.astype(np.int64)).cuda(),
                                                   len(seqs), int(np.diff(off).max()), "DNA", circular, ds)
        torch.cuda.synchronize()
        assert np.array_equal(d_dig.cpu().numpy(), dig) and np.array_equal(d_code.cpu().numpy(), code)
        assert np.array_equal(d_pos.cpu().numpy().astype(np.uint64), pos)


def test_fasta_chain_uniprot(gpu):
    text = gzip.open(os.path.join(HERE, "golden", "fasta", "uniprot_1mb_test_head.fasta.gz")).read()
    dig, code, pos, err = seqhash.hash_fasta_records(text, "PROTEIN", False, False)
    recs, ec, _ = oracle_ffi.fasta_parse(text)
    assert err is None and ec == 0 and len(recs) == len(dig) > 100
    for i, (_, s) in enumerate(recs):
        c, d, p = seqhash_oracle.seqhash(s, "PROTEIN", False, False)
        assert (int(code[i]), int(pos[i])) == (c, p) and dig[i].tobytes() == (d or bytes(32)), i


def test_forced_small_groups(gpu, monkeypatch):
    rng = random.Random(13)
    seqs = [s.encode() for s in _random_batch(rng, "ACGTZ", 200, 6000)] + [b"ACGT" * 5000]
    flat, off, _ = seqhash._flatten(seqs)
    base = [seqhash.hash_arrays(flat, off, "DNA", c, d) for c, d in FLAGS]
    monkeypatch.setenv("PG_GROUP_BYTES", "4096")
    for (c, d), (dig, code, pos) in zip(FLAGS, base):
        g_dig, g_code, g_pos = seqhash.hash_arrays(flat, off, "DNA", c, d)
        assert np.array_equal(g_dig, dig) and np.array_equal(g_code, code) and np.array_equal(g_pos, pos)


def test_argument_errors(gpu):
    L = _lib.lib()
    seq = np.frombuffer(b"ACGT", np.uint8)
    off = np.array([0, 4], np.uint64)
    out = np.zeros(32, np.uint8)
    assert L.pg_seqhash_batch(seq.ctypes.data, off.ctypes.data, 1, 3, 0, out.ctypes.data, None, None) == _lib.PG_ERR_ARG
    assert L.pg_seqhash_batch(seq.ctypes.data, off.ctypes.data, 1, 0, 4, out.ctypes.data, None, None) == _lib.PG_ERR_ARG
    bad = np.array([4, 0], np.uint64)
    assert L.pg_seqhash_batch(seq.ctypes.data, bad.ctypes.data, 1, 0, 0, out.ctypes.data, None, None) == _lib.PG_ERR_ARG
    assert L.pg_seqhash_batch(seq.ctypes.data, off.ctypes.data, 0, 0, 0, out.ctypes.data, None, None) == _lib.PG_OK


def test_cpp_mirror_reference_tests(gpu):
    import subprocess

    root = os.path.dirname(HERE)
    subprocess.check_call(["make", "-C", os.path.join(root, "hostcpp"), "-s", "CXX=g++", "seqhash_tests"])
    out = subprocess.run([os.path.join(root, "hostcpp", "seqhash_tests"), os.path.join(HERE, "golden", "seqhash", "puc19.txt")],
                         capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "ok: seqhash tests pass" in out.stdout, out.stdout + out.stderr
