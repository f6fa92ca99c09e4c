"""CPU tier for seqhash: the C restatement (oracle/seqhash_oracle.c, through tests/seqhash_oracle.py) against the reference's pinned hashes,
independent BLAKE3 digests and a brute-force least rotation; the Python mirror's host-side formatting; and
the new entry points failing loudly without a GPU."""
import ctypes as C
import json
import os
import random

import numpy as np
import pytest

import seqhash_oracle as oracle
from poly_b200 import _lib, seqhash

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDENS = json.load(open(os.path.join(HERE, "golden", "seqhash_goldens.json")))
PUC19 = open(os.path.join(HERE, "golden", "seqhash", "puc19.txt")).read().strip()


def test_oracle_reproduces_reference_pins():
    assert len(GOLDENS["pins"]) == 7
    for seq, t, circular, ds, want in GOLDENS["pins"]:
        assert oracle.seqhash_string(seq, t, circular, ds) == want


def test_oracle_error_cases():
    assert len(GOLDENS["errors"]) == 4
    for seq, t, circular, ds, msg in GOLDENS["errors"]:
        if t not in oracle.TYPES:
            assert msg.startswith("Only sequenceTypes")
            continue
        code, dig, pos = oracle.seqhash(seq, t, circular, ds)
        assert dig is None
        if code == 1:
            assert msg.endswith("Got letter: " + seq[pos].upper())
        else:
            assert (code, msg) == (2, "Proteins cannot be double stranded")


def test_oracle_blake3_vectors():
    assert len(GOLDENS["blake3"]) == 28
    for n, want in GOLDENS["blake3"]:
        assert oracle.blake3(bytes(i % 251 for i in range(n))).hex() == want, n


def test_oracle_random_goldens():
    assert len(GOLDENS["random"]) >= 300
    for seq, t, circular, ds, want in GOLDENS["random"]:
        assert oracle.seqhash_string(seq, t, circular, ds) == want, (seq, t, circular, ds)


def test_oracle_puc19_doc_hash():
    """The package doc's example Seqhash (seqhash.go:46) is pUC19, circular and double-stranded."""
    assert len(PUC19) == 2686
    want = "v1_DCD_4b0616d1b3fc632e42d78521deb38b44fba95cca9fde159e01cd567fa996ceb9"
    assert GOLDENS["puc19_circular_double_stranded"] == want == oracle.seqhash_string(PUC19, "DNA", True, True)


def _brute_least_start(s: bytes) -> int:
    rots = [s[i:] + s[:i] for i in range(len(s))]
    return min(range(len(s)), key=lambda i: (rots[i], i)) if s else 0


def test_oracle_booth_is_smallest_least_rotation():
    rng = random.Random(7)
    for alphabet in ("A", "AB", "AAB", "ABC", "ACGT"):
        for _ in range(1500):
            s = "".join(rng.choice(alphabet) for _ in range(rng.randint(1, 20))).encode()
            assert oracle.booth_least_rotation(s) == _brute_least_start(s), s
    assert oracle.booth_least_rotation(b"") == 0


def test_oracle_least_rotation_puc19():
    """TestLeastRotation (seqhash_test.go:68-91) and ExampleRotateSequence (example_test.go:33-40)."""
    want = oracle.rotate_sequence(PUC19)
    for r in range(len(PUC19)):
        assert oracle.rotate_sequence(PUC19[r:] + PUC19[:r]) == want, r
    half = len(PUC19) // 2
    assert oracle.rotate_sequence(PUC19[half:] + PUC19[:half]) == want


def test_oracle_reverse_complement_quirks():
    """U and Z are DNA letters without a complement: they become NUL bytes, which then win the strand choice."""
    code, dig, _ = oracle.seqhash("AZ", "DNA", False, True)
    assert code == 0 and dig == oracle.blake3(b"\x00T")
    code, dig, _ = oracle.seqhash("uu", "DNA", False, True)
    assert code == 0 and dig == oracle.blake3(b"\x00\x00")


def test_mirror_messages_and_type_check():
    assert seqhash.Hash("ATGGGCTAA", "TNA", True, True)[1].args[0] == GOLDENS["errors"][0][4]
    assert [str(e) for _, e in seqhash.HashBatch(["A", "C"], "XNA", False, False)] == \
        ["Only sequenceTypes of DNA, RNA, or PROTEIN allowed. Got sequenceType: XNA"] * 2
    assert str(seqhash.item_error(1, 0, b"xTGG", seqhash.DNA)) == GOLDENS["errors"][1][4]
    assert str(seqhash.item_error(1, 3, b"MGCj*", seqhash.PROTEIN)) == GOLDENS["errors"][2][4]
    assert str(seqhash.item_error(2, 0, b"MGCS*", seqhash.PROTEIN)) == GOLDENS["errors"][3][4]
    assert isinstance(seqhash.item_error(3, 1, "aſ".encode(), seqhash.DNA), seqhash.UnsupportedError)
    assert seqhash.item_error(0, 0, b"", seqhash.DNA) is None
    assert seqhash.format_hash(bytes(range(32)), seqhash.RNA, True, False) == "v1_RCS_" + bytes(range(32)).hex()


def _no_gpu():
    n = C.c_int(0)
    _lib.lib().pg_device_count(C.byref(n))
    return n.value == 0


@pytest.mark.skipif(not _no_gpu(), reason="this check is for the GPU-less tier")
def test_seqhash_entry_points_fail_without_gpu():
    L = _lib.lib()
    seq = np.frombuffer(b"ACGT", np.uint8)
    off = np.array([0, 4], np.uint64)
    out = np.zeros(32, np.uint8)
    assert L.pg_seqhash_batch(seq.ctypes.data, off.ctypes.data, 1, 0, 0, out.ctypes.data, None, None) == _lib.PG_ERR_NO_DEVICE
    assert L.pg_seqhash_batch_dev(seq.ctypes.data, off.ctypes.data, 1, 0, 0, out.ctypes.data, None, None, 4, None) == _lib.PG_ERR_NO_DEVICE
    rot = np.zeros(1, np.uint64)
    assert L.pg_least_rotation_batch(seq.ctypes.data, off.ctypes.data, 1, rot.ctypes.data) == _lib.PG_ERR_NO_DEVICE
    with pytest.raises(_lib.PolyError) as e:
        seqhash.Hash("ACGT", seqhash.DNA, False, False)
    assert e.value.code == _lib.PG_ERR_NO_DEVICE
