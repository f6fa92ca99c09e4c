"""CPU tier of the grouped sketch grown in place (pg_mash_sketcher): the create rules in their order, the null-handle
rules of add, add_dev, rows and rows_dev (no device needed), the Python mirror's rules, and the restatement in
tests/sketcher_oracle.py against the one-shot restatement in tests/sketch_groups_oracle.py on random splits.  The add
and rows rules that need a live sketcher are checked in tests/test_gpu_mash_sketcher.py."""
import ctypes as C

import numpy as np
import pytest

import sketch_groups_oracle
import sketcher_oracle
from poly_b200 import _lib, mash

ARG = _lib.PG_ERR_ARG
ACGT = np.frombuffer(b"ACGT", np.uint8)


def create(G=2, k=21, s=10, m=1, B=None, out=True):
    h = C.c_void_p()
    rc = _lib.lib().pg_mash_sketcher_create(G, k, s, m, 64 * s if B is None else B, C.byref(h) if out else None)
    return rc, h


def test_create_rules_in_order():
    # every rule broken at once: the first one decides, then each is fixed in turn
    assert create(G=0, k=-1, s=0, m=0, B=0, out=False)[0] == ARG and "null sketcher pointer" in _lib.last_error()
    assert create(G=0, k=-1, s=0, m=0, B=0)[0] == ARG and "groups" in _lib.last_error()
    assert create(G=1 << 32, k=-1, s=0, m=0, B=0)[0] == ARG and "groups" in _lib.last_error()
    assert create(k=-1, s=0, m=0, B=0)[0] == ARG and "kmerSize" in _lib.last_error()
    assert create(s=0, m=0, B=0)[0] == ARG and "sketchSize" in _lib.last_error()
    assert create(m=0, B=0)[0] == ARG and "min_copies" in _lib.last_error()
    assert create(B=9)[0] == ARG and "max_values" in _lib.last_error()
    rc, h = create(G=(1 << 32) - 1, B=10)  # every rule met: only the device (or host memory) can refuse it now
    if rc == _lib.PG_OK:
        _lib.check(_lib.lib().pg_mash_sketcher_free(h))
    else:
        assert rc in (_lib.PG_ERR_NO_DEVICE, _lib.PG_ERR_NOMEM)


def test_null_sketcher_rules():
    L = _lib.lib()
    b, off, goff = np.zeros(4, np.uint8), np.array([0, 4], np.uint64), np.array([0, 1], np.uint64)
    out, n = np.zeros(10, np.uint32), np.zeros(1, np.uint32)
    assert L.pg_mash_sketcher_add(None, b.ctypes.data, off.ctypes.data, 1, goff.ctypes.data, 0, 1) == ARG and "null sketcher" in _lib.last_error()
    assert L.pg_mash_sketcher_add(None, None, None, 0, None, 0, 0) == ARG
    assert L.pg_mash_sketcher_add_dev(None, None, None, 0, None, 0, 0, None) == ARG and "null sketcher" in _lib.last_error()
    assert L.pg_mash_sketcher_rows(None, 0, 1, out.ctypes.data, 10, n.ctypes.data, None, None) == ARG and "null sketcher" in _lib.last_error()
    assert L.pg_mash_sketcher_rows_dev(None, 0, 0, None, 10, None, None, None, None) == ARG
    assert L.pg_mash_sketcher_free(None) == _lib.PG_OK


def test_python_mirror_rules():
    for args in ((2, 21, 0), (2, 21, 10, 0), (2, -1, 10), (2, 21, 1 << 31), (2, 21, 10, 1 << 32)):
        with pytest.raises(_lib.PolyError) as e:
            mash.Sketcher(*args)
        assert e.value.code == ARG
    for kw in ({"max_values": 9}, {"max_values": -1}, {"max_values": 1 << 64}):
        with pytest.raises(_lib.PolyError) as e:
            mash.Sketcher(2, 21, 10, **kw)
        assert e.value.code == ARG
    with pytest.raises(_lib.PolyError) as e:
        mash.Sketcher(0, 21, 10)
    assert e.value.code == ARG


def rand_groups(rng, G, k):
    """G groups of 0..30 records (0..400 bytes) cut from a small per-group source, so values recur."""
    groups = []
    for _ in range(G):
        src = ACGT[rng.integers(0, 4, int(rng.integers(k + 50, 1500)))]
        recs = []
        for _ in range(int(rng.integers(0, 31))):
            L = int(min(rng.integers(0, 401), len(src)))
            a = int(rng.integers(0, len(src) - L + 1))
            recs.append(src[a:a + L].copy())
        groups.append(recs)
    return groups


def random_adds(rng, groups):
    """The records of every group, in order, as adds of (first group, [records per group]): each add starts where the
    last one stopped, takes 0..3 groups' worth of records, and may begin or end inside a group."""
    flat = [(g, r) for g, recs in enumerate(groups) for r in recs]
    adds, i = [], 0
    while i < len(flat) or not adds:
        n = int(rng.integers(0, 12))
        part = flat[i:i + n]
        i += n
        if not part:
            adds.append((int(rng.integers(0, len(groups))), [[]]))
            continue
        first = part[0][0]
        per = [[] for _ in range(part[-1][0] - first + 1)]
        for g, r in part:
            per[g - first].append(r)
        adds.append((first, per))
    return adds


@pytest.mark.parametrize("m", [1, 2, 3])
@pytest.mark.parametrize("s,B", [(1, 1), (5, 5), (5, 10), (20, 20), (20, 80), (50, 3200)])
def test_restatement_against_the_one_shot(m, s, B):
    rng = np.random.default_rng(100 * m + s + B)
    k, G = 11, 5
    groups = rand_groups(rng, G, k)
    sk = sketcher_oracle.Sketcher(G, k, s, m, B)
    done = [[] for _ in range(G)]
    for first, per in random_adds(rng, groups):
        bases, off, goff = sketch_groups_oracle.flatten_groups(per)
        sk.add(bases, off, goff, first)
        for i, recs in enumerate(per):
            done[first + i] += recs
        rows, count, complete, held = sk.rows()
        b2, o2, g2 = sketch_groups_oracle.flatten_groups(done)
        want_rows, want_count = sketch_groups_oracle.sketch_groups(b2, o2, g2, k, s, m)
        for g in range(G):
            c = int(count[g])
            assert c <= want_count[g] and rows[g, :c].tobytes() == want_rows[g, :c].tobytes()  # always a prefix
            assert not rows[g, c:].any()
            if complete[g]:
                assert c == want_count[g] and rows[g].tobytes() == want_rows[g].tobytes()
            assert held[g] <= B
            if m == 1:
                assert complete[g] and held[g] <= s
