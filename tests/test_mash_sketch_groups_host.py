"""CPU tier of the grouped sketch (pg_mash_sketch_groups): every argument rule, in its order, before any device
work, and the Python mirror's rules."""
import numpy as np
import pytest

from poly_b200 import _lib, mash

ARG = _lib.PG_ERR_ARG


def call(dev, bases, off, n, goff, G, k=21, s=10, m=1, out=True, stride=None, count=True):
    L = _lib.lib()
    o = np.zeros(max(G, 1) * (stride or s), np.uint32)
    c = np.zeros(max(G, 1), np.uint32)
    args = (_lib.ptr(bases), _lib.ptr(off), n, _lib.ptr(goff), G, k, s, m, o.ctypes.data if out else None, stride if stride is not None else s,
            c.ctypes.data if count else None)
    if dev:
        return L.pg_mash_sketch_groups_dev(*args, None)
    return L.pg_mash_sketch_groups(*args)


@pytest.mark.parametrize("dev", [False, True])
def test_rules_in_order(dev):
    b = np.frombuffer(b"ACGTACGTAC", np.uint8)
    off = np.array([0, 4, 10], np.uint64)
    goff = np.array([0, 2], np.uint64)
    # every rule broken at once: the first one decides, then each is fixed in turn
    assert call(dev, None, None, 2, None, 1, k=-1, s=0, m=0, out=False, stride=0) == ARG and "null out" in _lib.last_error()
    assert call(dev, None, None, 2, None, 1, k=-1, s=0, m=0, count=False, stride=0) == ARG and "null out" in _lib.last_error()
    assert call(dev, None, None, 2, None, 1, k=-1, s=0, m=0, stride=0) == ARG and "kmerSize" in _lib.last_error()
    assert call(dev, None, None, 2, None, 1, s=0, m=0, stride=0) == ARG and "sketchSize" in _lib.last_error()
    assert call(dev, None, None, 2, None, 1, m=0, stride=0) == ARG and "min_copies" in _lib.last_error()
    assert call(dev, None, None, 2, None, 1, stride=9) == ARG and "row_stride" in _lib.last_error()
    assert call(dev, None, off, 2, goff, 1) == ARG and "null buffer" in _lib.last_error()
    assert call(dev, b, None, 2, goff, 1) == ARG and "null buffer" in _lib.last_error()
    assert call(dev, b, off, 2, None, 1) == ARG and "null buffer" in _lib.last_error()
    # no group: valid, no buffer needed, but the scalar rules still hold
    assert call(dev, None, None, 0, None, 0, out=False, count=False) == _lib.PG_OK
    assert call(dev, None, None, 5, None, 0, out=False, count=False) == _lib.PG_OK
    assert call(dev, None, None, 0, None, 0, s=0, out=False, count=False) == ARG


def test_host_offsets_rules():
    b = np.frombuffer(b"ACGTACGTAC", np.uint8)
    off = np.array([0, 4, 10], np.uint64)
    for goff in ([0, 1], [1, 2], [0, 3], [0, 2, 1], [0, 1, 0, 2]):
        g = np.array(goff, np.uint64)
        assert call(False, b, off, 2, g, len(g) - 1) == ARG, goff
    bad = np.array([0, 6, 4], np.uint64)
    assert call(False, b, bad, 2, np.array([0, 2], np.uint64), 1) == ARG and "decrease" in _lib.last_error()
    # the partition is checked before the record offsets
    assert call(False, b, bad, 2, np.array([0, 1], np.uint64), 1) == ARG and "group offsets" in _lib.last_error()


def test_python_mirror_rules():
    b, off, goff = np.zeros(4, np.uint8), np.array([0, 4], np.uint64), np.array([0, 1], np.uint64)
    for k, s, m in ((21, 0, 1), (21, 10, 0), (-1, 10, 1), (21, 1 << 31, 1), (21, 10, 1 << 32)):
        with pytest.raises(_lib.PolyError) as e:
            mash.sketch_groups(b, off, goff, k, s, m)
        assert e.value.code == ARG
    with pytest.raises(_lib.PolyError) as e:
        mash.sketch_groups(b, off, np.array([0, 2], np.uint64), 21, 10)
    assert e.value.code == ARG
    with pytest.raises(ValueError):
        mash.SketchGroups(["ACGT", "ACGT"], 21, 10)
    with pytest.raises(_lib.PolyError):
        mash.SketchGroups([["ACGT"]], 21, 10, min_copies=0)
    rows, count = mash.sketch_groups(b, np.zeros(1, np.uint64), np.zeros(1, np.uint64), 21, 10)
    assert rows.shape == (0, 10) and count.shape == (0,)
    assert mash.SketchGroups([], 21, 10) == []
