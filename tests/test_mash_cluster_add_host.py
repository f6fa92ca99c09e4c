"""CPU tier of growing a clustering: argument checks that need no device."""
import ctypes as C

import numpy as np
import pytest

from poly_b200 import _lib, mash


def test_null_clusterer_is_an_argument_error():
    b = np.zeros((2, 16), np.uint32)
    label = np.zeros(2, np.uint32)
    L = _lib.lib()
    first, ng, nl, nm = (C.c_uint64(9) for _ in range(4))
    assert L.pg_mash_clusterer_add(None, b.ctypes.data, 2, 16, label.ctypes.data, C.byref(first), C.byref(ng), C.byref(nl),
                                   C.byref(nm)) == _lib.PG_ERR_ARG
    assert L.pg_mash_clusterer_add(None, None, 0, 0, None, None, None, None, None) == _lib.PG_ERR_ARG  # before m == 0 and s
    assert L.pg_mash_clusterer_add_dev(None, None, 2, 16, None, None, None, None, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_clusterer_add_dev(None, None, 0, -1, None, None, None, None, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_clusterer_labels(None, 0, 2, label.ctypes.data) == _lib.PG_ERR_ARG
    assert L.pg_mash_clusterer_labels(None, 0, 0, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_clusterer_labels_dev(None, 0, 0, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_clusterer_free(None) == _lib.PG_OK
    assert L.pg_mash_clusterer_index(None) is None


def test_create_rules_come_before_the_device():
    L = _lib.lib()
    h = C.c_void_p()
    # in order: a null out, then s <= 0, then min_same outside [1, s]
    assert L.pg_mash_clusterer_create(0, 0, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_clusterer_create(0, 0, C.byref(h)) == _lib.PG_ERR_PANIC
    assert L.pg_mash_clusterer_create(-3, 1, C.byref(h)) == _lib.PG_ERR_PANIC
    for bad in (0, 17):
        assert L.pg_mash_clusterer_create(16, bad, C.byref(h)) == _lib.PG_ERR_ARG and "min_same" in _lib.last_error()
    assert h.value is None


def test_python_thresholds_that_need_no_launch():
    with pytest.raises(ValueError):
        mash.Clusterer(16)
    with pytest.raises(ValueError):
        mash.Clusterer(16, min_same=1, max_distance=0.5)
    with pytest.raises(ValueError, match="every pair"):
        mash.Clusterer(16, max_distance=1.0)
    with pytest.raises(ValueError, match="no pair"):
        mash.Clusterer(16, max_distance=-0.25)
    with pytest.raises(_lib.GoPanic):
        mash.Clusterer(0, min_same=1)
    with pytest.raises(_lib.PolyError) as e:
        mash.Clusterer(16, min_same=17)
    assert e.value.code == _lib.PG_ERR_ARG
