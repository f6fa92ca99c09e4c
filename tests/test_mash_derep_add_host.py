"""CPU tier of growing a dereplication: argument checks that need no device."""
import ctypes as C

import numpy as np
import pytest

from poly_b200 import _lib, mash


def test_null_dereplicator_is_an_argument_error():
    b = np.zeros((2, 16), np.uint32)
    rep = np.zeros(2, np.uint32)
    L = _lib.lib()
    first, n_new = C.c_uint64(9), C.c_uint64(9)
    assert L.pg_mash_dereplicator_add(None, b.ctypes.data, 2, 16, rep.ctypes.data, C.byref(first), C.byref(n_new)) == _lib.PG_ERR_ARG
    assert L.pg_mash_dereplicator_add(None, None, 0, 0, None, None, None) == _lib.PG_ERR_ARG  # before m == 0 and s
    assert L.pg_mash_dereplicator_add_dev(None, None, 2, 16, None, None, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_dereplicator_add_dev(None, None, 0, -1, None, None, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_dereplicator_reps(None, rep.ctypes.data, 2, C.byref(n_new)) == _lib.PG_ERR_ARG
    assert L.pg_mash_dereplicator_free(None) == _lib.PG_OK
    assert L.pg_mash_dereplicator_index(None) is None


def test_create_rules_come_before_the_device():
    L = _lib.lib()
    h = C.c_void_p()
    # in order: unknown flag bits, then s <= 0, then min_same outside [1, s]
    assert L.pg_mash_dereplicator_create(0, 0, 2, C.byref(h)) == _lib.PG_ERR_ARG and "flags" in _lib.last_error()
    assert L.pg_mash_dereplicator_create(0, 0, 1, C.byref(h)) == _lib.PG_ERR_PANIC
    assert L.pg_mash_dereplicator_create(-3, 1, 0, C.byref(h)) == _lib.PG_ERR_PANIC
    for bad in (0, 17):
        assert L.pg_mash_dereplicator_create(16, bad, 0, C.byref(h)) == _lib.PG_ERR_ARG and "min_same" in _lib.last_error()
    assert h.value is None
    assert L.pg_mash_dereplicator_create(16, 1, 0, None) == _lib.PG_ERR_ARG


def test_python_thresholds_that_need_no_launch():
    with pytest.raises(ValueError):
        mash.Dereplicator(16)
    with pytest.raises(ValueError):
        mash.Dereplicator(16, min_same=1, max_distance=0.5)
    with pytest.raises(ValueError, match="every pair"):
        mash.Dereplicator(16, max_distance=1.0)
    with pytest.raises(ValueError, match="no pair"):
        mash.Dereplicator(16, max_distance=-0.25, nearest=True)
    with pytest.raises(_lib.GoPanic):
        mash.Dereplicator(0, min_same=1)
    with pytest.raises(_lib.PolyError) as e:
        mash.Dereplicator(16, min_same=17)
    assert e.value.code == _lib.PG_ERR_ARG
