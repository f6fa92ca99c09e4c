"""CPU tier of the screen: the argument and handle rules that need no device."""
import ctypes as C

import numpy as np
import pytest

from poly_b200 import _lib, mash


def test_null_screen_is_an_argument_error():
    L = _lib.lib()
    bases = np.frombuffer(b"ACGTACGT", np.uint8)
    off = np.array([0, 8], np.uint64)
    out = np.zeros(1, np.uint32)
    assert L.pg_mash_screen_add(None, bases.ctypes.data, off.ctypes.data, 1) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_add(None, None, None, 0) == _lib.PG_ERR_ARG  # before n_reads == 0
    assert L.pg_mash_screen_add_dev(None, None, None, 0, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_reset(None) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_results(None, out.ctypes.data, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_results(None, None, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_results_dev(None, None, None, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_free(None) == _lib.PG_OK


@pytest.mark.parametrize("dev", [False, True])
def test_create_rules_come_before_the_device(dev):
    L = _lib.lib()
    sk = np.zeros((2, 4), np.uint32)
    h = C.c_void_p()

    def create(ptr, n, s, k, out):
        if dev:
            return L.pg_mash_screen_create_dev(ptr, n, s, k, None, out)
        return L.pg_mash_screen_create(ptr, n, s, k, out)

    # in order: a null out, k < 0, s <= 0 with n > 0, n > 2^32 - 1, a null buffer
    assert create(sk.ctypes.data, 2, 4, 21, None) == _lib.PG_ERR_ARG
    assert create(None, 2, 0, -1, C.byref(h)) == _lib.PG_ERR_ARG and "k-mer" in _lib.last_error()
    assert create(None, 2, 0, 21, C.byref(h)) == _lib.PG_ERR_PANIC
    assert create(None, 2, -5, 21, C.byref(h)) == _lib.PG_ERR_PANIC
    assert create(None, 1 << 32, 4, 21, C.byref(h)) == _lib.PG_ERR_ARG and "2^32" in _lib.last_error()
    assert create(None, 2, 4, 21, C.byref(h)) == _lib.PG_ERR_ARG and "null" in _lib.last_error()
    assert h.value is None


def test_python_mirror_rules_that_need_no_launch():
    with pytest.raises(_lib.GoPanic):
        mash.Screen(np.zeros((3, 0), np.uint32), 21)
    with pytest.raises(_lib.PolyError) as e:
        mash.Screen(np.zeros((3, 4), np.uint32), -1)
    assert e.value.code == _lib.PG_ERR_ARG
    with pytest.raises(ValueError):
        mash.Screen(np.zeros(4, np.uint32), 21)
