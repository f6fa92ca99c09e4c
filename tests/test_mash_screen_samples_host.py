"""CPU tier of the screen's several samples: the argument and handle rules that need no device."""
import ctypes as C

import numpy as np
import pytest

from poly_b200 import _lib, mash


def test_null_screen_is_an_argument_error_in_every_sample_call():
    L = _lib.lib()
    bases = np.frombuffer(b"ACGTACGT", np.uint8)
    off = np.array([0, 8], np.uint64)
    ids = np.zeros(1, np.uint32)
    out = np.zeros(1, np.uint32)
    assert L.pg_mash_screen_add_samples(None, bases.ctypes.data, off.ctypes.data, ids.ctypes.data, 1) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_add_samples(None, None, None, None, 0) == _lib.PG_ERR_ARG  # before n_reads == 0
    assert L.pg_mash_screen_add_samples_dev(None, None, None, None, 0, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_add_samples_dev(None, None, None, None, 5, None) == _lib.PG_ERR_ARG
    for fn in (L.pg_mash_screen_results_samples, L.pg_mash_screen_winners_samples):
        assert fn(None, 0, 1, out.ctypes.data, None, None) == _lib.PG_ERR_ARG
        assert fn(None, 0, 0, None, None, None) == _lib.PG_ERR_ARG
    for fn in (L.pg_mash_screen_results_samples_dev, L.pg_mash_screen_winners_samples_dev):
        assert fn(None, 0, 1, None, None, None, None) == _lib.PG_ERR_ARG


@pytest.mark.parametrize("dev", [False, True])
def test_create_samples_rules_come_before_the_device(dev):
    L = _lib.lib()
    sk = np.zeros((2, 4), np.uint32)
    h = C.c_void_p()

    def create(ptr, n, s, k, samples, out):
        if dev:
            return L.pg_mash_screen_create_samples_dev(ptr, n, s, k, samples, None, out)
        return L.pg_mash_screen_create_samples(ptr, n, s, k, samples, out)

    # in order: a null out, k < 0, s <= 0 with n > 0, n > 2^32 - 1, n_samples == 0, a null buffer
    assert create(sk.ctypes.data, 2, 4, 21, 1, None) == _lib.PG_ERR_ARG
    assert create(None, 2, 0, -1, 0, C.byref(h)) == _lib.PG_ERR_ARG and "k-mer" in _lib.last_error()
    assert create(None, 2, 0, 21, 0, C.byref(h)) == _lib.PG_ERR_PANIC
    assert create(None, 1 << 32, 4, 21, 0, C.byref(h)) == _lib.PG_ERR_ARG and "2^32" in _lib.last_error()
    assert create(None, 2, 4, 21, 0, C.byref(h)) == _lib.PG_ERR_ARG and "0 samples" in _lib.last_error()
    assert create(None, 0, 4, 21, 0, C.byref(h)) == _lib.PG_ERR_ARG and "0 samples" in _lib.last_error()  # no references still needs a sample
    assert create(None, 2, 4, 21, 3, C.byref(h)) == _lib.PG_ERR_ARG and "null" in _lib.last_error()
    assert h.value is None


def test_python_mirror_sample_rules_that_need_no_launch():
    with pytest.raises(_lib.PolyError) as e:
        mash.Screen(np.zeros((3, 4), np.uint32), 21, samples=0)
    assert e.value.code == _lib.PG_ERR_ARG
    with pytest.raises(_lib.PolyError) as e:
        mash.Screen(np.zeros((3, 4), np.uint32), 21, samples=1 << 32)
    assert e.value.code == _lib.PG_ERR_ARG
    with pytest.raises(_lib.PolyError) as e:
        mash.Screen(np.zeros((3, 4), np.uint32), 21, samples=-1)
    assert e.value.code == _lib.PG_ERR_ARG
    with pytest.raises(_lib.GoPanic):  # the existing rule order still holds with samples
        mash.Screen(np.zeros((3, 0), np.uint32), 21, samples=4)
