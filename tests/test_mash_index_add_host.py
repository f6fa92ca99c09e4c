"""CPU tier of growing the sketch index: argument checks that need no device."""
import numpy as np

from poly_b200 import _lib


def test_null_index_is_an_argument_error():
    b = np.zeros((2, 16), np.uint32)
    L = _lib.lib()
    assert L.pg_mash_index_add(None, b.ctypes.data, 2, 16) == _lib.PG_ERR_ARG
    assert L.pg_mash_index_add(None, None, 0, 0) == _lib.PG_ERR_ARG  # before m == 0 and s
    assert L.pg_mash_index_add_dev(None, None, 2, 16, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_index_add_dev(None, None, 0, -1, None) == _lib.PG_ERR_ARG
