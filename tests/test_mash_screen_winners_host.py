"""CPU tier of the screen's winner-take-all: the argument rules of pg_mash_screen_winners(_dev) that need no device."""
import numpy as np

from poly_b200 import _lib


def test_null_screen_is_an_argument_error():
    L = _lib.lib()
    out = np.zeros(1, np.uint32)
    cont = np.zeros(1, np.float64)
    assert L.pg_mash_screen_winners(None, out.ctypes.data, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_winners(None, None, cont.ctypes.data, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_winners(None, None, None, None) == _lib.PG_ERR_ARG  # before the all-NULL no-op
    assert "null screen" in _lib.last_error()
    assert L.pg_mash_screen_winners_dev(None, None, None, None, None) == _lib.PG_ERR_ARG
    assert L.pg_mash_screen_winners_dev(None, out.ctypes.data, None, None, None) == _lib.PG_ERR_ARG


def test_winners_is_exported_beside_results():
    assert {"pg_mash_screen_winners", "pg_mash_screen_winners_dev"} <= set(_lib.EXPORTS)
    L = _lib.lib()
    assert L.pg_mash_screen_winners.argtypes == L.pg_mash_screen_results.argtypes
    assert L.pg_mash_screen_winners_dev.argtypes == L.pg_mash_screen_results_dev.argtypes
