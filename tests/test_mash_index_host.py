"""CPU tier of the sketch index: the max_distance -> min_same conversion, and no CPU fallback."""
import ctypes as C

import numpy as np
import pytest

from poly_b200 import _lib, mash


@pytest.mark.parametrize("den", [1, 3, 7, 10, 100, 499, 500, 1000, 2000, 4096, 16384])
def test_max_distance_to_min_same_agrees_with_f64_expression(den):
    same = np.arange(den + 1, dtype=np.float64)
    dist = 1 - same / np.float64(den)  # mash.go:134,139
    cuts = sorted(set(dist[:: max(1, den // 256)].tolist()) | set(dist[-8:].tolist()) | {0.0, 1.0, -0.5, 1.5, 0.5, 0.1, 0.9, 1e-12, np.nextafter(1.0, 0.0)})
    for md in cuts + [np.nextafter(x, 2.0) for x in cuts] + [np.nextafter(x, -1.0) for x in cuts]:
        m = mash.min_same_for_distance(md, den)
        keep = dist <= md
        assert keep.tolist() == (np.arange(den + 1) >= m).tolist(), (den, md, m)


def _no_gpu():
    n = C.c_int(0)
    _lib.lib().pg_device_count(C.byref(n))
    return n.value == 0


@pytest.mark.skipif(not _no_gpu(), reason="this check is for the GPU-less tier")
def test_index_creation_fails_without_device():
    with pytest.raises(_lib.PolyError) as e:
        mash.SketchIndex(np.arange(64, dtype=np.uint32).reshape(4, 16))
    assert e.value.code == _lib.PG_ERR_NO_DEVICE
    h = C.c_void_p()
    assert _lib.lib().pg_mash_index_create(np.zeros(16, np.uint32).ctypes.data, 1, 16, C.byref(h)) == _lib.PG_ERR_NO_DEVICE
    assert not h.value
