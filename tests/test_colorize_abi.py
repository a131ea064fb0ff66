"""The C ABI of the coloured LiDAR map (boundary B8, include/lvba_b200.h): arguments are validated before any device work, and
without a device the stage refuses to run (there is no CPU fallback)."""
import ctypes as C

import numpy as np
import pytest


def _create(pkg, sp, xyz, ts, stride=3):
    lib = pkg.load_library()
    h = C.c_void_p()
    rc = lib.lvba_colorizer_create(C.c_int32(len(sp) - 1), pkg._p(sp, C.c_int64), pkg._p(xyz, C.c_float), C.c_int32(stride),
                                   pkg._p(ts, C.c_double), C.c_int32(-1), C.byref(h))
    return rc, h


def test_create_validates_before_device_work(pkg):
    xyz = np.zeros((10, 3), np.float32); ts = np.zeros(2)
    assert _create(pkg, np.array([0, 6, 4], np.int64), xyz, ts)[0] == -1          # scan_ptr not monotone
    assert _create(pkg, np.array([1, 4, 10], np.int64), xyz, ts)[0] == -1         # scan_ptr[0] != 0
    assert _create(pkg, np.array([0, 4, 10], np.int64), xyz, ts, stride=2)[0] == -1
    lib = pkg.load_library()
    assert lib.lvba_colorizer_create(C.c_int32(2), None, None, C.c_int32(3), None, C.c_int32(-1), None) == -1
    assert lib.lvba_colorizer_begin(None, None, C.c_double(0.5), C.c_double(0.01)) == -1
    assert lib.lvba_colorizer_finish(None, None, None) == -1
    assert lib.lvba_colorizer_export(None, None, None) == -1
    assert lib.lvba_colorizer_destroy(None) == 0


def test_no_device_is_an_error(pkg):
    if pkg.device_count() > 0:
        pytest.skip("a device is present")
    with pytest.raises(pkg.LvbaError) as e:
        pkg.Colorizer([np.zeros((5, 3), np.float32)], [0.0])
    assert e.value.status == -2
