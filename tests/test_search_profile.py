"""The search launch's cycle accounting is compiled only into a library built with -DPINB200_SEARCH_PROFILE=1
(scripts/exp_decode.py prints its phase table); the default build has none and says so when asked for it."""
import ctypes

import numpy as np


def test_default_build_has_no_search_profile():
    """No GPU: the readback of the default build fails with an error instead of returning stale or zero counters."""
    from pin_slam_b200 import _lib

    lib = _lib.load()
    buf = np.zeros(132 * 4 * 4 * 8, dtype=np.uint64)
    assert lib.pinb200_debug_read(b"search_profile", buf.ctypes.data_as(ctypes.c_void_p), buf.size) != 0
    assert b"PINB200_SEARCH_PROFILE" in lib.pinb200_last_error()
    assert not buf.any()
