"""CPU tests of the encoder-features entry points: argument errors come back as a non-zero return and a message before any device
is touched."""
import ctypes as C

import numpy as np

from tests.util import pkg

eng = pkg.engine


def test_features_entry_points_reject_null_engine_and_null_request():
    L = eng.lib()
    req = eng.FeaturesReq(1, 1, 0)
    img = np.zeros(16, np.float32)
    out = np.zeros(16, np.float32)
    u8 = (C.c_void_p * 1)(img.ctypes.data)
    n = (C.c_int * 1)(4)
    for r in (C.byref(req), None):
        calls = {
            "vitb200_features": lambda: L.vitb200_features(None, img.ctypes.data, 1, r, out.ctypes.data, None),
            "vitb200_features_device": lambda: L.vitb200_features_device(None, img.ctypes.data, 1, r, out.ctypes.data, None, None),
            "vitb200_features_u8": lambda: L.vitb200_features_u8(None, u8, n, n, 1, 0, r, out.ctypes.data, None),
        }
        for name, call in calls.items():
            assert call() != 0, name
            assert b"null argument" in L.vitb200_last_error(), name
