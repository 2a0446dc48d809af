"""CPU tests of the text-recognition entry points: a NULL engine or a NULL argument comes back as a non-zero return and a message
before any device is touched."""
import ctypes as C

import numpy as np

from tests.util import pkg

eng = pkg.engine


def test_recognize_entry_points_reject_null_engine_and_null_arguments():
    L = eng.lib()
    img = np.zeros((4, 4, 3), np.uint8)
    chars = np.zeros((1, 24), np.int32)
    lengths = np.zeros(1, np.int32)
    scores = np.zeros(1, np.float64)
    u8 = (C.c_void_p * 1)(img.ctypes.data)
    n = (C.c_int * 1)(4)
    outs = (chars.ctypes.data, lengths.ctypes.data, scores.ctypes.data, None)
    for images, nx, ny in ((u8, n, n), (None, n, n), (u8, None, n), (u8, n, None)):
        calls = {
            "vitb200_recognize_u8": lambda: L.vitb200_recognize_u8(None, images, nx, ny, 1, None, *outs),
            "vitb200_recognize_u8_async": lambda: L.vitb200_recognize_u8_async(None, images, nx, ny, 1, *outs),
        }
        for name, call in calls.items():
            assert call() != 0, name
            assert b"null argument" in L.vitb200_last_error(), name
