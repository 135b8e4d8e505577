"""ctypes driver for the oracle's camera-image models (oracle/ingest_oracle.cpp): System::Track*'s cv::resize and
Tracking::GrabImage*'s cv::cvtColor to grey.  TEST INFRASTRUCTURE, like pyoracle."""
import ctypes as C

import numpy as np

from oracle import pyoracle

FORMATS = {"gray": 0, "rgb": 1, "bgr": 2, "rgba": 3, "bgra": 4}
CHANNELS = {0: 1, 1: 3, 2: 3, 3: 4, 4: 4}


def _lib():
    L = pyoracle.lib()
    L.orc_ingest.restype = C.c_int
    L.orc_ingest.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int]
    return L


def ingest(img, fmt, size=None):
    """img: (H, W) or (H, W, C) uint8 (any row stride); fmt: a FORMATS key or value; size: (width, height) of the result, None = the
    image's own.  Returns the (height, width) grey image Frame::Frame would see."""
    fmt = FORMATS.get(fmt, fmt)
    assert img.dtype == np.uint8 and img.shape[2:] == ((CHANNELS[fmt],) if img.ndim == 3 else ())
    assert img.strides[-1] == 1 and (img.ndim == 2 or img.strides[1] == CHANNELS[fmt])
    sh, sw = img.shape[:2]
    dw, dh = size or (sw, sh)
    out = np.zeros((dh, dw), np.uint8)
    assert _lib().orc_ingest(C.c_void_p(img.ctypes.data), fmt, sw, sh, img.strides[0], C.c_void_p(out.ctypes.data), dw, dh) == 0
    return out
