"""ctypes driver for the oracle's RGB-D depth model (oracle/rgbd_oracle.cpp): Tracking::GrabImageRGBD's depth conversion and
Frame::ComputeStereoFromRGBD.  TEST INFRASTRUCTURE, like pyoracle."""
import ctypes as C

import numpy as np

from oracle import pyoracle


def _lib():
    L = pyoracle.lib()
    L.orc_stereo_from_rgbd.restype = None
    L.orc_stereo_from_rgbd.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_float, C.c_float,
                                       C.c_void_p, C.c_void_p]
    return L


def stereo_from_rgbd(kps, depth, factor, bf):
    """Tracking::GrabImageRGBD's depth conversion + Frame::ComputeStereoFromRGBD restated (mvKeysUn = mvKeys).  kps: pyoracle.KP_DTYPE
    records; depth: (H, W) uint16 or float32 map (any row stride); factor: Tracking::mDepthMapFactor.  Returns (mvuRight, mvDepth)."""
    assert depth.dtype in (np.uint16, np.float32) and depth.ndim == 2 and depth.strides[1] == depth.itemsize
    kps = np.ascontiguousarray(kps)
    uR = np.zeros(max(len(kps), 1), np.float32)
    dep = np.zeros(max(len(kps), 1), np.float32)
    _lib().orc_stereo_from_rgbd(C.c_void_p(kps.ctypes.data), len(kps), C.c_void_p(depth.ctypes.data), 1 if depth.dtype == np.uint16 else 2,
                                depth.strides[0], depth.shape[1], depth.shape[0], float(factor), float(bf), C.c_void_p(uR.ctypes.data),
                                C.c_void_p(dep.ctypes.data))
    return uR[:len(kps)], dep[:len(kps)]
